// kalman.cc - see kalman.h.
#include "kalman.h"

#include <algorithm>
#include <cstring>

#include "planner.h"
#include "unscented.h"

namespace mjpc_b200_host {

Kalman::~Kalman() { if (engine_) mjpc_b200_destroy(engine_); }

int Kalman::Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep_, double epsilon_,
                       bool centered_, int device) {
  if (!model || !(timestep_ > 0) || !(epsilon_ > 0)) { error = "kalman: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = m_.Load(model)) { error = "kalman: bad blob"; return rc; }
  std::vector<int> dims;
  if (LoadEstimatorBlob(model, m_, &dims, &nmocap_, &mocap0_, &key_state_)) {
    error = "kalman: blob without sensor entries";
    return MJPC_B200_ERR_BAD_BLOB;
  }
  if (sensor_start < 0 || nsensor < 1 || sensor_start > (int)dims.size() - nsensor) {
    error = "kalman: sensor range outside the model's sensors";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  sensor_start_ = sensor_start; nsensor_ = nsensor;
  nsensordata = 0;
  for (int i = sensor_start; i < sensor_start + nsensor; i++) nsensordata += dims[i];
  timestep = timestep_; epsilon = epsilon_; centered = centered_;
  ndstate = 2 * m_.nv;
  nstates = (centered ? 2 : 1) * ndstate + 1;
  if (int rc = mjpc_b200_create(model, 2 * ndstate + 1, 1, device, &engine_)) { error = mjpc_b200_last_error(); return rc; }
  if (int rc = mjpc_b200_set_options(engine_, timestep, 0)) { error = mjpc_b200_last_error(); return rc; }
  const size_t ns = nstates, nx = m_.nq + m_.nv;
  jacobian_.resize((size_t)std::max(nsensordata, ndstate) * ndstate);
  fstates_.resize(ns * nx); fnext_.resize(ns * nx); fsensor_.resize(ns * nsensordata); fqacc_.resize(ns * m_.nv);
  fwarm_.resize(ns * m_.nv); counts_.resize(4 * ns);
  Reset(nullptr, 0.0, 1e-4, 1e-4, 1e-4);
  // one step of the reset state: the engine refuses a sensor in the range that it does not evaluate
  if (int rc = Perturbed(ctrl_.data(), nullptr)) return rc;
  Reset(nullptr, 0.0, 1e-4, 1e-4, 1e-4);
  return 0;
}

void Kalman::Reset(const double* s, double t, double covariance_scale, double process_scale, double sensor_scale) {
  state.assign(s ? s : key_state_.data(), (s ? s : key_state_.data()) + m_.nq + m_.nv);
  time = t;
  covariance.assign((size_t)ndstate * ndstate, 0.0);
  for (int i = 0; i < ndstate; i++) covariance[(size_t)i * ndstate + i] = covariance_scale;
  noise_process.assign(ndstate, process_scale);
  noise_sensor.assign(nsensordata, sensor_scale);
  qacc_warmstart_.assign(m_.nv, 0.0);
  ctrl_.assign(m_.nu, 0.0);
  mocap_ = mocap0_;
  warnings = 0;
}

int Kalman::Perturbed(const double* ctrl, const float* mocap) {
  const int nq = m_.nq, nv = m_.nv, nx = nq + nv;
  std::vector<double> x(nx), dq(nv, 0.0);
  for (int r = 0; r < nstates; r++) {
    x = state;
    if (r > 0) {
      const int i = (r - 1) % ndstate;
      const double e = r - 1 < ndstate ? epsilon : -epsilon;
      if (i < nv) {
        dq[i] = 1.0;
        IntegratePos(m_, x.data(), dq.data(), e);
        dq[i] = 0.0;
      } else {
        x[nq + i - nv] += e;
      }
    }
    for (int k = 0; k < nx; k++) fstates_[(size_t)r * nx + k] = (float)x[k];
    for (int k = 0; k < nv; k++) fwarm_[(size_t)r * nv + k] = (float)qacc_warmstart_[k];
  }
  std::vector<float> u(m_.nu);
  for (int k = 0; k < m_.nu; k++) u[k] = (float)ctrl[k];
  if (int rc = mjpc_b200_step_sensors(engine_, nstates, fstates_.data(), u.data(), fwarm_.data(),
                                      mocap ? mocap : mocap0_.data(), time, sensor_start_, nsensor_, fnext_.data(),
                                      fsensor_.data(), fqacc_.data(), counts_.data())) {
    error = mjpc_b200_last_error();
    return rc;
  }
  return 0;
}

int Kalman::UpdateMeasurement(const double* ctrl, const double* sensor, const float* mocap) {
  if (!engine_ || (!ctrl && m_.nu) || !sensor) { error = "kalman update: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = Perturbed(ctrl, mocap)) return rc;
  const int ny = nsensordata, ns = ndstate, nq = m_.nq, nv = m_.nv;
  // C [ny][ns] from the sensor differences, y_hat = the centre's sensors
  double* C = jacobian_.data();
  const float* y0 = fsensor_.data();
  for (int i = 0; i < ns; i++) {
    const float* yp = &fsensor_[(size_t)(1 + i) * ny];
    const float* ym = centered ? &fsensor_[(size_t)(1 + ns + i) * ny] : y0;
    const double h = centered ? 2 * epsilon : epsilon;
    for (int r = 0; r < ny; r++) C[(size_t)r * ns + i] = ((double)yp[r] - (double)ym[r]) / h;
  }
  // P C' [ns][ny], S = C P C' + R
  std::vector<double> PCt((size_t)ns * ny, 0.0), S((size_t)ny * ny, 0.0);
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ny; c++) {
      double a = 0;
      for (int k = 0; k < ns; k++) a += covariance[(size_t)r * ns + k] * C[(size_t)c * ns + k];
      PCt[(size_t)r * ny + c] = a;
    }
  for (int r = 0; r < ny; r++)
    for (int c = 0; c < ny; c++) {
      double a = 0;
      for (int k = 0; k < ns; k++) a += C[(size_t)r * ns + k] * PCt[(size_t)k * ny + c];
      S[(size_t)r * ny + c] = a + (r == c ? noise_sensor[r] : 0.0);
    }
  if (CholFactor(S.data(), ny, 1e-15) < ny) {
    error = "kalman update: sensor covariance factorisation failed";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  // correction = P C' S^-1 (y - y_hat)
  std::vector<double> e(ny), corr(ns, 0.0);
  for (int k = 0; k < ny; k++) e[k] = sensor[k] - (double)y0[k];
  CholSolve(S.data(), ny, e.data());
  for (int r = 0; r < ns; r++) for (int c = 0; c < ny; c++) corr[r] += PCt[(size_t)r * ny + c] * e[c];
  // P -= P C' S^-1 C P, symmetrised
  std::vector<double> T(PCt);
  for (int r = 0; r < ns; r++) CholSolve(S.data(), ny, &T[(size_t)r * ny]);
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ns; c++) {
      double a = 0;
      for (int k = 0; k < ny; k++) a += PCt[(size_t)r * ny + k] * T[(size_t)c * ny + k];
      covariance[(size_t)r * ns + c] -= a;
    }
  for (int r = 0; r < ns; r++)
    for (int c = r + 1; c < ns; c++) {
      const double s = 0.5 * (covariance[(size_t)r * ns + c] + covariance[(size_t)c * ns + r]);
      covariance[(size_t)r * ns + c] = covariance[(size_t)c * ns + r] = s;
    }
  IntegratePos(m_, state.data(), corr.data(), 1.0);
  for (int k = 0; k < nv; k++) state[nq + k] += corr[nv + k];
  ctrl_.assign(ctrl, ctrl + m_.nu);
  if (mocap) mocap_.assign(mocap, mocap + 7 * (size_t)nmocap_); else mocap_ = mocap0_;
  for (int k = 0; k < nv; k++) qacc_warmstart_[k] = fqacc_[k];
  for (int i = 0; i < nstates; i++) warnings += counts_[4 * i + 3] != 0;
  return 0;
}

int Kalman::UpdatePrediction() {
  if (!engine_) { error = "kalman prediction: no engine"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = Perturbed(ctrl_.data(), mocap_.data())) return rc;
  const int ns = ndstate, nx = m_.nq + m_.nv;
  // A [ns][ns]: column i = (next(x (+) eps e_i) (-) next(x [(+) -eps e_i])) / h
  std::vector<double> a(nx), b(nx), col(ns);
  double* A = jacobian_.data();
  for (int k = 0; k < nx; k++) b[k] = fnext_[k];
  std::vector<double> next(b);
  for (int i = 0; i < ns; i++) {
    for (int k = 0; k < nx; k++) a[k] = fnext_[(size_t)(1 + i) * nx + k];
    if (centered)
      for (int k = 0; k < nx; k++) b[k] = fnext_[(size_t)(1 + ns + i) * nx + k];
    StateDiff(m_, col.data(), a.data(), b.data());
    const double h = centered ? 2 * epsilon : epsilon;
    for (int r = 0; r < ns; r++) A[(size_t)r * ns + i] = col[r] / h;
  }
  // P = A P A' + diag(process noise), symmetrised
  std::vector<double> PAt((size_t)ns * ns, 0.0);
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ns; c++) {
      double s = 0;
      for (int k = 0; k < ns; k++) s += covariance[(size_t)r * ns + k] * A[(size_t)c * ns + k];
      PAt[(size_t)r * ns + c] = s;
    }
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ns; c++) {
      double s = 0;
      for (int k = 0; k < ns; k++) s += A[(size_t)r * ns + k] * PAt[(size_t)k * ns + c];
      covariance[(size_t)r * ns + c] = s + (r == c ? noise_process[r] : 0.0);
    }
  for (int r = 0; r < ns; r++)
    for (int c = r + 1; c < ns; c++) {
      const double s = 0.5 * (covariance[(size_t)r * ns + c] + covariance[(size_t)c * ns + r]);
      covariance[(size_t)r * ns + c] = covariance[(size_t)c * ns + r] = s;
    }
  state = next;
  time += timestep;
  for (int k = 0; k < m_.nv; k++) qacc_warmstart_[k] = fqacc_[k];
  for (int i = 0; i < nstates; i++) warnings += counts_[4 * i + 3] != 0;
  return 0;
}

int Kalman::Update(const double* ctrl, const double* sensor, const float* mocap) {
  if (int rc = UpdateMeasurement(ctrl, sensor, mocap)) return rc;
  return UpdatePrediction();
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using mjpc_b200_host::Kalman;

extern "C" {

int mjpc_b200_kalman_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                            double epsilon, int centered, int device, mjpc_b200_kalman_t** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* k = new Kalman;
  if (int rc = k->Initialize(model, sensor_start, nsensor, timestep, epsilon, centered != 0, device)) {
    delete k;
    return rc;
  }
  *out = reinterpret_cast<mjpc_b200_kalman_t*>(k);
  return 0;
}

void mjpc_b200_kalman_destroy(mjpc_b200_kalman_t* k) { delete reinterpret_cast<Kalman*>(k); }

int mjpc_b200_kalman_reset(mjpc_b200_kalman_t* k, const double* state, double time, double covariance_scale,
                           double process_scale, double sensor_scale) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  reinterpret_cast<Kalman*>(k)->Reset(state, time, covariance_scale, process_scale, sensor_scale);
  return 0;
}

int mjpc_b200_kalman_set_noise(mjpc_b200_kalman_t* k, const double* process, const double* sensor) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  Kalman* f = reinterpret_cast<Kalman*>(k);
  if (process) f->noise_process.assign(process, process + f->ndstate);
  if (sensor) f->noise_sensor.assign(sensor, sensor + f->nsensordata);
  return 0;
}

int mjpc_b200_kalman_set(mjpc_b200_kalman_t* k, const double* state, const double* covariance, double time) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  Kalman* f = reinterpret_cast<Kalman*>(k);
  if (state) f->state.assign(state, state + f->state.size());
  if (covariance) f->covariance.assign(covariance, covariance + f->covariance.size());
  f->time = time;
  return 0;
}

int mjpc_b200_kalman_update_measurement(mjpc_b200_kalman_t* k, const double* ctrl, const double* sensor,
                                        const float* mocap) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  return reinterpret_cast<Kalman*>(k)->UpdateMeasurement(ctrl, sensor, mocap);
}

int mjpc_b200_kalman_update_prediction(mjpc_b200_kalman_t* k) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  return reinterpret_cast<Kalman*>(k)->UpdatePrediction();
}

int mjpc_b200_kalman_update(mjpc_b200_kalman_t* k, const double* ctrl, const double* sensor, const float* mocap) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  return reinterpret_cast<Kalman*>(k)->Update(ctrl, sensor, mocap);
}

int mjpc_b200_kalman_get(const mjpc_b200_kalman_t* k, double* state, double* covariance, double* time,
                         double* scalars) {
  if (!k) return MJPC_B200_ERR_BAD_ARGUMENT;
  const Kalman* f = reinterpret_cast<const Kalman*>(k);
  if (state) std::copy(f->state.begin(), f->state.end(), state);
  if (covariance) std::copy(f->covariance.begin(), f->covariance.end(), covariance);
  if (time) *time = f->time;
  if (scalars) {
    scalars[0] = f->ndstate; scalars[1] = f->nstates; scalars[2] = f->nsensordata; scalars[3] = f->warnings;
    scalars[4] = f->timestep; scalars[5] = f->epsilon;
  }
  return 0;
}

const char* mjpc_b200_kalman_last_error(const mjpc_b200_kalman_t* k) {
  return k ? reinterpret_cast<const Kalman*>(k)->error.c_str() : "";
}

}  // extern "C"
