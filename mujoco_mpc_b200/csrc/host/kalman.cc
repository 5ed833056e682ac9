// kalman.cc - see kalman.h.
#include "kalman.h"

#include <algorithm>

namespace mjpc_b200_host {

int Kalman::Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep_, double epsilon_,
                       bool centered_, int device) {
  if (!(epsilon_ > 0)) { error = "kalman: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  epsilon = epsilon_; centered = centered_;
  if (int rc = InitializeBase(model, sensor_start, nsensor, timestep_, device)) return rc;
  nstates = (centered ? 2 : 1) * ndstate + 1;
  jacobian_.resize((size_t)std::max(nsensordata, ndstate) * ndstate);
  return 0;
}

void Kalman::Reset(const double* s, double t, double covariance_scale, double process_scale, double sensor_scale) {
  Estimator::Reset(s, t, covariance_scale, process_scale, sensor_scale);
  ctrl_.assign(m_.nu, 0.0);
  mocap_ = mocap0_;
}

int Kalman::Perturbed(const double* ctrl, const float* mocap) {
  const int nq = m_.nq, nv = m_.nv, nx = nq + nv;
  std::vector<double> dq(nv, 0.0);
  for (int r = 0; r < nstates; r++) {
    double* x = &states_[(size_t)r * nx];
    std::copy(state.begin(), state.end(), x);
    if (r > 0) {
      const int i = (r - 1) % ndstate;
      const double e = r - 1 < ndstate ? epsilon : -epsilon;
      // positions through IntegratePos, velocities added: not StateAdd, whose IntegratePos would renormalise the
      // quaternions of a velocity perturbation too
      if (i < nv) {
        dq[i] = 1.0;
        IntegratePos(m_, x, dq.data(), e);
        dq[i] = 0.0;
      } else {
        x[nq + i - nv] += e;
      }
    }
  }
  return StepSensors(nstates, ctrl, mocap);
}

int Kalman::UpdateMeasurement(const double* ctrl, const double* sensor, const float* mocap) {
  if (!engine_ || (!ctrl && m_.nu) || !sensor) { error = "kalman update: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = Perturbed(ctrl, mocap)) return rc;
  const int ny = nsensordata, ns = ndstate;
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
  // correction = P C' S^-1 (y - y_hat), P -= P C' S^-1 C P
  std::vector<double> e(ny), corr(ns);
  for (int k = 0; k < ny; k++) e[k] = sensor[k] - (double)y0[k];
  if (int rc = GainUpdate(PCt.data(), S.data(), e.data(), covariance.data(), corr.data(), covariance.data())) return rc;
  StateAdd(state.data(), corr.data(), 1.0);
  ctrl_.assign(ctrl, ctrl + m_.nu);
  if (mocap) mocap_.assign(mocap, mocap + 7 * (size_t)nmocap_); else mocap_ = mocap0_;
  Commit(0);
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
  Symmetrize(covariance.data());
  state = next;
  time += timestep;
  Commit(0);
  return 0;
}

int Kalman::Update(const double* ctrl, const double* sensor, const float* mocap) {
  if (int rc = UpdateMeasurement(ctrl, sensor, mocap)) return rc;
  return UpdatePrediction();
}

void Kalman::GetScalars(double* scalars) const {
  scalars[0] = ndstate; scalars[1] = nstates; scalars[2] = nsensordata; scalars[3] = warnings; scalars[4] = timestep;
  scalars[5] = epsilon;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using namespace mjpc_b200_host;

extern "C" {

int mjpc_b200_kalman_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                            double epsilon, int centered, int device, mjpc_b200_estimator_t** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* k = new Kalman;
  if (int rc = k->Initialize(model, sensor_start, nsensor, timestep, epsilon, centered != 0, device)) {
    delete k;
    return rc;
  }
  *out = ToHandle(k);
  return 0;
}

int mjpc_b200_kalman_update_measurement(mjpc_b200_estimator_t* h, const double* ctrl, const double* sensor,
                                        const float* mocap) {
  Kalman* k = EstimatorOf<Kalman>(h);
  return k ? k->UpdateMeasurement(ctrl, sensor, mocap) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_kalman_update_prediction(mjpc_b200_estimator_t* h) {
  Kalman* k = EstimatorOf<Kalman>(h);
  return k ? k->UpdatePrediction() : MJPC_B200_ERR_BAD_ARGUMENT;
}

}  // extern "C"
