// estimator.cc - see estimator.h.
#include "estimator.h"

#include <algorithm>

#include "../dev_model.h"   // Blob reader (plain C++)

namespace mjpc_b200_host {

int LoadEstimatorBlob(const mjpc_model_blob* model, const HostModel& m, std::vector<int>* dims, int* nmocap,
                      std::vector<float>* mocap0, std::vector<double>* key_state) {
  try {
    mjpc_dev::Blob b(model->data, model->nbytes);
    *dims = b.ints("sensor_dim");
    *nmocap = b.i("nmocap");
    const std::vector<int> mid = b.ints("body_mocapid");
    const std::vector<double> bp = b.reals("body_pos"), bq = b.reals("body_quat"), q0 = b.reals("qpos0");
    mocap0->assign(7 * (size_t)*nmocap, 0.f);
    for (size_t i = 0; i < mid.size(); i++)
      if (mid[i] >= 0) {
        for (int c = 0; c < 3; c++) (*mocap0)[7 * mid[i] + c] = (float)bp[3 * i + c];
        for (int c = 0; c < 4; c++) (*mocap0)[7 * mid[i] + 3 + c] = (float)bq[4 * i + c];
      }
    const int nkey = b.i("nkey");
    key_state->assign(m.nq + m.nv, 0.0);
    if (nkey > 0) {
      const std::vector<double> kq = b.reals("key_qpos"), kv = b.reals("key_qvel");
      std::copy(kq.begin(), kq.begin() + m.nq, key_state->begin());
      std::copy(kv.begin(), kv.begin() + m.nv, key_state->begin() + m.nq);
    } else {
      std::copy(q0.begin(), q0.end(), key_state->begin());
    }
  } catch (const std::exception&) {
    return MJPC_B200_ERR_BAD_BLOB;
  }
  return 0;
}

Estimator::~Estimator() { if (engine_) mjpc_b200_destroy(engine_); }

int Estimator::InitializeBase(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep_,
                              int device) {
  const std::string name(name_);
  if (!model || !(timestep_ > 0)) { error = name + ": bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = m_.Load(model)) { error = name + ": bad blob"; return rc; }
  std::vector<int> dims;
  if (LoadEstimatorBlob(model, m_, &dims, &nmocap_, &mocap0_, &key_state_)) {
    error = name + ": blob without sensor entries";
    return MJPC_B200_ERR_BAD_BLOB;
  }
  if (sensor_start < 0 || nsensor < 1 || sensor_start > (int)dims.size() - nsensor) {
    error = name + ": sensor range outside the model's sensors";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  sensor_start_ = sensor_start; nsensor_ = nsensor;
  nsensordata = 0;
  for (int i = sensor_start; i < sensor_start + nsensor; i++) nsensordata += dims[i];
  timestep = timestep_;
  ndstate = 2 * m_.nv;
  const size_t ns = 2 * ndstate + 1, nx = m_.nq + m_.nv;
  if (int rc = mjpc_b200_create(model, (int)ns, 1, device, &engine_)) { error = mjpc_b200_last_error(); return rc; }
  if (int rc = mjpc_b200_set_options(engine_, timestep, 0)) { error = mjpc_b200_last_error(); return rc; }
  states_.resize(ns * nx); fstates_.resize(ns * nx); fnext_.resize(ns * nx); fsensor_.resize(ns * nsensordata);
  fqacc_.resize(ns * m_.nv); fwarm_.resize(ns * m_.nv); counts_.resize(4 * ns);
  Reset(nullptr, 0.0, 1e-4, 1e-4, 1e-4);
  std::copy(key_state_.begin(), key_state_.end(), states_.begin());
  if (int rc = StepSensors(1, std::vector<double>(m_.nu, 0.0).data(), nullptr)) return rc;
  Reset(nullptr, 0.0, 1e-4, 1e-4, 1e-4);
  return 0;
}

void Estimator::Reset(const double* s, double t, double covariance_scale, double process_scale, double sensor_scale) {
  state.assign(s ? s : key_state_.data(), (s ? s : key_state_.data()) + m_.nq + m_.nv);
  time = t;
  covariance.assign((size_t)ndstate * ndstate, 0.0);
  for (int i = 0; i < ndstate; i++) covariance[(size_t)i * ndstate + i] = covariance_scale;
  noise_process.assign(ndstate, process_scale);
  noise_sensor.assign(nsensordata, sensor_scale);
  qacc_warmstart_.assign(m_.nv, 0.0);
  warnings = 0;
}

int Estimator::StepSensors(int n, const double* ctrl, const float* mocap) {
  const int nv = m_.nv;
  for (size_t i = 0; i < (size_t)n * (m_.nq + nv); i++) fstates_[i] = (float)states_[i];
  for (int i = 0; i < n; i++)
    for (int k = 0; k < nv; k++) fwarm_[(size_t)i * nv + k] = (float)qacc_warmstart_[k];
  std::vector<float> u(m_.nu);
  for (int k = 0; k < m_.nu; k++) u[k] = (float)ctrl[k];
  if (int rc = mjpc_b200_step_sensors(engine_, n, fstates_.data(), u.data(), fwarm_.data(),
                                      mocap ? mocap : mocap0_.data(), time, sensor_start_, nsensor_, fnext_.data(),
                                      fsensor_.data(), fqacc_.data(), counts_.data())) {
    error = mjpc_b200_last_error();
    return rc;
  }
  nstepped_ = n;
  return 0;
}

void Estimator::Commit(int centre) {
  for (int k = 0; k < m_.nv; k++) qacc_warmstart_[k] = fqacc_[(size_t)centre * m_.nv + k];
  for (int i = 0; i < nstepped_; i++) warnings += counts_[4 * i + 3] != 0;
}

int Estimator::GainUpdate(const double* X, double* S, double* e, const double* P0, double* corr, double* P) {
  const int ns = ndstate, ny = nsensordata;
  if (CholFactor(S, ny, 1e-15) < ny) {
    error = std::string(name_) + " update: sensor covariance factorisation failed";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  CholSolve(S, ny, e);
  for (int r = 0; r < ns; r++) {
    corr[r] = 0.0;
    for (int c = 0; c < ny; c++) corr[r] += X[(size_t)r * ny + c] * e[c];
  }
  std::vector<double> T(X, X + (size_t)ns * ny);   // rows S^-1 X[r]
  for (int r = 0; r < ns; r++) CholSolve(S, ny, &T[(size_t)r * ny]);
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ns; c++) {
      double a = 0;
      for (int k = 0; k < ny; k++) a += X[(size_t)r * ny + k] * T[(size_t)c * ny + k];
      P[(size_t)r * ns + c] = P0[(size_t)r * ns + c] - a;
    }
  Symmetrize(P);
  return 0;
}

void Estimator::Symmetrize(double* P) const {
  const int n = ndstate;
  for (int r = 0; r < n; r++)
    for (int c = r + 1; c < n; c++) {
      const double s = 0.5 * (P[(size_t)r * n + c] + P[(size_t)c * n + r]);
      P[(size_t)r * n + c] = P[(size_t)c * n + r] = s;
    }
}

void Estimator::StateAdd(double* x, const double* dx, double scale) const {
  IntegratePos(m_, x, dx, scale);
  for (int k = 0; k < m_.nv; k++) x[m_.nq + k] += scale * dx[m_.nv + k];
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
// (the generic estimator family of include/mjpc_b200.h: every kind's handle, a NULL one refused)
using mjpc_b200_host::Estimator;
using mjpc_b200_host::EstimatorOf;

extern "C" {

int mjpc_b200_estimator_destroy(mjpc_b200_estimator_t* h) {
  Estimator* f = EstimatorOf<Estimator>(h);
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  delete f;
  return 0;
}

int mjpc_b200_estimator_reset(mjpc_b200_estimator_t* h, const double* state, double time, double covariance_scale,
                              double process_scale, double sensor_scale) {
  Estimator* f = EstimatorOf<Estimator>(h);
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  f->Reset(state, time, covariance_scale, process_scale, sensor_scale);
  return 0;
}

int mjpc_b200_estimator_set_noise(mjpc_b200_estimator_t* h, const double* process, const double* sensor) {
  Estimator* f = EstimatorOf<Estimator>(h);
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (process) f->noise_process.assign(process, process + f->ndstate);
  if (sensor) f->noise_sensor.assign(sensor, sensor + f->nsensordata);
  return 0;
}

int mjpc_b200_estimator_set(mjpc_b200_estimator_t* h, const double* state, const double* covariance, double time) {
  Estimator* f = EstimatorOf<Estimator>(h);
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (state) f->state.assign(state, state + f->state.size());
  if (covariance) f->covariance.assign(covariance, covariance + f->covariance.size());
  f->time = time;
  return 0;
}

int mjpc_b200_estimator_update(mjpc_b200_estimator_t* h, const double* ctrl, const double* sensor, const float* mocap) {
  Estimator* f = EstimatorOf<Estimator>(h);
  return f ? f->Update(ctrl, sensor, mocap) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_estimator_get(const mjpc_b200_estimator_t* h, double* state, double* covariance, double* time,
                            double* scalars) {
  const Estimator* f = reinterpret_cast<const Estimator*>(h);
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (state) std::copy(f->state.begin(), f->state.end(), state);
  if (covariance) std::copy(f->covariance.begin(), f->covariance.end(), covariance);
  if (time) *time = f->time;
  if (scalars) f->GetScalars(scalars);
  return 0;
}

const char* mjpc_b200_estimator_last_error(const mjpc_b200_estimator_t* h) {
  const Estimator* f = reinterpret_cast<const Estimator*>(h);
  return f ? f->error.c_str() : "";
}

}  // extern "C"
