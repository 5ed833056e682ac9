// batch_estimator.cc - see batch_estimator.h.  Compiled into libmjpc_b200.so next to the engine.
#include "batch_estimator.h"

#include <algorithm>
#include <cmath>

#include "../filter_bank.h"
#include "estimator.h"

namespace mjpc_b200_host {

using mjpc_b200_bank::Access;

BatchEstimator::~BatchEstimator() { if (engine_) mjpc_b200_destroy(engine_); }

int BatchEstimator::Fail(int rc, const std::string& what) {
  error = "batch estimator: " + what;
  return rc;
}

int BatchEstimator::Initialize(const mjpc_model_blob* model, int kind_, int num_filters_, int sensor_start,
                               int nsensor, double timestep_, const double* settings, int device) {
  if (!model || (kind_ != 1 && kind_ != 2) || num_filters_ < 1 || !settings || !(timestep_ > 0))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "bad argument");
  if (kind_ == 1 && !(settings[0] > 0)) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "bad argument");
  if (int rc = m_.Load(model)) return Fail(rc, "bad blob");
  std::vector<int> dims;
  if (LoadEstimatorBlob(model, m_, &dims, &nmocap_, &mocap0_, &key_state_))
    return Fail(MJPC_B200_ERR_BAD_BLOB, "blob without sensor entries");
  if (sensor_start < 0 || nsensor < 1 || sensor_start > (int)dims.size() - nsensor)
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "sensor range outside the model's sensors");
  kind = kind_; num_filters = num_filters_; timestep = timestep_;
  ndstate = 2 * m_.nv;
  nsensordata = 0;
  for (int i = sensor_start; i < sensor_start + nsensor; i++) nsensordata += dims[i];
  mjpc_b200_bank::Desc d = {};
  d.kind = kind; d.num_filters = num_filters; d.sensor_start = sensor_start; d.nsensor = nsensor; d.timestep = timestep;
  if (kind == 2) {   // Unscented::Initialize's derived settings
    const double alpha = settings[0], beta = settings[1];
    rows = 2 * ndstate + 1;
    const double lambda = ndstate * (alpha * alpha - 1.0);
    d.sigma_step = std::sqrt(ndstate + lambda);
    d.weight_mean0 = lambda / (ndstate + lambda);
    d.weight_covariance0 = d.weight_mean0 + 1.0 - alpha * alpha + beta;
    d.weight_sigma = 1.0 / (2.0 * (ndstate + lambda));
  } else {
    epsilon = settings[0];
    d.epsilon = epsilon; d.centered = settings[1] != 0;
    rows = (d.centered ? 2 : 1) * ndstate + 1;
  }
  d.rows = rows;
  if ((long long)num_filters * rows > kBatchEstimatorMaxRows)
    return Fail(MJPC_B200_ERR_CAPACITY, "num_filters x rows per filter above " + std::to_string(kBatchEstimatorMaxRows));
  d.njnt = (int)m_.jnt_type.size();
  d.jnt_type = m_.jnt_type.data(); d.jnt_qposadr = m_.jnt_qposadr.data(); d.jnt_dofadr = m_.jnt_dofadr.data();
  if (int rc = mjpc_b200_create(model, num_filters * rows, 1, device, &engine_)) return Fail(rc, mjpc_b200_last_error());
  if (int rc = mjpc_b200_set_options(engine_, timestep, 0)) return Fail(rc, mjpc_b200_last_error());
  if (int rc = mjpc_b200_bank::Init(engine_, d)) return Fail(rc, mjpc_b200_last_error());
  fctrl_.resize((size_t)num_filters * m_.nu);
  fmocap_.resize((size_t)num_filters * 7 * nmocap_);
  for (int b = 0; b < num_filters; b++)
    if (int rc = Reset(b, nullptr, 0.0, 1e-4, 1e-4, 1e-4)) return rc;
  return 0;
}

int BatchEstimator::Reset(int b, const double* state, double time, double covariance_scale, double process_scale,
                          double sensor_scale) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  std::vector<double> P((size_t)ndstate * ndstate, 0.0), np(ndstate, process_scale), ns(nsensordata, sensor_scale);
  for (int i = 0; i < ndstate; i++) P[(size_t)i * ndstate + i] = covariance_scale;
  std::vector<float> warm(m_.nv, 0.f);
  int warnings = 0;
  const void* fields[] = {state ? state : key_state_.data(), P.data(), &time, np.data(), ns.data(), warm.data(),
                          &warnings};
  for (int f = mjpc_b200_bank::STATE; f <= mjpc_b200_bank::WARNINGS; f++)
    if (int rc = Access(engine_, b, f, const_cast<void*>(fields[f]), 1)) return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int BatchEstimator::SetNoise(int b, const double* process, const double* sensor) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (process)
    if (int rc = Access(engine_, b, mjpc_b200_bank::NOISE_PROCESS, const_cast<double*>(process), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (sensor)
    if (int rc = Access(engine_, b, mjpc_b200_bank::NOISE_SENSOR, const_cast<double*>(sensor), 1))
      return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int BatchEstimator::Set(int b, const double* state, const double* covariance, double time) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (state)
    if (int rc = Access(engine_, b, mjpc_b200_bank::STATE, const_cast<double*>(state), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (covariance)
    if (int rc = Access(engine_, b, mjpc_b200_bank::COVARIANCE, const_cast<double*>(covariance), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (int rc = Access(engine_, b, mjpc_b200_bank::TIME, &time, 1)) return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int BatchEstimator::Update(const double* ctrl, const double* sensor, const float* mocap, int* status) {
  if ((!ctrl && m_.nu) || !sensor || !status) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "update: bad argument");
  // ctrl as the single filters cast it; a NULL mocap is the model's for every filter
  for (size_t i = 0; i < fctrl_.size(); i++) fctrl_[i] = (float)ctrl[i];
  for (int b = 0; b < num_filters; b++)
    std::copy(mocap ? mocap + (size_t)b * mocap0_.size() : mocap0_.data(),
              (mocap ? mocap + (size_t)b * mocap0_.size() : mocap0_.data()) + mocap0_.size(),
              fmocap_.begin() + (size_t)b * mocap0_.size());
  if (int rc = mjpc_b200_bank::Update(engine_, fctrl_.data(), sensor, fmocap_.data(), status))
    return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int BatchEstimator::Get(int b, double* state, double* covariance, double* time, double* scalars) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (state)
    if (int rc = Access(engine_, b, mjpc_b200_bank::STATE, state, 0)) return Fail(rc, mjpc_b200_last_error());
  if (covariance)
    if (int rc = Access(engine_, b, mjpc_b200_bank::COVARIANCE, covariance, 0)) return Fail(rc, mjpc_b200_last_error());
  if (time)
    if (int rc = Access(engine_, b, mjpc_b200_bank::TIME, time, 0)) return Fail(rc, mjpc_b200_last_error());
  if (scalars) {
    int warnings = 0;
    if (int rc = Access(engine_, b, mjpc_b200_bank::WARNINGS, &warnings, 0)) return Fail(rc, mjpc_b200_last_error());
    // Unscented::GetScalars / Kalman::GetScalars
    scalars[0] = ndstate; scalars[1] = rows; scalars[2] = nsensordata; scalars[3] = warnings; scalars[4] = timestep;
    if (kind == 1) scalars[5] = epsilon;
  }
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using mjpc_b200_host::BatchEstimator;

extern "C" {

int mjpc_b200_batch_estimator_create(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start,
                                     int nsensor, double timestep, const double* settings, int device, void** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* f = new BatchEstimator;
  if (int rc = f->Initialize(model, kind, num_filters, sensor_start, nsensor, timestep, settings, device)) {
    delete f;
    return rc;
  }
  *out = f;
  return 0;
}

int mjpc_b200_batch_estimator_destroy(void* f) {
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  delete static_cast<BatchEstimator*>(f);
  return 0;
}

int mjpc_b200_batch_estimator_reset(void* f, int filter, const double* state, double time, double covariance_scale,
                                    double process_scale, double sensor_scale) {
  return f ? static_cast<BatchEstimator*>(f)->Reset(filter, state, time, covariance_scale, process_scale, sensor_scale)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_set_noise(void* f, int filter, const double* process, const double* sensor) {
  return f ? static_cast<BatchEstimator*>(f)->SetNoise(filter, process, sensor) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_set(void* f, int filter, const double* state, const double* covariance, double time) {
  return f ? static_cast<BatchEstimator*>(f)->Set(filter, state, covariance, time) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_update(void* f, const double* ctrl, const double* sensor, const float* mocap,
                                     int* status) {
  return f ? static_cast<BatchEstimator*>(f)->Update(ctrl, sensor, mocap, status) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_get(void* f, int filter, double* state, double* covariance, double* time,
                                  double* scalars) {
  return f ? static_cast<BatchEstimator*>(f)->Get(filter, state, covariance, time, scalars)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

const char* mjpc_b200_batch_estimator_last_error(const void* f) {
  return f ? static_cast<const BatchEstimator*>(f)->error.c_str() : "";
}

}  // extern "C"
