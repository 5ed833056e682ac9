// estimator.cc - see estimator.h.
#include "estimator.h"

#include <algorithm>
#include <cmath>

#include "../dev_model.h"   // Blob reader (plain C++)
#include "../filter_bank.h"

namespace mjpc_b200_host {

using mjpc_b200_bank::Access;

namespace {

// What the estimators read from the blob besides HostModel: every sensor's dimension, the model's mocap poses
// [7 nmocap] and the Reset state (the first keyframe, else qpos0 and zero qvel).  0, or MJPC_B200_ERR_BAD_BLOB for a
// blob without sensor entries.
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

// every one of the n values is finite (a NULL array has none)
template <class T>
bool AllFinite(const T* v, size_t n) {
  if (v)
    for (size_t i = 0; i < n; i++)
      if (!std::isfinite(v[i])) return false;
  return true;
}

}  // namespace

Estimator::~Estimator() { if (engine_) mjpc_b200_destroy(engine_); }

int Estimator::Fail(int rc, const std::string& what) {
  error = std::string(Name()) + ": " + what;
  return rc;
}

int Estimator::Initialize(const mjpc_model_blob* model, int kind_, int num_filters_, int sensor_start, int nsensor,
                          double timestep_, const double* settings, int device) {
  if (!model || (kind_ != kKalman && kind_ != kUnscented) || num_filters_ < 1 || !settings || !(timestep_ > 0))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "bad argument");
  kind = kind_;
  if (kind == kKalman && !(settings[0] > 0)) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "bad argument");
  if (int rc = m_.Load(model)) return Fail(rc, "bad blob");
  std::vector<int> dims;
  if (LoadEstimatorBlob(model, m_, &dims, &nmocap_, &model_mocap0_, &model_key_state_))
    return Fail(MJPC_B200_ERR_BAD_BLOB, "blob without sensor entries");
  if (sensor_start < 0 || nsensor < 1 || sensor_start > (int)dims.size() - nsensor)
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "sensor range outside the model's sensors");
  num_filters = num_filters_; timestep = timestep_;
  ndstate = 2 * m_.nv;
  nsensordata = 0;
  for (int i = sensor_start; i < sensor_start + nsensor; i++) nsensordata += dims[i];
  mjpc_b200_bank::Desc d = {};
  d.kind = kind; d.num_filters = num_filters; d.sensor_start = sensor_start; d.nsensor = nsensor; d.timestep = timestep;
  if (kind == kUnscented) {   // the derived settings (unscented.cc:171-290)
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
  if ((long long)num_filters * rows > kEstimatorMaxRows)
    return Fail(MJPC_B200_ERR_CAPACITY, "num_filters x rows per filter above " + std::to_string(kEstimatorMaxRows));
  d.njnt = (int)m_.jnt_type.size();
  d.jnt_type = m_.jnt_type.data(); d.jnt_qposadr = m_.jnt_qposadr.data(); d.jnt_dofadr = m_.jnt_dofadr.data();
  if (int rc = mjpc_b200_create(model, num_filters * rows, 1, device, &engine_))
    return Fail(rc, mjpc_b200_last_error());
  if (int rc = mjpc_b200_set_options(engine_, timestep, 0)) return Fail(rc, mjpc_b200_last_error());
  if (int rc = mjpc_b200_bank::Init(engine_, d)) return Fail(rc, mjpc_b200_last_error());
  fctrl_.resize((size_t)num_filters * m_.nu); ctrl_.resize(fctrl_.size());
  fmocap_.resize((size_t)num_filters * model_mocap0_.size()); mocap_.resize(fmocap_.size());
  for (int b = 0; b < num_filters; b++) {
    key_state_.insert(key_state_.end(), model_key_state_.begin(), model_key_state_.end());
    mocap0_.insert(mocap0_.end(), model_mocap0_.begin(), model_mocap0_.end());
  }
  for (int b = 0; b < num_filters; b++)
    if (int rc = Reset(b, nullptr, 0.0, 1e-4, 1e-4, 1e-4)) return rc;
  return 0;
}

int Estimator::Reset(int b, const double* state, double time, double covariance_scale, double process_scale,
                     double sensor_scale) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (!AllFinite(state, model_key_state_.size()) || !std::isfinite(time) || !std::isfinite(covariance_scale) ||
      !std::isfinite(process_scale) || !std::isfinite(sensor_scale))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "reset: a value is not finite");
  std::vector<double> P((size_t)ndstate * ndstate, 0.0), np(ndstate, process_scale), ns(nsensordata, sensor_scale);
  for (int i = 0; i < ndstate; i++) P[(size_t)i * ndstate + i] = covariance_scale;
  std::vector<float> warm(m_.nv, 0.f);
  int warnings = 0;
  const size_t nx = model_key_state_.size(), nm = model_mocap0_.size();
  const void* fields[] = {state ? state : key_state_.data() + b * nx, P.data(), &time, np.data(), ns.data(), warm.data(),
                          &warnings};
  for (int f = mjpc_b200_bank::STATE; f <= mjpc_b200_bank::WARNINGS; f++)
    if (int rc = Access(engine_, b, f, const_cast<void*>(fields[f]), 1)) return Fail(rc, mjpc_b200_last_error());
  std::fill_n(ctrl_.begin() + (size_t)b * m_.nu, m_.nu, 0.f);
  std::copy_n(mocap0_.begin() + b * nm, nm, mocap_.begin() + b * nm);
  return 0;
}

int Estimator::SetModels(const mjpc_model_blob* models, int count) {
  if (count != 0 && (count != num_filters || !models)) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_models: count is not num_filters or 0");
  if (int rc = mjpc_b200_set_model_variants(engine_, models, count)) return Fail(rc, mjpc_b200_last_error());
  const size_t nx = model_key_state_.size(), nm = model_mocap0_.size();
  for (int b = 0; b < num_filters; b++) {
    std::vector<int> dims;
    int nmocap = 0;
    std::vector<float> mocap0 = model_mocap0_;
    std::vector<double> key_state = model_key_state_;
    if (count && LoadEstimatorBlob(&models[b], m_, &dims, &nmocap, &mocap0, &key_state))
      return Fail(MJPC_B200_ERR_BAD_BLOB, "set_models: blob without sensor entries");
    std::copy_n(key_state.begin(), nx, key_state_.begin() + b * nx);
    std::copy_n(mocap0.begin(), nm, mocap0_.begin() + b * nm);
  }
  return 0;
}

int Estimator::SetNoise(int b, const double* process, const double* sensor) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (!AllFinite(process, ndstate) || !AllFinite(sensor, nsensordata))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_noise: a value is not finite");
  if (process)
    if (int rc = Access(engine_, b, mjpc_b200_bank::NOISE_PROCESS, const_cast<double*>(process), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (sensor)
    if (int rc = Access(engine_, b, mjpc_b200_bank::NOISE_SENSOR, const_cast<double*>(sensor), 1))
      return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int Estimator::Set(int b, const double* state, const double* covariance, double time) {
  if (b < 0 || b >= num_filters) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter index outside [0, num_filters)");
  if (!AllFinite(state, model_key_state_.size()) || !AllFinite(covariance, (size_t)ndstate * ndstate) ||
      !std::isfinite(time))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "set: a value is not finite");
  if (state)
    if (int rc = Access(engine_, b, mjpc_b200_bank::STATE, const_cast<double*>(state), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (covariance)
    if (int rc = Access(engine_, b, mjpc_b200_bank::COVARIANCE, const_cast<double*>(covariance), 1))
      return Fail(rc, mjpc_b200_last_error());
  if (int rc = Access(engine_, b, mjpc_b200_bank::TIME, &time, 1)) return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int Estimator::Update(const double* ctrl, const double* sensor, const float* mocap, int phases, int* status) {
  const bool measure = kind == kUnscented || phases != mjpc_b200_bank::PREDICTION;
  if ((measure && ((!ctrl && m_.nu) || !sensor)) || !status)
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "update: bad argument");
  if (!measure) {
    if (int rc = mjpc_b200_bank::Update(engine_, ctrl_.data(), nullptr, mocap_.data(), phases, status))
      return Fail(rc, mjpc_b200_last_error());
    return 0;
  }
  if (!AllFinite(sensor, (size_t)num_filters * nsensordata))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "update: a sensor value is not finite");
  if (int rc = StageInputs(ctrl, mocap)) return rc;
  const size_t nu = m_.nu, nm = model_mocap0_.size();
  if (int rc = mjpc_b200_bank::Update(engine_, fctrl_.data(), sensor, fmocap_.data(), phases, status))
    return Fail(rc, mjpc_b200_last_error());
  for (int b = 0; b < num_filters; b++)
    if (status[b] == mjpc_b200_bank::UPDATED) {
      std::copy_n(fctrl_.begin() + b * nu, nu, ctrl_.begin() + b * nu);
      std::copy_n(fmocap_.begin() + b * nm, nm, mocap_.begin() + b * nm);
    }
  return 0;
}

int Estimator::StageInputs(const double* ctrl, const float* mocap) {
  const size_t nm = model_mocap0_.size();
  if (!AllFinite(ctrl, fctrl_.size()) || !AllFinite(mocap, (size_t)num_filters * nm))
    return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "update: a ctrl or mocap value is not finite");
  // ctrl in the engine's float; a NULL mocap is the model's for every filter
  for (size_t i = 0; i < fctrl_.size(); i++) fctrl_[i] = (float)ctrl[i];
  for (int b = 0; b < num_filters; b++)
    std::copy_n((mocap ? mocap : mocap0_.data()) + b * nm, nm, fmocap_.begin() + b * nm);
  return 0;
}

int Estimator::DebugRows(int phase, const double* ctrl, const float* mocap, float* qpos, float* qvel, float* warm,
                         int* status) {
  if (!ctrl && m_.nu) return Fail(MJPC_B200_ERR_BAD_ARGUMENT, "debug_rows: bad argument");
  if (int rc = StageInputs(ctrl, mocap)) return rc;
  if (int rc = mjpc_b200_bank::DebugRows(engine_, phase, fctrl_.data(), fmocap_.data(), qpos, qvel, warm, status))
    return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int Estimator::DebugFinish(int phase, const double* sensor, const float* next_qpos, const float* next_qvel,
                           const float* qacc, const float* sensordata, const int* counts, int* status) {
  if (int rc = mjpc_b200_bank::DebugFinish(engine_, phase, sensor, next_qpos, next_qvel, qacc, sensordata, counts,
                                           status))
    return Fail(rc, mjpc_b200_last_error());
  return 0;
}

int Estimator::Get(int b, double* state, double* covariance, double* time, double* scalars) {
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
    scalars[0] = ndstate; scalars[1] = rows; scalars[2] = nsensordata; scalars[3] = warnings; scalars[4] = timestep;
    if (kind == kKalman) scalars[5] = epsilon;
  }
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using namespace mjpc_b200_host;

namespace {

int Create(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start, int nsensor, double timestep,
           const double* settings, int device, Estimator** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* f = new Estimator;
  if (int rc = f->Initialize(model, kind, num_filters, sensor_start, nsensor, timestep, settings, device)) {
    delete f;
    return rc;
  }
  *out = f;
  return 0;
}

// the single filter behind a handle of the mjpc_b200_estimator_* family (nullptr for a NULL handle); non-const
// because get, which takes a const handle, reads through the filter's engine and may record an error
Estimator* Single(const mjpc_b200_estimator_t* h) {
  return reinterpret_cast<Estimator*>(const_cast<mjpc_b200_estimator_t*>(h));
}

// one update of a single filter; a failed factorisation or a result that is not finite is MJPC_B200_ERR_BAD_ARGUMENT
// with last_error naming it
int UpdateSingle(Estimator* f, const double* ctrl, const double* sensor, const float* mocap, int phases) {
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  int status = 0;
  if (int rc = f->Update(ctrl, sensor, mocap, phases, &status)) return rc;
  if (status == mjpc_b200_bank::UPDATED) return 0;
  f->error = std::string(f->Name()) + " update: " +
             (status == mjpc_b200_bank::COVARIANCE_FACTOR_FAILED ? "covariance factorisation failed"
              : status == mjpc_b200_bank::SENSOR_FACTOR_FAILED   ? "sensor covariance factorisation failed"
                                                                 : "non-finite result (state or covariance)");
  return MJPC_B200_ERR_BAD_ARGUMENT;
}

}  // namespace

extern "C" {

// ---- single filters: filter 0 of a one-filter bank
int mjpc_b200_unscented_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                               double alpha, double beta, int device, mjpc_b200_estimator_t** out) {
  const double settings[2] = {alpha, beta};
  return Create(model, kUnscented, 1, sensor_start, nsensor, timestep, settings, device,
                reinterpret_cast<Estimator**>(out));
}

int mjpc_b200_kalman_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                            double epsilon, int centered, int device, mjpc_b200_estimator_t** out) {
  const double settings[2] = {epsilon, centered != 0 ? 1.0 : 0.0};
  return Create(model, kKalman, 1, sensor_start, nsensor, timestep, settings, device,
                reinterpret_cast<Estimator**>(out));
}

int mjpc_b200_estimator_destroy(mjpc_b200_estimator_t* h) {
  if (!h) return MJPC_B200_ERR_BAD_ARGUMENT;
  delete Single(h);
  return 0;
}

int mjpc_b200_estimator_reset(mjpc_b200_estimator_t* h, const double* state, double time, double covariance_scale,
                              double process_scale, double sensor_scale) {
  return h ? Single(h)->Reset(0, state, time, covariance_scale, process_scale, sensor_scale)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_estimator_set_noise(mjpc_b200_estimator_t* h, const double* process, const double* sensor) {
  return h ? Single(h)->SetNoise(0, process, sensor) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_estimator_set(mjpc_b200_estimator_t* h, const double* state, const double* covariance, double time) {
  return h ? Single(h)->Set(0, state, covariance, time) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_estimator_update(mjpc_b200_estimator_t* h, const double* ctrl, const double* sensor, const float* mocap) {
  return UpdateSingle(Single(h), ctrl, sensor, mocap, mjpc_b200_bank::MEASUREMENT_AND_PREDICTION);
}

int mjpc_b200_estimator_get(const mjpc_b200_estimator_t* h, double* state, double* covariance, double* time,
                            double* scalars) {
  return h ? Single(h)->Get(0, state, covariance, time, scalars) : MJPC_B200_ERR_BAD_ARGUMENT;
}

const char* mjpc_b200_estimator_last_error(const mjpc_b200_estimator_t* h) { return h ? Single(h)->error.c_str() : ""; }

int mjpc_b200_kalman_update_measurement(mjpc_b200_estimator_t* h, const double* ctrl, const double* sensor,
                                        const float* mocap) {
  Estimator* f = Single(h);
  return f && f->kind == kKalman ? UpdateSingle(f, ctrl, sensor, mocap, mjpc_b200_bank::MEASUREMENT)
                                 : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_kalman_update_prediction(mjpc_b200_estimator_t* h) {
  Estimator* f = Single(h);
  return f && f->kind == kKalman ? UpdateSingle(f, nullptr, nullptr, nullptr, mjpc_b200_bank::PREDICTION)
                                 : MJPC_B200_ERR_BAD_ARGUMENT;
}

// ---- filter banks
int mjpc_b200_batch_estimator_create(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start,
                                     int nsensor, double timestep, const double* settings, int device, void** out) {
  return Create(model, kind, num_filters, sensor_start, nsensor, timestep, settings, device,
                reinterpret_cast<Estimator**>(out));
}

int mjpc_b200_batch_estimator_destroy(void* f) {
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  delete static_cast<Estimator*>(f);
  return 0;
}

int mjpc_b200_batch_estimator_reset(void* f, int filter, const double* state, double time, double covariance_scale,
                                    double process_scale, double sensor_scale) {
  return f ? static_cast<Estimator*>(f)->Reset(filter, state, time, covariance_scale, process_scale, sensor_scale)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_set_noise(void* f, int filter, const double* process, const double* sensor) {
  return f ? static_cast<Estimator*>(f)->SetNoise(filter, process, sensor) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_set(void* f, int filter, const double* state, const double* covariance, double time) {
  return f ? static_cast<Estimator*>(f)->Set(filter, state, covariance, time) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_update(void* f, const double* ctrl, const double* sensor, const float* mocap,
                                     int* status) {
  if (!f) return MJPC_B200_ERR_BAD_ARGUMENT;
  Estimator* e = static_cast<Estimator*>(f);
  if (int rc = e->Update(ctrl, sensor, mocap, mjpc_b200_bank::MEASUREMENT_AND_PREDICTION, status)) return rc;
  for (int b = 0; b < e->num_filters; b++)
    if (status[b] != mjpc_b200_bank::UPDATED) status[b] = MJPC_B200_ERR_BAD_ARGUMENT;
  return 0;
}

int mjpc_b200_batch_estimator_get(void* f, int filter, double* state, double* covariance, double* time,
                                  double* scalars) {
  return f ? static_cast<Estimator*>(f)->Get(filter, state, covariance, time, scalars) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_set_models(void* f, const mjpc_model_blob* models, int count) {
  return f && count >= 0 ? static_cast<Estimator*>(f)->SetModels(models, count) : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_debug_rows(void* f, int phase, const double* ctrl, const float* mocap, float* qpos,
                                         float* qvel, float* warm, int* status) {
  return f ? static_cast<Estimator*>(f)->DebugRows(phase, ctrl, mocap, qpos, qvel, warm, status)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

int mjpc_b200_batch_estimator_debug_finish(void* f, int phase, const double* sensor, const float* next_qpos,
                                           const float* next_qvel, const float* qacc, const float* sensordata,
                                           const int* counts, int* status) {
  return f ? static_cast<Estimator*>(f)->DebugFinish(phase, sensor, next_qpos, next_qvel, qacc, sensordata, counts,
                                                     status)
           : MJPC_B200_ERR_BAD_ARGUMENT;
}

const char* mjpc_b200_batch_estimator_last_error(const void* f) {
  return f ? static_cast<const Estimator*>(f)->error.c_str() : "";
}

}  // extern "C"
