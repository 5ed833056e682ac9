// unscented.cc - see unscented.h.
#include "unscented.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "../dev_model.h"
#include "planner.h"

namespace mjpc_b200_host {

namespace {

// Principal eigenvector of a symmetric 4 x 4 matrix by cyclic Jacobi rotations (converged to rounding), with the sign
// that agrees with `ref`.  Stands for PrincipalEigenVector4 (utilities.cc:1476+) in QuaternionMeans.
void PrincipalEigenVector4(double* out, const double* K, const double* ref) {
  double A[16], V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  std::memcpy(A, K, sizeof(A));
  for (int sweep = 0; sweep < 50; sweep++) {
    double off = 0;
    for (int p = 0; p < 4; p++) for (int q = p + 1; q < 4; q++) off += A[4 * p + q] * A[4 * p + q];
    if (off < 1e-300) break;
    for (int p = 0; p < 4; p++)
      for (int q = p + 1; q < 4; q++) {
        if (A[4 * p + q] == 0) continue;
        const double th = (A[4 * q + q] - A[4 * p + p]) / (2 * A[4 * p + q]);
        const double t = std::fabs(th) > 1e150 ? 0.5 / th : (th >= 0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1));
        const double c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 4; k++) {   // A <- A J
          const double akp = A[4 * k + p], akq = A[4 * k + q];
          A[4 * k + p] = c * akp - s * akq; A[4 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 4; k++) {   // A <- J' A
          const double apk = A[4 * p + k], aqk = A[4 * q + k];
          A[4 * p + k] = c * apk - s * aqk; A[4 * q + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 4; k++) {   // V <- V J
          const double vkp = V[4 * k + p], vkq = V[4 * k + q];
          V[4 * k + p] = c * vkp - s * vkq; V[4 * k + q] = s * vkp + c * vkq;
        }
      }
  }
  int best = 0;
  for (int k = 1; k < 4; k++) if (A[5 * k] > A[5 * best]) best = k;
  double dot = 0;
  for (int k = 0; k < 4; k++) dot += V[4 * k + best] * ref[k];
  const double sg = dot >= 0 ? 1.0 : -1.0;
  double n = 0;
  for (int k = 0; k < 4; k++) n += V[4 * k + best] * V[4 * k + best];
  n = std::sqrt(n);
  for (int k = 0; k < 4; k++) out[k] = sg * V[4 * k + best] / n;
}

}  // namespace

int LoadEstimatorBlob(const mjpc_model_blob* model, const iLQGPolicyModel& m, std::vector<int>* dims, int* nmocap,
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

Unscented::~Unscented() { if (engine_) mjpc_b200_destroy(engine_); }

int Unscented::Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep_,
                          double alpha, double beta, int device) {
  if (!model || !(timestep_ > 0)) { error = "unscented: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  if (int rc = m_.Load(model)) { error = "unscented: bad blob"; return rc; }
  std::vector<int> dims;
  if (LoadEstimatorBlob(model, m_, &dims, &nmocap_, &mocap0_, &key_state_)) {
    error = "unscented: blob without sensor entries";
    return MJPC_B200_ERR_BAD_BLOB;
  }
  if (sensor_start < 0 || nsensor < 1 || sensor_start > (int)dims.size() - nsensor) {
    error = "unscented: sensor range outside the model's sensors";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  sensor_start_ = sensor_start; nsensor_ = nsensor;
  nsensordata = 0;
  for (int i = sensor_start; i < sensor_start + nsensor; i++) nsensordata += dims[i];
  timestep = timestep_;
  // derived settings (unscented.cc:171-290)
  ndstate = 2 * m_.nv;
  nsigma = 2 * ndstate + 1;
  const double lambda = ndstate * (alpha * alpha - 1.0);
  sigma_step = std::sqrt(ndstate + lambda);
  weight_mean0 = lambda / (ndstate + lambda);
  weight_covariance0 = weight_mean0 + 1.0 - alpha * alpha + beta;
  weight_sigma = 1.0 / (2.0 * (ndstate + lambda));
  if (int rc = mjpc_b200_create(model, nsigma, 1, device, &engine_)) { error = mjpc_b200_last_error(); return rc; }
  if (int rc = mjpc_b200_set_options(engine_, timestep, 0)) { error = mjpc_b200_last_error(); return rc; }
  const size_t ns = nsigma, nx = m_.nq + m_.nv;
  factor_.resize((size_t)ndstate * ndstate); sigma_.resize(ns * nx); states_.resize(ns * nx);
  sensors_.resize(ns * nsensordata); state_mean_.resize(nx); sensor_mean_.resize(nsensordata);
  state_difference_.resize(ns * ndstate); sensor_difference_.resize(ns * nsensordata);
  cov_yy_.resize((size_t)nsensordata * nsensordata); cov_sy_.resize((size_t)ndstate * nsensordata);
  cov_ss_.resize((size_t)ndstate * ndstate);
  fstates_.resize(ns * nx); fnext_.resize(ns * nx); fsensor_.resize(ns * nsensordata); fqacc_.resize(ns * m_.nv);
  fwarm_.resize(ns * m_.nv); counts_.resize(4 * ns);
  Reset(nullptr, 0.0, 1e-4, 1e-4, 1e-4);
  return 0;
}

void Unscented::Reset(const double* s, double t, double covariance_scale, double process_scale, double sensor_scale) {
  state.assign(s ? s : key_state_.data(), (s ? s : key_state_.data()) + m_.nq + m_.nv);
  time = t;
  covariance.assign((size_t)ndstate * ndstate, 0.0);
  for (int i = 0; i < ndstate; i++) covariance[(size_t)i * ndstate + i] = covariance_scale;
  noise_process.assign(ndstate, process_scale);
  noise_sensor.assign(nsensordata, sensor_scale);
  qacc_warmstart_.assign(m_.nv, 0.0);
  warnings = 0;
}

void Unscented::SigmaPoints() {
  const int nq = m_.nq, nv = m_.nv, nx = nq + nv;
  std::copy(state.begin(), state.end(), sigma_.begin() + (size_t)(nsigma - 1) * nx);   // nominal point last
  std::vector<double> column(ndstate);
  for (int i = 0; i < ndstate; i++) {
    for (int j = 0; j < ndstate; j++) column[j] = j >= i ? sigma_step * factor_[(size_t)j * ndstate + i] : 0.0;
    double* plus = &sigma_[(size_t)i * nx];
    double* minus = &sigma_[(size_t)(i + ndstate) * nx];
    std::copy(state.begin(), state.end(), plus);
    std::copy(state.begin(), state.end(), minus);
    IntegratePos(m_, plus, column.data(), 1.0);
    IntegratePos(m_, minus, column.data(), -1.0);
    for (int k = 0; k < nv; k++) { plus[nq + k] += column[nv + k]; minus[nq + k] -= column[nv + k]; }
  }
}

int Unscented::EvaluateSigmaPoints(const double* ctrl, const float* mocap) {
  const int nx = m_.nq + m_.nv, nv = m_.nv;
  for (size_t i = 0; i < sigma_.size(); i++) fstates_[i] = (float)sigma_[i];
  for (int i = 0; i < nsigma; i++)
    for (int k = 0; k < nv; k++) fwarm_[(size_t)i * nv + k] = (float)qacc_warmstart_[k];
  std::vector<float> u(m_.nu);
  for (int k = 0; k < m_.nu; k++) u[k] = (float)ctrl[k];
  if (int rc = mjpc_b200_step_sensors(engine_, nsigma, fstates_.data(), u.data(), fwarm_.data(),
                                      mocap ? mocap : mocap0_.data(), time, sensor_start_, nsensor_, fnext_.data(),
                                      fsensor_.data(), fqacc_.data(), counts_.data())) {
    error = mjpc_b200_last_error();
    return rc;
  }
  std::fill(state_mean_.begin(), state_mean_.end(), 0.0);
  std::fill(sensor_mean_.begin(), sensor_mean_.end(), 0.0);
  for (int i = 0; i < nsigma; i++) {
    const double w = i == nsigma - 1 ? weight_mean0 : weight_sigma;
    for (int k = 0; k < nx; k++) {
      states_[(size_t)i * nx + k] = fnext_[(size_t)i * nx + k];
      state_mean_[k] += w * states_[(size_t)i * nx + k];
    }
    for (int k = 0; k < nsensordata; k++) {
      sensors_[(size_t)i * nsensordata + k] = fsensor_[(size_t)i * nsensordata + k];
      sensor_mean_[k] += w * sensors_[(size_t)i * nsensordata + k];
    }
  }
  QuaternionMeans();
  return 0;
}

void Unscented::QuaternionMeans() {
  const int nx = m_.nq + m_.nv;
  for (size_t j = 0; j < m_.jnt_type.size(); j++) {
    if (m_.jnt_type[j] != 0 && m_.jnt_type[j] != 1) continue;
    const int a = m_.jnt_qposadr[j] + (m_.jnt_type[j] == 0 ? 3 : 0);
    double K[16] = {0};
    for (int i = 0; i < nsigma; i++) {
      const double* q = &states_[(size_t)i * nx + a];
      const double w = 4.0 * (i == nsigma - 1 ? weight_covariance0 : weight_sigma);   // covariance weights, as :611
      for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) K[4 * r + c] += w * q[r] * q[c];
    }
    const double total = weight_covariance0 + (nsigma - 1) * weight_sigma;
    for (int r = 0; r < 4; r++) K[5 * r] -= total;
    PrincipalEigenVector4(&state_mean_[a], K, &states_[(size_t)(nsigma - 1) * nx + a]);
  }
}

void Unscented::SigmaPointDifferences() {
  const int nx = m_.nq + m_.nv;
  for (int i = 0; i < nsigma; i++) {
    StateDiff(m_, &state_difference_[(size_t)i * ndstate], &states_[(size_t)i * nx], state_mean_.data());
    for (int k = 0; k < nsensordata; k++)
      sensor_difference_[(size_t)i * nsensordata + k] = sensors_[(size_t)i * nsensordata + k] - sensor_mean_[k];
  }
}

void Unscented::SigmaCovariances() {
  const int ny = nsensordata, ns = ndstate;
  std::fill(cov_yy_.begin(), cov_yy_.end(), 0.0);
  std::fill(cov_sy_.begin(), cov_sy_.end(), 0.0);
  std::fill(cov_ss_.begin(), cov_ss_.end(), 0.0);
  for (int i = 0; i < ny; i++) cov_yy_[(size_t)i * ny + i] = noise_sensor[i];
  for (int i = 0; i < ns; i++) cov_ss_[(size_t)i * ns + i] = noise_process[i];
  for (int p = 0; p < nsigma; p++) {
    const double w = p == nsigma - 1 ? weight_covariance0 : weight_sigma;
    const double* dy = &sensor_difference_[(size_t)p * ny];
    const double* ds = &state_difference_[(size_t)p * ns];
    for (int r = 0; r < ny; r++) for (int c = 0; c < ny; c++) cov_yy_[(size_t)r * ny + c] += w * dy[r] * dy[c];
    for (int r = 0; r < ns; r++) for (int c = 0; c < ny; c++) cov_sy_[(size_t)r * ny + c] += w * ds[r] * dy[c];
    for (int r = 0; r < ns; r++) for (int c = 0; c < ns; c++) cov_ss_[(size_t)r * ns + c] += w * ds[r] * ds[c];
  }
}

int Unscented::Update(const double* ctrl, const double* sensor, const float* mocap) {
  if (!engine_ || (!ctrl && m_.nu) || !sensor) { error = "unscented update: bad argument"; return MJPC_B200_ERR_BAD_ARGUMENT; }
  factor_ = covariance;
  if (CholFactor(factor_.data(), ndstate, 1e-15) < ndstate) {
    error = "unscented update: covariance factorisation failed";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  SigmaPoints();
  if (int rc = EvaluateSigmaPoints(ctrl, mocap)) return rc;
  SigmaPointDifferences();
  SigmaCovariances();
  const int ny = nsensordata, ns = ndstate, nq = m_.nq, nv = m_.nv;
  std::vector<double> Ly = cov_yy_;
  if (CholFactor(Ly.data(), ny, 1e-15) < ny) {
    error = "unscented update: sensor covariance factorisation failed";
    return MJPC_B200_ERR_BAD_ARGUMENT;
  }
  // correction = cov_sy cov_yy^-1 (y - y_mean)
  std::vector<double> e(ny), corr(ns, 0.0);
  for (int k = 0; k < ny; k++) e[k] = sensor[k] - sensor_mean_[k];
  CholSolve(Ly.data(), ny, e.data());
  for (int r = 0; r < ns; r++) for (int c = 0; c < ny; c++) corr[r] += cov_sy_[(size_t)r * ny + c] * e[c];
  // covariance = cov_ss - cov_sy cov_yy^-1 cov_sy'
  std::vector<double> T((size_t)ns * ny);
  for (int r = 0; r < ns; r++) {
    std::copy(&cov_sy_[(size_t)r * ny], &cov_sy_[(size_t)r * ny] + ny, &T[(size_t)r * ny]);
    CholSolve(Ly.data(), ny, &T[(size_t)r * ny]);
  }
  for (int r = 0; r < ns; r++)
    for (int c = 0; c < ns; c++) {
      double a = 0;
      for (int k = 0; k < ny; k++) a += cov_sy_[(size_t)r * ny + k] * T[(size_t)c * ny + k];
      covariance[(size_t)r * ns + c] = cov_ss_[(size_t)r * ns + c] - a;
    }
  for (int r = 0; r < ns; r++)
    for (int c = r + 1; c < ns; c++) {
      const double s = 0.5 * (covariance[(size_t)r * ns + c] + covariance[(size_t)c * ns + r]);
      covariance[(size_t)r * ns + c] = covariance[(size_t)c * ns + r] = s;
    }
  state = state_mean_;
  IntegratePos(m_, state.data(), corr.data(), 1.0);
  for (int k = 0; k < nv; k++) state[nq + k] += corr[nv + k];
  time += timestep;
  for (int k = 0; k < nv; k++) qacc_warmstart_[k] = fqacc_[(size_t)(nsigma - 1) * nv + k];
  for (int i = 0; i < nsigma; i++) warnings += counts_[4 * i + 3] != 0;
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using mjpc_b200_host::Unscented;

extern "C" {

int mjpc_b200_unscented_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                               double alpha, double beta, int device, mjpc_b200_unscented_t** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* u = new Unscented;
  if (int rc = u->Initialize(model, sensor_start, nsensor, timestep, alpha, beta, device)) {
    delete u;
    return rc;
  }
  *out = reinterpret_cast<mjpc_b200_unscented_t*>(u);
  return 0;
}

void mjpc_b200_unscented_destroy(mjpc_b200_unscented_t* u) { delete reinterpret_cast<Unscented*>(u); }

int mjpc_b200_unscented_reset(mjpc_b200_unscented_t* u, const double* state, double time, double covariance_scale,
                              double process_scale, double sensor_scale) {
  if (!u) return MJPC_B200_ERR_BAD_ARGUMENT;
  reinterpret_cast<Unscented*>(u)->Reset(state, time, covariance_scale, process_scale, sensor_scale);
  return 0;
}

int mjpc_b200_unscented_set_noise(mjpc_b200_unscented_t* u, const double* process, const double* sensor) {
  if (!u) return MJPC_B200_ERR_BAD_ARGUMENT;
  Unscented* f = reinterpret_cast<Unscented*>(u);
  if (process) f->noise_process.assign(process, process + f->ndstate);
  if (sensor) f->noise_sensor.assign(sensor, sensor + f->nsensordata);
  return 0;
}

int mjpc_b200_unscented_set(mjpc_b200_unscented_t* u, const double* state, const double* covariance, double time) {
  if (!u) return MJPC_B200_ERR_BAD_ARGUMENT;
  Unscented* f = reinterpret_cast<Unscented*>(u);
  if (state) f->state.assign(state, state + f->state.size());
  if (covariance) f->covariance.assign(covariance, covariance + f->covariance.size());
  f->time = time;
  return 0;
}

int mjpc_b200_unscented_update(mjpc_b200_unscented_t* u, const double* ctrl, const double* sensor, const float* mocap) {
  if (!u) return MJPC_B200_ERR_BAD_ARGUMENT;
  Unscented* f = reinterpret_cast<Unscented*>(u);
  return f->Update(ctrl, sensor, mocap);
}

int mjpc_b200_unscented_get(const mjpc_b200_unscented_t* u, double* state, double* covariance, double* time,
                            double* scalars) {
  if (!u) return MJPC_B200_ERR_BAD_ARGUMENT;
  const Unscented* f = reinterpret_cast<const Unscented*>(u);
  if (state) std::copy(f->state.begin(), f->state.end(), state);
  if (covariance) std::copy(f->covariance.begin(), f->covariance.end(), covariance);
  if (time) *time = f->time;
  if (scalars) {
    scalars[0] = f->ndstate; scalars[1] = f->nsigma; scalars[2] = f->nsensordata; scalars[3] = f->warnings;
    scalars[4] = f->timestep;
  }
  return 0;
}

const char* mjpc_b200_unscented_last_error(const mjpc_b200_unscented_t* u) {
  return u ? reinterpret_cast<const Unscented*>(u)->error.c_str() : "";
}

}  // extern "C"
