// unscented.cc - see unscented.h.
#include "unscented.h"

#include <algorithm>
#include <cmath>
#include <cstring>

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

int Unscented::Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep_,
                          double alpha, double beta, int device) {
  if (int rc = InitializeBase(model, sensor_start, nsensor, timestep_, device)) return rc;
  // derived settings (unscented.cc:171-290)
  nsigma = 2 * ndstate + 1;
  const double lambda = ndstate * (alpha * alpha - 1.0);
  sigma_step = std::sqrt(ndstate + lambda);
  weight_mean0 = lambda / (ndstate + lambda);
  weight_covariance0 = weight_mean0 + 1.0 - alpha * alpha + beta;
  weight_sigma = 1.0 / (2.0 * (ndstate + lambda));
  const size_t ns = nsigma, nx = m_.nq + m_.nv;
  factor_.resize((size_t)ndstate * ndstate); next_states_.resize(ns * nx);
  sensors_.resize(ns * nsensordata); state_mean_.resize(nx); sensor_mean_.resize(nsensordata);
  state_difference_.resize(ns * ndstate); sensor_difference_.resize(ns * nsensordata);
  cov_yy_.resize((size_t)nsensordata * nsensordata); cov_sy_.resize((size_t)ndstate * nsensordata);
  cov_ss_.resize((size_t)ndstate * ndstate);
  return 0;
}

void Unscented::SigmaPoints() {
  const int nx = m_.nq + m_.nv;
  std::copy(state.begin(), state.end(), states_.begin() + (size_t)(nsigma - 1) * nx);   // nominal point last
  std::vector<double> column(ndstate);
  for (int i = 0; i < ndstate; i++) {
    for (int j = 0; j < ndstate; j++) column[j] = j >= i ? sigma_step * factor_[(size_t)j * ndstate + i] : 0.0;
    double* plus = &states_[(size_t)i * nx];
    double* minus = &states_[(size_t)(i + ndstate) * nx];
    std::copy(state.begin(), state.end(), plus);
    std::copy(state.begin(), state.end(), minus);
    StateAdd(plus, column.data(), 1.0);
    StateAdd(minus, column.data(), -1.0);
  }
}

int Unscented::EvaluateSigmaPoints(const double* ctrl, const float* mocap) {
  const int nx = m_.nq + m_.nv;
  if (int rc = StepSensors(nsigma, ctrl, mocap)) return rc;
  std::fill(state_mean_.begin(), state_mean_.end(), 0.0);
  std::fill(sensor_mean_.begin(), sensor_mean_.end(), 0.0);
  for (int i = 0; i < nsigma; i++) {
    const double w = i == nsigma - 1 ? weight_mean0 : weight_sigma;
    for (int k = 0; k < nx; k++) {
      next_states_[(size_t)i * nx + k] = fnext_[(size_t)i * nx + k];
      state_mean_[k] += w * next_states_[(size_t)i * nx + k];
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
      const double* q = &next_states_[(size_t)i * nx + a];
      const double w = 4.0 * (i == nsigma - 1 ? weight_covariance0 : weight_sigma);   // covariance weights, as :611
      for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) K[4 * r + c] += w * q[r] * q[c];
    }
    const double total = weight_covariance0 + (nsigma - 1) * weight_sigma;
    for (int r = 0; r < 4; r++) K[5 * r] -= total;
    PrincipalEigenVector4(&state_mean_[a], K, &next_states_[(size_t)(nsigma - 1) * nx + a]);
  }
}

void Unscented::SigmaPointDifferences() {
  const int nx = m_.nq + m_.nv;
  for (int i = 0; i < nsigma; i++) {
    StateDiff(m_, &state_difference_[(size_t)i * ndstate], &next_states_[(size_t)i * nx], state_mean_.data());
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
  // correction = cov_sy cov_yy^-1 (y - y_mean), covariance = cov_ss - cov_sy cov_yy^-1 cov_sy'
  std::vector<double> e(nsensordata), corr(ndstate);
  for (int k = 0; k < nsensordata; k++) e[k] = sensor[k] - sensor_mean_[k];
  if (int rc = GainUpdate(cov_sy_.data(), cov_yy_.data(), e.data(), cov_ss_.data(), corr.data(), covariance.data()))
    return rc;
  state = state_mean_;
  StateAdd(state.data(), corr.data(), 1.0);
  time += timestep;
  Commit(nsigma - 1);
  return 0;
}

void Unscented::GetScalars(double* scalars) const {
  scalars[0] = ndstate; scalars[1] = nsigma; scalars[2] = nsensordata; scalars[3] = warnings; scalars[4] = timestep;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------------------------ C ABI
using namespace mjpc_b200_host;

extern "C" {

int mjpc_b200_unscented_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                               double alpha, double beta, int device, mjpc_b200_estimator_t** out) {
  if (!out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* u = new Unscented;
  if (int rc = u->Initialize(model, sensor_start, nsensor, timestep, alpha, beta, device)) {
    delete u;
    return rc;
  }
  *out = ToHandle(u);
  return 0;
}

}  // extern "C"
