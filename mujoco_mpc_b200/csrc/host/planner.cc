// planner.cc - see planner.h.
#include "planner.h"

#include <cmath>

#include <algorithm>

namespace mjpc_b200_host {

void FindInterval(int* b, const double* seq, double value, int length) {
  int upper = 0;
  while (upper < length && !(value < seq[upper])) upper++;
  const int lower = upper - 1;
  if (lower < 0) b[0] = b[1] = 0;
  else if (lower > length - 1) b[0] = b[1] = length - 1;
  else { b[0] = std::max(lower, 0); b[1] = std::min(upper, length - 1); }
}

Planner::~Planner() {
  if (gpu_ && owns_gpu_) mjpc_b200_destroy(gpu_);
}

int Planner::AttachEngine(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                          mjpc_b200_t* borrowed) {
  owns_gpu_ = borrowed == nullptr;
  if (borrowed) gpu_ = borrowed;
  else if (int rc = mjpc_b200_create(model, max_candidates, max_horizon, device, &gpu_)) return rc;
  mjpc_b200_get_info(gpu_, &info_);
  state_.assign(info_.dim_state, 0.0); mocap_.assign(7 * info_.nmocap, 0.0);
  return 0;
}

void Planner::SetState(const double* state, double time, const double* mocap) {
  std::copy(state, state + state_.size(), state_.begin());
  if (mocap && !mocap_.empty()) std::copy(mocap, mocap + mocap_.size(), mocap_.begin());
  time_ = time;
}

int Planner::RolloutSpline(const float* knots, const double* knot_times, int interpolation, int P, int N, int horizon,
                           float* returns, uint8_t* failure, int* order) {
  const std::vector<float> st(state_.begin(), state_.end()), mc(mocap_.begin(), mocap_.end());
  horizon_ = horizon;
  return mjpc_b200_rollout_spline(gpu_, st.data(), time_, mc.empty() ? nullptr : mc.data(), nullptr, knots, knot_times,
                                  interpolation, P, N, horizon, returns, failure, order);
}

int Planner::FetchTrajectory(int candidate, int horizon, Trajectory* t) {
  const size_t H = horizon;
  t->horizon = horizon; t->dim_state = info_.dim_state; t->dim_action = info_.nu; t->dim_residual = info_.num_residual;
  t->dim_trace = 3 * info_.num_trace;
  t->states.resize(H * t->dim_state); t->actions.resize(H * t->dim_action); t->times.resize(H);
  t->residual.resize(H * t->dim_residual); t->costs.resize(H); t->trace.resize(H * t->dim_trace);
  return mjpc_b200_fetch_trajectory(gpu_, candidate, t->states.data(), t->actions.data(), t->times.data(),
                                    t->residual.data(), t->costs.data(), t->trace.data());
}

int CholFactor(double* M, int n, double mindiag) {
  int rank = 0;
  for (int j = 0; j < n; j++) {
    for (int k = 0; k < j; k++) M[(size_t)j * n + j] -= M[(size_t)j * n + k] * M[(size_t)j * n + k];
    double d = M[(size_t)j * n + j];
    if (d < mindiag) d = mindiag; else rank++;
    M[(size_t)j * n + j] = std::sqrt(d);
    for (int i = j + 1; i < n; i++) {
      for (int k = 0; k < j; k++) M[(size_t)i * n + j] -= M[(size_t)i * n + k] * M[(size_t)j * n + k];
      M[(size_t)i * n + j] /= M[(size_t)j * n + j];
    }
  }
  return rank;
}

void CholSolve(const double* L, int n, double* x) {
  for (int i = 0; i < n; i++) { double a = x[i]; for (int k = 0; k < i; k++) a -= L[(size_t)i * n + k] * x[k]; x[i] = a / L[(size_t)i * n + i]; }
  for (int i = n - 1; i >= 0; i--) { double a = x[i]; for (int k = i + 1; k < n; k++) a -= L[(size_t)k * n + i] * x[k]; x[i] = a / L[(size_t)i * n + i]; }
}

}  // namespace mjpc_b200_host
