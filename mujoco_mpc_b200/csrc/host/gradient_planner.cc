// gradient_planner.cc - see gradient_planner.h.  Host logic only; every sweep goes through the C ABI.
#include "gradient_planner.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>

namespace mjpc_b200_host {

namespace {
std::vector<double> LogScaleSteps(int K, double min_step) {   // LogScale (utilities.cc:819-825) + trailing 0
  std::vector<double> s(K, 0.0);
  const int steps = K - 1;
  if (steps > 0) LogScale(s.data(), 1.0, min_step, steps);
  s[K - 1] = 0.0;
  return s;
}
}  // namespace

void SplineMapping(int representation, const std::vector<double>& ti, const double* to, int T, std::vector<double>* Wout) {
  const int P = (int)ti.size();
  std::vector<double>& W = *Wout;
  W.assign((size_t)T * P, 0.0);
  int b[2];
  if (representation == 0) {                                   // ZeroSplineMapping (spline_mapping.cc:35-58)
    for (int i = 0; i < T; i++) { FindInterval(b, ti.data(), to[i], P); W[(size_t)i * P + b[0]] = 1.0; }
    return;
  }
  if (representation == 1) {                                   // LinearSplineMapping (:72-106)
    for (int i = 0; i < T; i++) {
      FindInterval(b, ti.data(), to[i], P);
      if (b[0] == b[1]) { W[(size_t)i * P + b[0]] = 1.0; continue; }
      const double a = (to[i] - ti[b[0]]) / (ti[b[1]] - ti[b[0]]);
      W[(size_t)i * P + b[0]] = 1.0 - a; W[(size_t)i * P + b[1]] = a;
    }
    return;
  }
  // CubicSplineMapping (:118-205): points + finite-difference slopes, then Hermite coefficients
  std::vector<double> S((size_t)2 * P * P, 0.0), O((size_t)T * 2 * P, 0.0);
  for (int i = 0; i < P; i++) S[(size_t)i * P + i] = 1.0;
  for (int i = 0; i < P; i++) {
    double dt1 = i > 0 ? 1.0 / (ti[i] - ti[i - 1]) : 0.0;
    double dt2 = i < P - 1 ? 1.0 / (ti[i + 1] - ti[i]) : 0.0;
    if (i > 0 && i < P - 1) { dt1 *= 0.5; dt2 *= 0.5; }
    double* row = &S[(size_t)(P + i) * P];
    if (i - 1 >= 0) row[i - 1] = -dt1;
    row[i] = dt1 - dt2;
    if (i + 1 <= P - 1) row[i + 1] = dt2;
  }
  for (int i = 0; i < T; i++) {
    FindInterval(b, ti.data(), to[i], P);
    double c[4] = {1.0, 0.0, 0.0, 0.0};
    if (b[0] != b[1]) {
      const double d = ti[b[1]] - ti[b[0]], t = (to[i] - ti[b[0]]) / d;
      c[0] = 2.0 * t * t * t - 3.0 * t * t + 1.0; c[1] = (t * t * t - 2.0 * t * t + t) * d;
      c[2] = -2.0 * t * t * t + 3 * t * t;         c[3] = (t * t * t - t * t) * d;
    }
    double* row = &O[(size_t)i * 2 * P];
    row[b[0]] = c[0]; row[P + b[0]] = c[1];
    if (b[0] != b[1]) { row[b[1]] = c[2]; row[P + b[1]] = c[3]; }
  }
  for (int i = 0; i < T; i++)
    for (int k = 0; k < 2 * P; k++) {
      const double o = O[(size_t)i * 2 * P + k];
      if (o == 0.0) continue;
      for (int p = 0; p < P; p++) W[(size_t)i * P + p] += o * S[(size_t)k * P + p];
    }
}

void GradientSweep(const float* A, const float* B, const float* cx, const float* cu, int n, int m, int T,
                   std::vector<double>* kout, double* dV0) {
  std::vector<double>& k = *kout;
  k.assign((size_t)T * m, 0.0);
  std::vector<double> Vx(cx + (size_t)(T - 1) * n, cx + (size_t)T * n), Qx(n), Qu(m);
  *dV0 = 0.0;
  for (int t = T - 1; t > 0; t--) {
    const float* At = A + (size_t)(t - 1) * n * n; const float* Bt = B + (size_t)(t - 1) * n * m;
    for (int j = 0; j < n; j++) { double a = cx[(size_t)(t - 1) * n + j]; for (int i = 0; i < n; i++) a += (double)At[(size_t)i * n + j] * Vx[i]; Qx[j] = a; }
    for (int j = 0; j < m; j++) { double a = cu[(size_t)(t - 1) * m + j]; for (int i = 0; i < n; i++) a += (double)Bt[(size_t)i * m + j] * Vx[i]; Qu[j] = a; }
    for (int j = 0; j < m; j++) { k[(size_t)(t - 1) * m + j] = -Qu[j]; *dV0 += -Qu[j] * Qu[j]; }
    Vx = Qx;
  }
  if (T >= 2) for (int j = 0; j < m; j++) k[(size_t)(T - 1) * m + j] = k[(size_t)(T - 2) * m + j];
}

void GradientPolicy::Action(double* action, double time) const {
  // the same function as TimeSpline::Sample for >= 3 points (see the header): reuse it
  TimeSpline s(nu, (SplineInterpolation)representation);
  for (int i = 0; i < num_spline_points; i++) s.AddNode(times[i], parameters.data() + (size_t)i * nu);
  s.Sample(time, action);
  for (int i = 0; i < nu; i++) action[i] = std::max(ctrlrange[2 * i], std::min(ctrlrange[2 * i + 1], action[i]));
}

int GradientPlanner::Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int representation,
                                double timestep, const double* ctrlrange, int max_horizon, int device) {
  K_ = std::max(num_trajectory, 1);
  if (int rc = AttachEngine(model, K_, max_horizon, device)) return rc;
  nu_ = info_.nu; n_ = info_.dim_dstate; nr_ = info_.num_residual; Hmax_ = info_.max_horizon;
  timestep_ = timestep;
  policy.nu = nu_; policy.num_spline_points = num_spline_points; policy.representation = representation;
  policy.ctrlrange.assign(ctrlrange, ctrlrange + 2 * nu_);
  Reset(max_horizon, nullptr);
  return 0;
}

void GradientPlanner::Reset(int, const double* a) {
  const std::unique_lock<std::shared_mutex> lock(mtx_);
  const int P = policy.num_spline_points;
  policy.parameters.assign((size_t)P * nu_, 0.0);
  if (a) for (int t = 0; t < P; t++) for (int i = 0; i < nu_; i++) policy.parameters[(size_t)t * nu_ + i] = a[i];
  policy.times.assign(P, 0.0);
  previous_policy = policy; cand_ = policy;
  winner = -1; action_step = expected = improvement = surprise = total_return = 0;
}

void GradientPlanner::ResamplePolicy(int horizon) {
  const int P = cand_.num_spline_points;
  const double shift = std::max((horizon - 1) * timestep_ / std::max(P - 1, 1), 1.0e-5);
  std::vector<double> p((size_t)P * nu_), t(P);
  double nominal_time = time_;
  for (int k = 0; k < P; k++) { t[k] = nominal_time; cand_.Action(&p[(size_t)k * nu_], nominal_time); nominal_time += shift; }
  cand_.parameters = p;
  for (int k = 0; k < P; k++) cand_.times[k] = t[0] + shift * k;     // LinearRange (planner.cc:381-382)
}

int GradientPlanner::Rollouts(const std::vector<double>& parameters, int count, int horizon) {
  const int P = cand_.num_spline_points;
  knots_.resize((size_t)count * P * nu_);
  for (size_t i = 0; i < knots_.size(); i++) knots_[i] = (float)parameters[i];
  ret_.assign(count, 0.f); fail_.assign(count, 0); order_.assign(count, 0);
  return RolloutSpline(knots_.data(), cand_.times.data(), cand_.representation, P, count, horizon, ret_.data(),
                       fail_.data(), order_.data());
}

int GradientPlanner::Fetch(int candidate, int horizon, double ret) {
  if (FetchTrajectory(candidate, horizon, &best_)) return -1;
  best_.total_return = ret; best_.failure = false;
  return 0;
}

int GradientPlanner::OptimizePolicy(int horizon) {
  if (horizon < 2 || horizon > Hmax_) return -1;
  const size_t H = horizon, n = n_, m = nu_, nr = nr_;
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  {
    const std::shared_lock<std::shared_mutex> lock(mtx_);
    cand_ = policy;
  }
  const int P = cand_.num_spline_points;
  ResamplePolicy(horizon);
  // nominal rollout: trajectory[0]
  if (Rollouts(cand_.parameters, 1, horizon)) return -1;
  const double c_prev = fail_[0] ? 1.0e6 : (double)ret_[0];
  if (Fetch(0, horizon, c_prev)) return -1;
  double c_best = c_prev;
  const std::vector<double> steps = LogScaleSteps(K_, settings.min_linesearch_step);
  A_.resize(H * n * n); B_.resize(H * n * m); C_.resize(H * nr * n); D_.resize(H * nr * m);
  cx_.resize(H * n); cu_.resize(H * m); cxx_.resize(H * n * n); cuu_.resize(H * m * m); cxu_.resize(H * n * m);
  std::vector<float> mc(mocap_.begin(), mocap_.end());
  std::vector<double> k, W, update((size_t)P * nu_), candidates((size_t)K_ * P * nu_);
  for (int c = 0; c < K_; c++) std::copy(cand_.parameters.begin(), cand_.parameters.end(), candidates.begin() + (size_t)c * P * nu_);
  winner = K_ - 1;
  for (int it = 0; it < settings.max_rollout; it++) {
    if (mjpc_b200_model_derivatives(gpu_, best_.states.data(), best_.actions.data(), best_.times.data(),
                                    mc.empty() ? nullptr : mc.data(), horizon, settings.derivative_skip,
                                    (float)settings.fd_tolerance, settings.fd_mode, A_.data(), B_.data(), C_.data(), D_.data()))
      return -1;
    if (mjpc_b200_cost_derivatives(gpu_, best_.residual.data(), C_.data(), D_.data(), horizon, cx_.data(), cu_.data(),
                                   cxx_.data(), cuu_.data(), cxu_.data()))
      return -1;
    double dV0 = 0;
    GradientSweep(A_.data(), B_.data(), cx_.data(), cu_.data(), (int)n, (int)m, horizon, &k, &dV0);
    SplineMapping(cand_.representation, cand_.times, best_.times.data(), horizon - 1, &W);
    std::fill(update.begin(), update.end(), 0.0);                       // parameter_update = mapping^T k (:240-245)
    for (int t = 0; t < horizon - 1; t++)
      for (int p = 0; p < P; p++) {
        const double w = W[(size_t)t * P + p];
        if (w == 0.0) continue;
        for (int j = 0; j < nu_; j++) update[(size_t)p * nu_ + j] += w * k[(size_t)t * nu_ + j];
      }
    for (int c = 0; c < K_; c++)                                        // Rollouts (:386-420): parameters += step * update
      for (size_t q = 0; q < (size_t)P * nu_; q++) candidates[(size_t)c * P * nu_ + q] = cand_.parameters[q] + steps[c] * update[q];
    if (Rollouts(candidates, K_, horizon)) return -1;
    winner = K_ - 1;
    for (int j = K_ - 1; j >= 0; j--) {
      const double c_sample = fail_[j] ? 1.0e6 : (double)ret_[j];
      if (c_sample < c_best) { c_best = c_sample; winner = j; }
    }
    std::copy(candidates.begin() + (size_t)winner * P * nu_, candidates.begin() + (size_t)(winner + 1) * P * nu_, cand_.parameters.begin());
    if (Fetch(winner, horizon, fail_[winner] ? 1.0e6 : (double)ret_[winner])) return -1;   // trajectory[0] = trajectory[winner]
    action_step = steps[winner];
    expected = -action_step * dV0 - 1.0e-16;
    improvement = c_prev - c_best;
    surprise = std::min(std::max(0.0, improvement / expected), 2.0);
  }
  if (c_best >= c_prev) {
    winner = K_ - 1;     // step 0: the resampled nominal
    std::copy(candidates.begin() + (size_t)winner * P * nu_, candidates.begin() + (size_t)(winner + 1) * P * nu_, cand_.parameters.begin());
  }
  {
    const std::unique_lock<std::shared_mutex> lock(mtx_);
    previous_policy = policy;
    policy.parameters = cand_.parameters; policy.times = cand_.times;     // CopyParametersFrom (:319-320)
  }
  total_return = c_best;
  return c_best < c_prev ? 1 : 0;
}

void GradientPlanner::ActionFromPolicy(double* action, const double*, double time, bool use_previous) {
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  (use_previous ? previous_policy : policy).Action(action, time);
}

// ------------------------------------------------------------------------------------------ iLQS
int iLQSPlanner::Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                            double exploration, double timestep, const double* ctrlrange, uint32_t seed, int ilqg_num_rollouts,
                            int ilqg_representation, double fd_tolerance, int max_horizon, int device) {
  int rc = sampling.Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep, ctrlrange,
                               seed, num_trajectory, max_horizon, device);
  if (rc) return rc;
  rc = ilqg.Initialize(model, ilqg_num_rollouts, ilqg_representation, max_horizon, device);
  if (rc) return rc;
  if (fd_tolerance > 0) ilqg.settings.fd_tolerance = fd_tolerance;
  nu_ = sampling.NumParameters() / std::max(sampling.policy.num_spline_points, 1);
  timestep_ = timestep;
  return 0;
}

void iLQSPlanner::Reset(int horizon, const double* a) {
  sampling.Reset(horizon, a); ilqg.Reset(horizon, a);
  active_policy = previous_active_policy = kSampling;
}

void iLQSPlanner::SetState(const double* state, double time, const double* mocap) {
  sampling.SetState(state, time, mocap); ilqg.SetState(state, time, mocap);
}

int iLQSPlanner::OptimizePolicy(int horizon) {
  previous_active_policy = active_policy;
  if (previous_active_policy == kiLQG) {
    // the trajectory policy of iLQG (the previous winner) -> spline parameters: least-squares inverse of the
    // parameter-to-action mapping (ilqs/planner.cc:98-172)
    if (ilqg.NominalTrajectory(horizon) < 0) return -1;
    const int P = sampling.policy.num_spline_points, T = horizon - 1;
    const double shift = std::max((horizon - 1) * timestep_ / std::max(P - 1, 1), 1.0e-5);
    std::vector<double> times(P), W;
    for (int t = 0; t < P; t++) times[t] = sampling.time() + shift * t;
    SplineMapping((int)sampling.interpolation(), times, ilqg.candidate_times().data(), T, &W);
    // M = W' W (P x P), Cholesky, parameters = M^-1 W' actions
    std::vector<double> M((size_t)P * P, 0.0), rhs((size_t)P * nu_, 0.0);
    for (int t = 0; t < T; t++)
      for (int p = 0; p < P; p++) {
        const double w = W[(size_t)t * P + p];
        if (w == 0.0) continue;
        for (int q = 0; q < P; q++) M[(size_t)p * P + q] += w * W[(size_t)t * P + q];
        for (int j = 0; j < nu_; j++) rhs[(size_t)p * nu_ + j] += w * (double)ilqg.candidate_actions()[(size_t)t * nu_ + j];
      }
    for (int j = 0; j < P; j++) {                                   // in-place Cholesky (mju_cholFactor)
      for (int k = 0; k < j; k++) M[(size_t)j * P + j] -= M[(size_t)j * P + k] * M[(size_t)j * P + k];
      M[(size_t)j * P + j] = std::sqrt(std::max(M[(size_t)j * P + j], 1e-15));
      for (int i = j + 1; i < P; i++) {
        for (int k = 0; k < j; k++) M[(size_t)i * P + j] -= M[(size_t)i * P + k] * M[(size_t)j * P + k];
        M[(size_t)i * P + j] /= M[(size_t)j * P + j];
      }
    }
    for (int j = 0; j < nu_; j++) {                                 // L L' x = rhs, column by column
      for (int i = 0; i < P; i++) { double a = rhs[(size_t)i * nu_ + j]; for (int k = 0; k < i; k++) a -= M[(size_t)i * P + k] * rhs[(size_t)k * nu_ + j]; rhs[(size_t)i * nu_ + j] = a / M[(size_t)i * P + i]; }
      for (int i = P - 1; i >= 0; i--) { double a = rhs[(size_t)i * nu_ + j]; for (int k = i + 1; k < P; k++) a -= M[(size_t)k * P + i] * rhs[(size_t)k * nu_ + j]; rhs[(size_t)i * nu_ + j] = a / M[(size_t)i * P + i]; }
    }
    const std::vector<double>& cr = sampling.policy.ctrlrange;
    for (int t = 0; t < P; t++)
      for (int j = 0; j < nu_; j++) rhs[(size_t)t * nu_ + j] = std::max(cr[2 * j], std::min(cr[2 * j + 1], rhs[(size_t)t * nu_ + j]));
    sampling.SetPolicy(times.data(), rhs.data(), P);
  }
  // try sampling
  if (sampling.OptimizePolicy(horizon) < 0) return -1;
  const double ref = previous_active_policy == kSampling ? (double)sampling.returns()[0] : ilqg.candidate_return();
  if (sampling.winner > 0 && (double)sampling.returns()[sampling.winner] < ref) {
    active_policy = kSampling;   // best rollout is from sampling: terminate early (:190-207)
    return 1;
  }
  if (previous_active_policy == kSampling) {
    Trajectory t0;               // ilqg.candidate_policy[0].trajectory = sampling.trajectory[0] (:209-212)
    if (sampling.CandidateTrajectory(0, horizon, &t0)) return -1;
    ilqg.SetCandidateTrajectory(t0);
  }
  const int ok = ilqg.Iteration(horizon);
  if (ok < 0) return -1;
  if (ok == 1) {
    // ilqg.trajectory[0] is the action rollout with the SMALLEST non-zero step (LogScale ascends): restated literally (:220-224)
    const double old = previous_active_policy == kSampling ? (double)sampling.returns()[sampling.winner] : (double)ilqg.rollout_return(0);
    if (ilqg.total_return < old) active_policy = kiLQG;
  }
  return ok;
}

int iLQSPlanner::NominalTrajectory(int horizon) {
  if (active_policy == kSampling) return sampling.NominalTrajectory(horizon) ? -1 : 1;
  return ilqg.NominalTrajectory(horizon);
}

void iLQSPlanner::ActionFromPolicy(double* action, const double* state, double time, bool use_previous) {
  if (use_previous && previous_active_policy == kSampling) { sampling.ActionFromPolicy(action, state, time, true); return; }
  if (!use_previous && active_policy == kSampling) { sampling.ActionFromPolicy(action, state, time, false); return; }
  ilqg.ActionFromPolicy(action, state, time);
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::GradientPlanner;
using mjpc_b200_host::iLQSPlanner;

extern "C" {

void mjpc_b200_host_spline_mapping(int representation, const double* input_times, int num_input, const double* output_times,
                                   int num_output, double* W) {
  std::vector<double> ti(input_times, input_times + num_input), w;
  mjpc_b200_host::SplineMapping(representation, ti, output_times, num_output, &w);
  std::copy(w.begin(), w.end(), W);
}

int mjpc_b200_gradient_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int representation,
                                      double fd_tolerance, double timestep, const double* ctrlrange, int max_horizon, int device,
                                      void** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 1 || num_spline_points < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new GradientPlanner;
  int rc = p->Initialize(model, num_trajectory, num_spline_points, representation, timestep, ctrlrange, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  if (fd_tolerance > 0) p->settings.fd_tolerance = fd_tolerance;
  *out = p;
  return 0;
}
void mjpc_b200_gradient_planner_destroy(void* p) { delete (GradientPlanner*)p; }
void mjpc_b200_gradient_planner_set_fd(void* p, double tolerance, int mode, int derivative_skip) {
  auto& s = ((GradientPlanner*)p)->settings;
  if (tolerance > 0) s.fd_tolerance = tolerance;
  if (mode >= 0) s.fd_mode = mode ? 1 : 0;
  if (derivative_skip >= 0) s.derivative_skip = derivative_skip;
}
void mjpc_b200_gradient_planner_reset(void* p, int horizon, const double* a) { ((GradientPlanner*)p)->Reset(horizon, a); }
void mjpc_b200_gradient_planner_set_state(void* p, const double* state, double time, const double* mocap) {
  ((GradientPlanner*)p)->SetState(state, time, mocap);
}
int mjpc_b200_gradient_planner_optimize_policy(void* p, int horizon) { return ((GradientPlanner*)p)->OptimizePolicy(horizon); }
void mjpc_b200_gradient_planner_action_from_policy(void* p, double* action, double time, int use_previous) {
  ((GradientPlanner*)p)->ActionFromPolicy(action, nullptr, time, use_previous != 0);
}
// scalars[6] = {total_return, winner, action_step, expected, improvement, surprise}; parameters [P][nu], times [P]
int mjpc_b200_gradient_planner_get_result(void* pv, double* scalars, double* parameters, double* times) {
  auto* p = (GradientPlanner*)pv;
  if (scalars) {
    scalars[0] = p->total_return; scalars[1] = p->winner; scalars[2] = p->action_step; scalars[3] = p->expected;
    scalars[4] = p->improvement; scalars[5] = p->surprise;
  }
  if (parameters) std::copy(p->policy.parameters.begin(), p->policy.parameters.end(), parameters);
  if (times) std::copy(p->policy.times.begin(), p->policy.times.end(), times);
  return p->policy.num_spline_points;
}

int mjpc_b200_ilqs_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                                  double exploration, double timestep, const double* ctrlrange, uint32_t seed,
                                  int ilqg_num_rollouts, int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                                  void** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 1 || ilqg_num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new iLQSPlanner;
  int rc = p->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, timestep, ctrlrange, seed,
                         ilqg_num_rollouts, ilqg_representation, fd_tolerance, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  *out = p;
  return 0;
}
void mjpc_b200_ilqs_planner_destroy(void* p) { delete (iLQSPlanner*)p; }
void mjpc_b200_ilqs_planner_set_fd(void* p, double tolerance, int mode, int derivative_skip) {
  auto& s = ((iLQSPlanner*)p)->ilqg.settings;
  if (tolerance > 0) s.fd_tolerance = tolerance;
  if (mode >= 0) s.fd_mode = mode ? 1 : 0;
  if (derivative_skip >= 0) s.derivative_skip = derivative_skip;
}
void mjpc_b200_ilqs_planner_reset(void* p, int horizon, const double* a) { ((iLQSPlanner*)p)->Reset(horizon, a); }
void mjpc_b200_ilqs_planner_set_state(void* p, const double* state, double time, const double* mocap) {
  ((iLQSPlanner*)p)->SetState(state, time, mocap);
}
void mjpc_b200_ilqs_planner_set_exploration(void* p, double exploration) { ((iLQSPlanner*)p)->sampling.SetExploration(exploration, 0.0); }
int mjpc_b200_ilqs_planner_optimize_policy(void* p, int horizon) { return ((iLQSPlanner*)p)->OptimizePolicy(horizon); }
void mjpc_b200_ilqs_planner_action_from_policy(void* p, double* action, const double* state, double time, int use_previous) {
  ((iLQSPlanner*)p)->ActionFromPolicy(action, state, time, use_previous != 0);
}
// scalars[4] = {active_policy (0 sampling, 1 iLQG), sampling winner return, iLQG total_return, sampling winner}
int mjpc_b200_ilqs_planner_get_result(void* pv, double* scalars) {
  auto* p = (iLQSPlanner*)pv;
  if (scalars) {
    scalars[0] = p->active_policy; scalars[1] = p->sampling.returns()[p->sampling.winner]; scalars[2] = p->ilqg.total_return;
    scalars[3] = p->sampling.winner;
  }
  return p->active_policy;
}

}  // extern "C"
