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
                                double timestep, const double* ctrlrange, int max_horizon, int device, mjpc_b200_t* borrowed) {
  K_ = std::max(num_trajectory, 1);
  if (int rc = AttachEngine(model, K_, max_horizon, device, borrowed)) return rc;
  nu_ = info_.nu; nr_ = info_.num_residual; Hmax_ = info_.max_horizon;
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

void GradientPlanner::Candidates(const std::vector<double>& parameters, int count, SplineCandidates* c) const {
  const int P = cand_.num_spline_points;
  c->Resize(count, P, nu_);
  c->interpolation = cand_.representation;
  for (size_t i = 0; i < c->knots.size(); i++) c->knots[i] = (float)parameters[i];
  std::copy(cand_.times.begin(), cand_.times.end(), c->knot_times.begin());
}

int GradientPlanner::Fetch(int candidate, int horizon, double ret) {
  if (FetchTrajectory(candidate, horizon, &best_)) return -1;
  best_.total_return = ret; best_.failure = false;
  return 0;
}

const SplineCandidates* GradientPlanner::PrepareNominal(int horizon) {
  if (horizon < 2 || horizon > Hmax_) return nullptr;
  {
    const std::shared_lock<std::shared_mutex> lock(mtx_);
    cand_ = policy;
  }
  ResamplePolicy(horizon);
  Candidates(cand_.parameters, 1, &nominal_);   // nominal rollout: trajectory[0]
  return &nominal_;
}

int GradientPlanner::InstallNominal(int horizon, const float* returns, const uint8_t* failure, int offset) {
  launch_offset_ = offset; horizon_ = horizon;
  c_prev_ = failure[0] ? 1.0e6 : (double)returns[0];
  if (Fetch(0, horizon, c_prev_)) return -1;
  c_best_ = c_prev_;
  steps_ = LogScaleSteps(K_, settings.min_linesearch_step);
  const size_t Pn = (size_t)cand_.num_spline_points * nu_;
  update_.resize(Pn); candidates_.resize((size_t)K_ * Pn);
  for (int c = 0; c < K_; c++) std::copy(cand_.parameters.begin(), cand_.parameters.end(), candidates_.begin() + c * Pn);
  winner = K_ - 1;
  return 0;
}

const SplineCandidates& GradientPlanner::PrepareLineSearch(int horizon, const double* k, double dV0) {
  const int P = cand_.num_spline_points;
  dV0_ = dV0;
  SplineMapping(cand_.representation, cand_.times, best_.times.data(), horizon - 1, &W_);
  std::fill(update_.begin(), update_.end(), 0.0);                      // parameter_update = mapping^T k (:240-245)
  for (int t = 0; t < horizon - 1; t++)
    for (int p = 0; p < P; p++) {
      const double w = W_[(size_t)t * P + p];
      if (w == 0.0) continue;
      for (int j = 0; j < nu_; j++) update_[(size_t)p * nu_ + j] += w * k[(size_t)t * nu_ + j];
    }
  for (int c = 0; c < K_; c++)                                        // Rollouts (:386-420): parameters += step * update
    for (size_t q = 0; q < (size_t)P * nu_; q++) candidates_[(size_t)c * P * nu_ + q] = cand_.parameters[q] + steps_[c] * update_[q];
  Candidates(candidates_, K_, &lines_);
  return lines_;
}

int GradientPlanner::InstallLineSearch(int horizon, const float* returns, const uint8_t* failure, int offset) {
  const size_t Pn = (size_t)cand_.num_spline_points * nu_;
  launch_offset_ = offset; horizon_ = horizon;
  winner = K_ - 1;
  for (int j = K_ - 1; j >= 0; j--) {
    const double c_sample = failure[j] ? 1.0e6 : (double)returns[j];
    if (c_sample < c_best_) { c_best_ = c_sample; winner = j; }
  }
  std::copy(candidates_.begin() + winner * Pn, candidates_.begin() + (winner + 1) * Pn, cand_.parameters.begin());
  if (Fetch(winner, horizon, failure[winner] ? 1.0e6 : (double)returns[winner])) return -1;   // trajectory[0] = trajectory[winner]
  action_step = steps_[winner];
  expected = -action_step * dV0_ - 1.0e-16;
  improvement = c_prev_ - c_best_;
  surprise = std::min(std::max(0.0, improvement / expected), 2.0);
  return 0;
}

int GradientPlanner::Publish() {
  const size_t Pn = (size_t)cand_.num_spline_points * nu_;
  if (c_best_ >= c_prev_) {
    winner = K_ - 1;     // step 0: the resampled nominal
    std::copy(candidates_.begin() + winner * Pn, candidates_.begin() + (winner + 1) * Pn, cand_.parameters.begin());
  }
  {
    const std::unique_lock<std::shared_mutex> lock(mtx_);
    previous_policy = policy;
    policy.parameters = cand_.parameters; policy.times = cand_.times;     // CopyParametersFrom (:319-320)
  }
  total_return = c_best_;
  return c_best_ < c_prev_ ? 1 : 0;
}

int GradientPlanner::Iterate(const std::vector<GradientPlanner*>& ps, const TaskRows& rows, int horizon,
                             SplineLaunch* launch, int* improved) {
  const size_t B = ps.size();
  std::fill(improved, improved + B, 0);
  const GradientPlannerSettings& s = ps[0]->settings;
  const DifferentiableScope diff(ps[0]->gpu_, s.differentiable != 0);
  const std::vector<const Planner*> from(ps.begin(), ps.end());
  std::vector<const SplineCandidates*> cands(B);
  for (size_t b = 0; b < B; b++)
    if (!(cands[b] = ps[b]->PrepareNominal(horizon))) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = launch->Run(from, cands, rows, horizon)) return rc;
  for (size_t b = 0; b < B; b++)
    if (ps[b]->InstallNominal(horizon, launch->returns.data() + b, launch->failure.data() + b, (int)b)) return -1;
  // the nominals' trajectories [B][H][..] and mocaps [B][7 nmocap] (float, as the handle stages its own)
  const size_t H = horizon, ds = ps[0]->info_.dim_state, nu = ps[0]->nu_, nr = ps[0]->nr_, nm = ps[0]->mocap_.size();
  std::vector<float> x(B * H * ds), u(B * H * nu), res(B * H * nr), mc(B * nm);
  std::vector<double> t(B * H), k(B * H * nu), dV0(B);
  for (int it = 0; it < s.max_rollout; it++) {
    for (size_t b = 0; b < B; b++) {
      const Trajectory& tr = ps[b]->best_;
      std::copy(tr.states.begin(), tr.states.begin() + H * ds, x.begin() + b * H * ds);
      std::copy(tr.actions.begin(), tr.actions.begin() + H * nu, u.begin() + b * H * nu);
      std::copy(tr.residual.begin(), tr.residual.begin() + H * nr, res.begin() + b * H * nr);
      std::copy(tr.times.begin(), tr.times.begin() + H, t.begin() + b * H);
      std::copy(ps[b]->mocap_.begin(), ps[b]->mocap_.end(), mc.begin() + b * nm);
    }
    if (int rc = mjpc_b200_gradient_batched(ps[0]->gpu_, (int)B, x.data(), u.data(), t.data(), nm ? mc.data() : nullptr,
                                            rows.nw ? rows.w : nullptr, rows.np ? rows.p : nullptr,
                                            rows.nts ? rows.ts : nullptr, res.data(), horizon, s.derivative_skip,
                                            (float)s.fd_tolerance, s.fd_mode, k.data(), dV0.data()))
      return rc;
    for (size_t b = 0; b < B; b++) cands[b] = &ps[b]->PrepareLineSearch(horizon, k.data() + b * H * nu, dV0[b]);
    if (int rc = launch->Run(from, cands, rows, horizon)) return rc;
    const int K = cands[0]->N;
    for (size_t b = 0; b < B; b++) {
      const size_t o = b * K;
      if (ps[b]->InstallLineSearch(horizon, launch->returns.data() + o, launch->failure.data() + o, (int)o)) return -1;
    }
  }
  for (size_t b = 0; b < B; b++) improved[b] = ps[b]->Publish();
  return 0;
}

int GradientPlanner::OptimizePolicy(int horizon) {
  int improved = 0;
  return Iterate({this}, TaskRows(), horizon, &launch_, &improved) ? -1 : improved;
}

void GradientPlanner::ActionFromPolicy(double* action, const double*, double time, bool use_previous) {
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  (use_previous ? previous_policy : policy).Action(action, time);
}

// ------------------------------------------------------------------------------------------ iLQS
int iLQSPlanner::Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                            double exploration, double timestep, const double* ctrlrange, uint32_t seed, int ilqg_num_rollouts,
                            int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                            mjpc_b200_t* sampling_gpu, mjpc_b200_t* ilqg_gpu) {
  int rc = sampling.Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep, ctrlrange,
                               seed, num_trajectory, max_horizon, device, sampling_gpu);
  if (rc) return rc;
  rc = ilqg.Initialize(model, ilqg_num_rollouts, ilqg_representation, max_horizon, device, ilqg_gpu);
  if (rc) return rc;
  ilqg.SetFD(fd_tolerance, -1, -1);
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

void iLQSPlanner::ConvertToSpline(int horizon) {
  // the trajectory policy of iLQG (the previous winner) -> spline parameters: least-squares inverse of the
  // parameter-to-action mapping (ilqs/planner.cc:98-172)
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
  CholFactor(M.data(), P, 1e-15);                                 // in-place Cholesky (mju_cholFactor)
  for (int j = 0; j < nu_; j++) {                                 // L L' x = rhs, column by column
    for (int i = 0; i < P; i++) { double a = rhs[(size_t)i * nu_ + j]; for (int k = 0; k < i; k++) a -= M[(size_t)i * P + k] * rhs[(size_t)k * nu_ + j]; rhs[(size_t)i * nu_ + j] = a / M[(size_t)i * P + i]; }
    for (int i = P - 1; i >= 0; i--) { double a = rhs[(size_t)i * nu_ + j]; for (int k = i + 1; k < P; k++) a -= M[(size_t)k * P + i] * rhs[(size_t)k * nu_ + j]; rhs[(size_t)i * nu_ + j] = a / M[(size_t)i * P + i]; }
  }
  const std::vector<double>& cr = sampling.policy.ctrlrange;
  for (int t = 0; t < P; t++)
    for (int j = 0; j < nu_; j++) rhs[(size_t)t * nu_ + j] = std::max(cr[2 * j], std::min(cr[2 * j + 1], rhs[(size_t)t * nu_ + j]));
  sampling.SetPolicy(times.data(), rhs.data(), P);
}

int iLQSPlanner::SamplingSettled(int horizon) {
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
  return 0;
}

int iLQSPlanner::Accept(int ok) {
  if (ok == 1) {
    // ilqg.trajectory[0] is the action rollout with the SMALLEST non-zero step (LogScale ascends): restated literally (:220-224)
    const double old = previous_active_policy == kSampling ? (double)sampling.returns()[sampling.winner] : (double)ilqg.rollout_return(0);
    if (ilqg.total_return < old) active_policy = kiLQG;
  }
  return ok;
}

int iLQSPlanner::Iterate(const std::vector<iLQSPlanner*>& ps, const TaskRows& rows, int horizon, SplineLaunch* launch,
                         ILQGSweeps* sweeps, int* improved) {
  const int B = (int)ps.size();
  std::fill(improved, improved + B, 0);
  mjpc_b200_t* ilqg_gpu = ps[0]->ilqg.gpu();
  const bool diff = ps[0]->ilqg.settings.differentiable != 0;
  auto ilqg_of = [&](const std::vector<int>& idx) {
    std::vector<iLQGPlanner*> q;
    for (int b : idx) q.push_back(&ps[b]->ilqg);
    return q;
  };
  // the iLQG nominals of the problems whose active policy was iLQG, then their conversion to splines
  std::vector<int> conv;
  for (int b = 0; b < B; b++) {
    ps[b]->BeginIteration();
    if (ps[b]->previous_active_policy == kiLQG) conv.push_back(b);
  }
  if (!conv.empty()) {
    const DifferentiableScope d(ilqg_gpu, diff);
    if (sweeps->Nominal(ilqg_of(conv), conv, rows, horizon, nullptr)) return -1;
  }
  for (int b : conv) ps[b]->ConvertToSpline(horizon);
  // try sampling: every problem in one launch
  std::vector<SamplingPlanner*> sampling(B);
  for (int b = 0; b < B; b++) sampling[b] = &ps[b]->sampling;
  if (int rc = SamplingPlanner::Iterate(sampling, rows, horizon, launch)) return rc;
  std::vector<int> rest;
  for (int b = 0; b < B; b++) {
    const int settled = ps[b]->SamplingSettled(horizon);
    if (settled < 0) return -1;
    if (settled) improved[b] = 1;
    else rest.push_back(b);
  }
  // one iLQG iteration of the problems sampling did not settle
  if (rest.empty()) return 0;
  std::vector<int> updated(rest.size(), 0);
  {
    const DifferentiableScope d(ilqg_gpu, diff);
    if (sweeps->Iterate(ilqg_of(rest), rest, rows, horizon, updated.data())) return -1;
  }
  for (size_t j = 0; j < rest.size(); j++) improved[rest[j]] = ps[rest[j]]->Accept(updated[j]);
  return 0;
}

int iLQSPlanner::OptimizePolicy(int horizon) {
  int improved = 0;
  return Iterate({this}, TaskRows(), horizon, &launch_, &sweeps_, &improved) ? -1 : improved;
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
using mjpc_b200_host::PlannerOf;

extern "C" {

void mjpc_b200_host_spline_mapping(int representation, const double* input_times, int num_input, const double* output_times,
                                   int num_output, double* W) {
  std::vector<double> ti(input_times, input_times + num_input), w;
  mjpc_b200_host::SplineMapping(representation, ti, output_times, num_output, &w);
  std::copy(w.begin(), w.end(), W);
}

void mjpc_b200_host_gradient_sweep(const float* A, const float* B, const float* cx, const float* cu, int n, int m, int T,
                                   double* k, double* dV0) {
  std::vector<double> kv;
  mjpc_b200_host::GradientSweep(A, B, cx, cu, n, m, T, &kv, dV0);
  std::copy(kv.begin(), kv.end(), k);
}

int mjpc_b200_gradient_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int representation,
                                      double fd_tolerance, double timestep, const double* ctrlrange, int max_horizon, int device,
                                      mjpc_b200_planner_t** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 1 || num_spline_points < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new GradientPlanner;
  int rc = p->Initialize(model, num_trajectory, num_spline_points, representation, timestep, ctrlrange, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  p->SetFD(fd_tolerance, -1, -1);
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
// scalars[6] = {total_return, winner, action_step, expected, improvement, surprise}; parameters [P][nu], times [P]
int mjpc_b200_gradient_planner_get_result(mjpc_b200_planner_t* h, double* scalars, double* parameters, double* times) {
  auto* p = PlannerOf<GradientPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
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
                                  mjpc_b200_planner_t** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 1 || ilqg_num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new iLQSPlanner;
  int rc = p->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, timestep, ctrlrange, seed,
                         ilqg_num_rollouts, ilqg_representation, fd_tolerance, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
int mjpc_b200_ilqs_planner_set_exploration(mjpc_b200_planner_t* h, double exploration) {
  auto* p = PlannerOf<iLQSPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  p->sampling.SetExploration(exploration, 0.0);
  return 0;
}
// scalars[4] = {active_policy (0 sampling, 1 iLQG), sampling winner return, iLQG total_return, sampling winner}
int mjpc_b200_ilqs_planner_get_result(mjpc_b200_planner_t* h, double* scalars) {
  auto* p = PlannerOf<iLQSPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (scalars) {
    scalars[0] = p->active_policy; scalars[1] = p->sampling.returns()[p->sampling.winner]; scalars[2] = p->ilqg.total_return;
    scalars[3] = p->sampling.winner;
  }
  return p->active_policy;
}

}  // extern "C"
