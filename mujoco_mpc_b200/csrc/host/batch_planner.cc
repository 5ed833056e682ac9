// batch_planner.cc - see batch_planner.h.  Compiled into libmjpc_b200.so next to the engine.
#include "batch_planner.h"

#include <algorithm>
#include <exception>

#include "../dev_model.h"   // Blob reader (plain C++)

namespace mjpc_b200_host {

BatchPlanner::~BatchPlanner() {
  problems_.clear();   // the planners borrow the handle
  if (gpu_) mjpc_b200_destroy(gpu_);
}

int BatchPlanner::Attach(const mjpc_model_blob* model, int num_problems, int max_candidates, int max_horizon, int device) {
  try {
    mjpc_dev::Blob blob(model->data, model->nbytes);
    weight_ = blob.reals("task_weight"); parameters_ = blob.reals("task_parameters"); task_state_ = blob.reals("task_state");
  } catch (const std::exception&) {
    return MJPC_B200_ERR_BAD_BLOB;
  }
  nw_ = (int)weight_.size(); np_ = (int)parameters_.size(); nts_ = (int)task_state_.size();
  std::vector<double> w(weight_), p(parameters_), s(task_state_);
  for (int b = 1; b < num_problems; b++) {
    weight_.insert(weight_.end(), w.begin(), w.end());
    parameters_.insert(parameters_.end(), p.begin(), p.end());
    task_state_.insert(task_state_.end(), s.begin(), s.end());
  }
  if (int rc = mjpc_b200_create(model, max_candidates, max_horizon, device, &gpu_)) return rc;
  mjpc_b200_info info;
  mjpc_b200_get_info(gpu_, &info);
  states_.resize((size_t)num_problems * info.dim_state);
  mocaps_.resize((size_t)num_problems * 7 * info.nmocap);
  times_.resize(num_problems);
  return 0;
}

void BatchPlanner::SetTask(int b, const double* weight, const double* parameters, const double* task_state) {
  if (weight) std::copy(weight, weight + nw_, weight_.begin() + (size_t)b * nw_);
  if (parameters) std::copy(parameters, parameters + np_, parameters_.begin() + (size_t)b * np_);
  if (task_state) std::copy(task_state, task_state + nts_, task_state_.begin() + (size_t)b * nts_);
}

int BatchPlanner::LaunchSpline(mjpc_b200_t* gpu, const std::vector<const SplineCandidates*>& cands, int horizon) {
  const int B = NumProblems(), N = cands[0]->N, P = cands[0]->P, interp = cands[0]->interpolation;
  for (const SplineCandidates* c : cands)
    if (c->N != N || c->P != P || c->interpolation != interp) return MJPC_B200_ERR_BAD_ARGUMENT;
  const size_t nk = cands[0]->knots.size();   // N P nu
  knots_.resize((size_t)B * nk);
  knot_times_.resize((size_t)B * P);
  for (int b = 0; b < B; b++) {
    const Planner& pl = launcher(b);
    std::copy(cands[b]->knots.begin(), cands[b]->knots.begin() + nk, knots_.begin() + b * nk);
    std::copy(cands[b]->knot_times.begin(), cands[b]->knot_times.begin() + P, knot_times_.begin() + (size_t)b * P);
    const size_t ds = pl.state().size(), nm = pl.mocap().size();
    std::copy(pl.state().begin(), pl.state().end(), states_.begin() + b * ds);
    std::copy(pl.mocap().begin(), pl.mocap().end(), mocaps_.begin() + b * nm);
    times_[b] = pl.time();
  }
  returns_.resize((size_t)B * N); failure_.resize(returns_.size()); order_.resize(returns_.size());
  return mjpc_b200_rollout_spline_batched(gpu, B, states_.data(), times_.data(), mocaps_.empty() ? nullptr : mocaps_.data(),
                                          nw_ ? weight_.data() : nullptr, np_ ? parameters_.data() : nullptr,
                                          nts_ ? task_state_.data() : nullptr, knots_.data(), knot_times_.data(), interp,
                                          P, N, horizon, returns_.data(), failure_.data(), order_.data());
}

TaskRows BatchPlanner::Rows() const {
  TaskRows r;
  r.w = weight_.data(); r.p = parameters_.data(); r.ts = task_state_.data(); r.nw = nw_; r.np = np_; r.nts = nts_;
  return r;
}

// ------------------------------------------------------------------------------------------ Cross-Entropy
int BatchCrossEntropyPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int n_elite,
                                         int num_spline_points, int interpolation, double std_initial, double std_min,
                                         double explore_fraction, double timestep, const double* ctrlrange,
                                         const uint32_t* seeds, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * (num_trajectory + 1), max_horizon, device)) return rc;
  for (int b = 0; b < num_problems; b++) {
    auto* p = new CrossEntropyPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, n_elite, num_spline_points, interpolation, std_initial, std_min,
                               explore_fraction, timestep, ctrlrange, seeds[b], max_horizon, device, gpu_))
      return rc;
  }
  return 0;
}

int BatchCrossEntropyPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++) cands[b] = &planner(b).PrepareCandidates(horizon);
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  const int N1 = cands[0]->N;
  for (int b = 0; b < B; b++) {
    const size_t o = (size_t)b * N1;
    planner(b).InstallRollouts(horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ Sample Gradient
int BatchSampleGradientPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                           int num_gradient, int num_spline_points, int interpolation,
                                           double exploration, double gradient_filter, double timestep,
                                           const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * num_trajectory, max_horizon, device)) return rc;
  for (int b = 0; b < num_problems; b++) {
    auto* p = new SampleGradientPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, num_gradient, num_spline_points, interpolation, exploration,
                               gradient_filter, timestep, ctrlrange, seeds[b], max_horizon, device, gpu_))
      return rc;
  }
  return 0;
}

int BatchSampleGradientPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++) cands[b] = &planner(b).PrepareCandidates(horizon);
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  const int N = cands[0]->N;
  for (int b = 0; b < B; b++) {
    const size_t o = (size_t)b * N;
    planner(b).InstallRollouts(horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ Robust
BatchRobustPlanner::~BatchRobustPlanner() {
  problems_.clear();   // the planners borrow both handles
  if (noisy_gpu_) mjpc_b200_destroy(noisy_gpu_);
}

int BatchRobustPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                   int num_spline_points, int interpolation, double exploration, double timestep,
                                   const double* ctrlrange, const uint32_t* seeds, int ncandidates, int nrepetitions,
                                   double xfrc_std, double xfrc_rate, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  const int rep = nrepetitions > 0 ? nrepetitions : 5;
  const int nc = ncandidates != -1 ? ncandidates : num_trajectory / rep;
  if (int rc = Attach(model, num_problems, num_problems * num_trajectory, max_horizon, device)) return rc;
  if (int rc = mjpc_b200_create(model, num_problems * std::max(nc * rep, 1), max_horizon, device, &noisy_gpu_)) return rc;
  seeds_.resize(num_problems);
  for (int b = 0; b < num_problems; b++) {
    std::unique_ptr<SamplingPlanner> d(new SamplingPlanner);
    if (int rc = d->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep,
                               ctrlrange, seeds[b], num_trajectory, max_horizon, device, gpu_))
      return rc;
    auto* p = new RobustPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(std::move(d), model, std::max(nc * rep, 1), max_horizon, device, noisy_gpu_)) return rc;
    p->Configure(num_trajectory, ncandidates, nrepetitions, xfrc_std, xfrc_rate, seeds[b]);
  }
  return 0;
}

int BatchRobustPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  // the delegates' OptimizePolicyCandidates: one clean launch
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++) cands[b] = &planner(b).delegate()->PrepareOptimize(horizon);
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  const int N = cands[0]->N;
  int noisy = 0;
  for (int b = 0; b < B; b++) {
    RobustPlanner& p = planner(b);
    const size_t o = (size_t)b * N;
    p.delegate()->InstallRollouts(N, horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
    noisy = p.PrepareNoisy(p.TopCandidates());   // the same for every problem: ncandidates and N are common
    cands[b] = &p.noisy();
    seeds_[b] = p.NoiseSeed();
  }
  if (noisy <= 0) return noisy;
  // the noisy re-evaluations: one launch, each problem with its own noise key
  RobustPlanner& p0 = planner(0);
  if (int rc = mjpc_b200_set_xfrc_noise_batched(noisy_gpu_, p0.xfrc_std(), p0.xfrc_rate(), B, seeds_.data())) return rc;
  if (int rc = LaunchSpline(noisy_gpu_, cands, horizon)) return rc;
  for (int b = 0; b < B; b++)
    planner(b).InstallNoisy(returns_.data() + (size_t)b * noisy, failure_.data() + (size_t)b * noisy);
  return 0;
}

// ------------------------------------------------------------------------------------------ Gradient
int BatchGradientPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                     int num_spline_points, int representation, double timestep,
                                     const double* ctrlrange, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * std::max(num_trajectory, 1), max_horizon, device)) return rc;
  improved_.assign(num_problems, 0);
  for (int b = 0; b < num_problems; b++) {
    auto* p = new GradientPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, num_spline_points, representation, timestep, ctrlrange,
                               max_horizon, device, gpu_))
      return rc;
  }
  return 0;
}

int BatchGradientPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  std::fill(improved_.begin(), improved_.end(), 0);
  const GradientPlannerSettings& s = planner(0).settings;
  const DifferentiableScope diff(gpu_, s.differentiable != 0);
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++)
    if (!(cands[b] = planner(b).PrepareNominal(horizon))) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  for (int b = 0; b < B; b++)
    if (planner(b).InstallNominal(horizon, returns_.data() + b, failure_.data() + b, b)) return -1;
  const size_t H = horizon;
  const Trajectory& t0 = planner(0).nominal();
  const size_t ds = t0.dim_state, nu = t0.dim_action, nr = t0.dim_residual, nm = planner(0).mocap().size();
  x_.resize(B * H * ds); u_.resize(B * H * nu); res_.resize(B * H * nr); t_.resize(B * H); mc_.resize(B * nm);
  k_.resize(B * H * nu); dV0_.resize(B);
  for (int it = 0; it < s.max_rollout; it++) {
    for (int b = 0; b < B; b++) {
      const Trajectory& tr = planner(b).nominal();
      std::copy(tr.states.begin(), tr.states.begin() + H * ds, x_.begin() + b * H * ds);
      std::copy(tr.actions.begin(), tr.actions.begin() + H * nu, u_.begin() + b * H * nu);
      std::copy(tr.residual.begin(), tr.residual.begin() + H * nr, res_.begin() + b * H * nr);
      std::copy(tr.times.begin(), tr.times.begin() + H, t_.begin() + b * H);
      const std::vector<double>& mc = planner(b).mocap();
      std::copy(mc.begin(), mc.end(), mc_.begin() + b * nm);   // float, as the single planner passes it
    }
    if (int rc = mjpc_b200_gradient_batched(gpu_, B, x_.data(), u_.data(), t_.data(), nm ? mc_.data() : nullptr,
                                            weights(), parameters(), task_states(), res_.data(), horizon,
                                            s.derivative_skip, (float)s.fd_tolerance, s.fd_mode, k_.data(),
                                            dV0_.data()))
      return rc;
    for (int b = 0; b < B; b++) cands[b] = &planner(b).PrepareLineSearch(horizon, k_.data() + b * H * nu, dV0_[b]);
    if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
    const int K = cands[0]->N;
    for (int b = 0; b < B; b++) {
      const size_t o = (size_t)b * K;
      if (planner(b).InstallLineSearch(horizon, returns_.data() + o, failure_.data() + o, (int)o)) return -1;
    }
  }
  for (int b = 0; b < B; b++) improved_[b] = planner(b).Publish();
  return 0;
}

// ------------------------------------------------------------------------------------------ iLQS
BatchILQSPlanner::~BatchILQSPlanner() {
  problems_.clear();   // the planners borrow both handles
  if (ilqg_gpu_) mjpc_b200_destroy(ilqg_gpu_);
}

int BatchILQSPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                 int num_spline_points, int interpolation, double exploration, double timestep,
                                 const double* ctrlrange, const uint32_t* seeds, int ilqg_num_rollouts,
                                 int ilqg_representation, double fd_tolerance, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * num_trajectory, max_horizon, device)) return rc;
  if (int rc = mjpc_b200_create(model, num_problems * ilqg_num_rollouts, max_horizon, device, &ilqg_gpu_)) return rc;
  sweeps_.Attach(ilqg_gpu_, ilqg_num_rollouts, ilqg_representation);
  improved_.assign(num_problems, 0);
  for (int b = 0; b < num_problems; b++) {
    auto* p = new iLQSPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, timestep, ctrlrange,
                               seeds[b], ilqg_num_rollouts, ilqg_representation, fd_tolerance, max_horizon, device, gpu_,
                               ilqg_gpu_))
      return rc;
  }
  return 0;
}

int BatchILQSPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  std::fill(improved_.begin(), improved_.end(), 0);
  const bool diff = planner(0).ilqg.settings.differentiable != 0;
  auto ilqg_of = [&](const std::vector<int>& idx) {
    std::vector<iLQGPlanner*> ps;
    for (int b : idx) ps.push_back(&planner(b).ilqg);
    return ps;
  };
  // the iLQG nominals of the problems whose active policy was iLQG, then their conversion to splines
  std::vector<int> conv;
  for (int b = 0; b < B; b++) {
    planner(b).BeginIteration();
    if (planner(b).previous_active_policy == iLQSPlanner::kiLQG) conv.push_back(b);
  }
  if (!conv.empty()) {
    const DifferentiableScope d(ilqg_gpu_, diff);
    if (sweeps_.Nominal(ilqg_of(conv), conv, Rows(), horizon)) return -1;
  }
  for (int b : conv) planner(b).ConvertToSpline(horizon);
  // every problem's sampling: one launch
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++) cands[b] = &planner(b).sampling.PrepareOptimize(horizon);
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  const int N = cands[0]->N;
  std::vector<int> rest;
  for (int b = 0; b < B; b++) {
    iLQSPlanner& p = planner(b);
    const size_t o = (size_t)b * N;
    p.sampling.InstallRollouts(N, horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
    p.sampling.InstallBest();
    const int settled = p.SamplingSettled(horizon);
    if (settled < 0) return -1;
    if (settled) improved_[b] = 1;
    else rest.push_back(b);
  }
  // one iLQG iteration of the problems sampling did not settle
  if (rest.empty()) return 0;
  std::vector<int> updated(rest.size(), 0);
  {
    const DifferentiableScope d(ilqg_gpu_, diff);
    if (sweeps_.Iterate(ilqg_of(rest), rest, Rows(), horizon, updated.data())) return -1;
  }
  for (size_t j = 0; j < rest.size(); j++) improved_[rest[j]] = planner(rest[j]).Accept(updated[j]);
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
// (the generic batch family of include/mjpc_b200.h: every batch kind's handle is its BatchPlanner base)
using mjpc_b200_host::BatchCrossEntropyPlanner;
using mjpc_b200_host::BatchGradientPlanner;
using mjpc_b200_host::BatchILQSPlanner;
using mjpc_b200_host::BatchPlanner;
using mjpc_b200_host::BatchRobustPlanner;
using mjpc_b200_host::BatchSampleGradientPlanner;

namespace {
BatchPlanner* batch_of(void* p) { return reinterpret_cast<BatchPlanner*>(p); }
// the batch planner behind a handle if it is a T and `problem` is one of its problems, else nullptr
template <class T>
T* problem_of(void* p, int problem) {
  T* bp = dynamic_cast<T*>(batch_of(p));
  return bp && problem >= 0 && problem < bp->NumProblems() ? bp : nullptr;
}
template <class T>
int finish_create(T* p, int rc, void** out) {
  if (rc) { delete p; return rc; }
  *out = static_cast<BatchPlanner*>(p);
  return 0;
}
}  // namespace

extern "C" {

void mjpc_b200_batch_planner_destroy(void* p) { delete batch_of(p); }
int mjpc_b200_batch_planner_reset(void* p, int problem, int horizon, const double* initial_repeated_action) {
  BatchPlanner* bp = problem_of<BatchPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).Reset(horizon, initial_repeated_action);
  return 0;
}
int mjpc_b200_batch_planner_set_state(void* p, int problem, const double* state, double time, const double* mocap) {
  BatchPlanner* bp = problem_of<BatchPlanner>(p, problem);
  if (!bp || !state) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).SetState(state, time, mocap);
  return 0;
}
int mjpc_b200_batch_planner_set_task(void* p, int problem, const double* weight, const double* parameters,
                                     const double* task_state) {
  BatchPlanner* bp = problem_of<BatchPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->SetTask(problem, weight, parameters, task_state);
  return 0;
}
int mjpc_b200_batch_planner_optimize_policy(void* p, int horizon) {
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  return batch_of(p)->OptimizePolicy(horizon);
}
int mjpc_b200_batch_planner_action_from_policy(void* p, int problem, double* action, double time, int use_previous) {
  BatchPlanner* bp = problem_of<BatchPlanner>(p, problem);
  if (!bp || !action) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).ActionFromPolicy(action, nullptr, time, use_previous != 0);
  return 0;
}

int mjpc_b200_batch_ce_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory, int n_elite,
                                      int num_spline_points, int interpolation, double std_initial, double std_min,
                                      double explore_fraction, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device, void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 2 || num_spline_points < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchCrossEntropyPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, n_elite, num_spline_points, interpolation,
                                        std_initial, std_min, explore_fraction, timestep, ctrlrange, seeds, max_horizon,
                                        device), out);
}
int mjpc_b200_batch_ce_planner_get_result(void* p, int problem, double* improvement, float* returns, int* order,
                                          double* knots, double* knot_times, double* variance) {
  BatchCrossEntropyPlanner* bp = problem_of<BatchCrossEntropyPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_ce_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), improvement, returns, order,
                                         knots, knot_times, variance);
}

int mjpc_b200_batch_sg_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                      int num_gradient, int num_spline_points, int interpolation, double exploration,
                                      double gradient_filter, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device, void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 1 || num_spline_points < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchSampleGradientPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_gradient, num_spline_points,
                                        interpolation, exploration, gradient_filter, timestep, ctrlrange, seeds,
                                        max_horizon, device), out);
}
int mjpc_b200_batch_sg_planner_get_result(void* p, int problem, int* winner, int* winner_type, double* improvement,
                                          float* returns, int* order, double* knots, double* knot_times,
                                          double* gradient_knots, double* gradient) {
  BatchSampleGradientPlanner* bp = problem_of<BatchSampleGradientPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_sg_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), winner, winner_type,
                                         improvement, returns, order, knots, knot_times, gradient_knots, gradient);
}

int mjpc_b200_batch_robust_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                          int num_spline_points, int interpolation, double exploration, double timestep,
                                          const double* ctrlrange, const uint32_t* seeds, int ncandidates,
                                          int nrepetitions, double xfrc_std, double xfrc_rate, int max_horizon,
                                          int device, void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchRobustPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation,
                                        exploration, timestep, ctrlrange, seeds, ncandidates, nrepetitions, xfrc_std,
                                        xfrc_rate, max_horizon, device), out);
}
int mjpc_b200_batch_robust_planner_get_result(void* p, int problem, int* winner, double* scores, float* returns,
                                              double* knots, double* knot_times) {
  BatchRobustPlanner* bp = problem_of<BatchRobustPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_robust_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), winner, scores, returns,
                                             knots, knot_times);
}

int mjpc_b200_batch_planner_set_fd(void* p, double tolerance, int mode, int derivative_skip) {
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  BatchPlanner* bp = batch_of(p);
  for (int b = 0; b < bp->NumProblems(); b++)
    if (int rc = bp->problem(b).SetFD(tolerance, mode, derivative_skip)) return rc;   // the kinds without: UNSUPPORTED
  return 0;
}

int mjpc_b200_batch_gradient_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                            int num_spline_points, int representation, double fd_tolerance,
                                            double timestep, const double* ctrlrange, int max_horizon, int device,
                                            void** out) {
  if (!model || !model->data || !ctrlrange || !out || num_trajectory < 1 || num_spline_points < 1 || max_horizon < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchGradientPlanner;
  int rc = p->Initialize(model, num_problems, num_trajectory, num_spline_points, representation, timestep, ctrlrange,
                         max_horizon, device);
  if (rc == 0) mjpc_b200_batch_planner_set_fd(static_cast<BatchPlanner*>(p), fd_tolerance, -1, -1);
  return finish_create(p, rc, out);
}
int mjpc_b200_batch_gradient_planner_get_result(void* p, int problem, double* scalars, double* parameters,
                                                double* times, int* improved) {
  BatchGradientPlanner* bp = problem_of<BatchGradientPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (improved) *improved = bp->improved(problem);
  return mjpc_b200_gradient_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), scalars, parameters,
                                               times);
}

int mjpc_b200_batch_ilqs_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                        int num_spline_points, int interpolation, double exploration, double timestep,
                                        const double* ctrlrange, const uint32_t* seeds, int ilqg_num_rollouts,
                                        int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                                        void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 1 || ilqg_num_rollouts < 1 ||
      max_horizon < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchILQSPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation,
                                        exploration, timestep, ctrlrange, seeds, ilqg_num_rollouts, ilqg_representation,
                                        fd_tolerance, max_horizon, device), out);
}
// scalars[4] as mjpc_b200_ilqs_planner_get_result; *improved (may be NULL) = the problem's 1/0 of the last iteration
int mjpc_b200_batch_ilqs_planner_get_result(void* p, int problem, double* scalars, int* improved) {
  BatchILQSPlanner* bp = problem_of<BatchILQSPlanner>(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (improved) *improved = bp->improved(problem);
  return mjpc_b200_ilqs_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), scalars);
}
int mjpc_b200_batch_ilqs_planner_set_exploration(void* p, double exploration) {
  BatchILQSPlanner* bp = problem_of<BatchILQSPlanner>(p, 0);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  for (int b = 0; b < bp->NumProblems(); b++) bp->planner(b).sampling.SetExploration(exploration, 0.0);
  return 0;
}
int mjpc_b200_batch_ilqs_planner_action_from_policy(void* p, int problem, double* action, const double* state,
                                                    double time, int use_previous) {
  BatchILQSPlanner* bp = problem_of<BatchILQSPlanner>(p, problem);
  if (!bp || !action) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->planner(problem).ActionFromPolicy(action, state, time, use_previous != 0);
  return 0;
}

}  // extern "C"
