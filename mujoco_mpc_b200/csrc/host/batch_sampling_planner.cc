// batch_sampling_planner.cc - see batch_sampling_planner.h.  Compiled into libmjpc_b200.so next to the engine.
#include "batch_sampling_planner.h"

#include <algorithm>
#include <exception>

#include "../dev_model.h"   // Blob reader (plain C++)

namespace mjpc_b200_host {

BatchSamplingPlanner::~BatchSamplingPlanner() {
  problems_.clear();   // the planners borrow the handle
  if (gpu_) mjpc_b200_destroy(gpu_);
}

int BatchSamplingPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                     int num_spline_points, int interpolation, double exploration, double timestep,
                                     const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device) {
  if (num_problems < 1 || num_trajectory < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  // every problem's task snapshot starts as the model's
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
  if (int rc = mjpc_b200_create(model, num_problems * num_trajectory, max_horizon, device, &gpu_)) return rc;
  mjpc_b200_info info;
  mjpc_b200_get_info(gpu_, &info);
  nu_ = info.nu;
  num_trajectory_ = num_trajectory;
  for (int b = 0; b < num_problems; b++) {
    problems_.emplace_back(new SamplingPlanner);
    if (int rc = problems_.back()->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0,
                                              timestep, ctrlrange, seeds[b], num_trajectory, max_horizon, device, gpu_))
      return rc;
  }
  states_.resize((size_t)num_problems * info.dim_state);
  mocaps_.resize((size_t)num_problems * 7 * info.nmocap);
  times_.resize(num_problems);
  returns_.resize((size_t)num_problems * num_trajectory);
  failure_.resize(returns_.size());
  order_.resize(returns_.size());
  return 0;
}

void BatchSamplingPlanner::SetTask(int b, const double* weight, const double* parameters, const double* task_state) {
  if (weight) std::copy(weight, weight + nw_, weight_.begin() + (size_t)b * nw_);
  if (parameters) std::copy(parameters, parameters + np_, parameters_.begin() + (size_t)b * np_);
  if (task_state) std::copy(task_state, task_state + nts_, task_state_.begin() + (size_t)b * nts_);
}

int BatchSamplingPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems(), N = num_trajectory_;
  int P = 0;
  // per problem, as SamplingPlanner::OptimizePolicyCandidates up to its launch
  for (int b = 0; b < B; b++) {
    SamplingPlanner& pl = *problems_[b];
    pl.UpdateNominalPolicy(horizon);
    pl.policy.plan.SetInterpolation(pl.interpolation());
    const int Pb = pl.policy.plan.Size();
    if (b == 0) {
      P = Pb;
      knots_.resize((size_t)B * N * P * nu_);
      knot_times_.resize((size_t)B * P);
    } else if (Pb != P) {
      return MJPC_B200_ERR_BAD_ARGUMENT;
    }
    pl.PrepareCandidates(N, knots_.data() + (size_t)b * N * P * nu_, knot_times_.data() + (size_t)b * P);
    const size_t ds = pl.state().size(), nm = pl.mocap().size();
    std::copy(pl.state().begin(), pl.state().end(), states_.begin() + b * ds);
    std::copy(pl.mocap().begin(), pl.mocap().end(), mocaps_.begin() + b * nm);
    times_[b] = pl.time();
  }
  if (int rc = mjpc_b200_rollout_spline_batched(gpu_, B, states_.data(), times_.data(), mocaps_.empty() ? nullptr : mocaps_.data(),
                                                nw_ ? weight_.data() : nullptr, np_ ? parameters_.data() : nullptr,
                                                nts_ ? task_state_.data() : nullptr, knots_.data(), knot_times_.data(),
                                                (int)problems_[0]->interpolation(), P, N, horizon, returns_.data(),
                                                failure_.data(), order_.data()))
    return rc;
  // per problem, as SamplingPlanner::OptimizePolicy after its launch
  for (int b = 0; b < B; b++) {
    const size_t o = (size_t)b * N;
    problems_[b]->InstallRollouts(N, horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
    problems_[b]->InstallBest();
  }
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::BatchSamplingPlanner;

namespace {
BatchSamplingPlanner* problem_of(void* p, int problem) {
  auto* bp = (BatchSamplingPlanner*)p;
  return bp && problem >= 0 && problem < bp->NumProblems() ? bp : nullptr;
}
}  // namespace

extern "C" {

int mjpc_b200_batch_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                                   int interpolation, double exploration, double timestep, const double* ctrlrange,
                                   const uint32_t* seeds, int max_horizon, int device, void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchSamplingPlanner;
  int rc = p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation, exploration, timestep,
                         ctrlrange, seeds, max_horizon, device);
  if (rc) { delete p; return rc; }
  *out = p;
  return 0;
}
void mjpc_b200_batch_planner_destroy(void* p) { delete (BatchSamplingPlanner*)p; }
int mjpc_b200_batch_planner_reset(void* p, int problem, int horizon, const double* initial_repeated_action) {
  BatchSamplingPlanner* bp = problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).Reset(horizon, initial_repeated_action);
  return 0;
}
int mjpc_b200_batch_planner_set_state(void* p, int problem, const double* state, double time, const double* mocap) {
  BatchSamplingPlanner* bp = problem_of(p, problem);
  if (!bp || !state) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).SetState(state, time, mocap);
  return 0;
}
int mjpc_b200_batch_planner_set_task(void* p, int problem, const double* weight, const double* parameters,
                                     const double* task_state) {
  BatchSamplingPlanner* bp = problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->SetTask(problem, weight, parameters, task_state);
  return 0;
}
int mjpc_b200_batch_planner_optimize_policy(void* p, int horizon) {
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  return ((BatchSamplingPlanner*)p)->OptimizePolicy(horizon);
}
int mjpc_b200_batch_planner_action_from_policy(void* p, int problem, double* action, double time, int use_previous) {
  BatchSamplingPlanner* bp = problem_of(p, problem);
  if (!bp || !action) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).ActionFromPolicy(action, nullptr, time, use_previous != 0);
  return 0;
}
int mjpc_b200_batch_planner_get_result(void* p, int problem, int* winner, double* improvement, float* returns,
                                       double* knots, double* knot_times) {
  BatchSamplingPlanner* bp = problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_sampling_planner_get_result(mjpc_b200_host::ToHandle(&bp->problem(problem)), winner, improvement,
                                               returns, knots, knot_times);
}

}  // extern "C"
