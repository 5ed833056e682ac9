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
  codes_.assign(num_problems, 0);
  std::vector<double> w(weight_), p(parameters_), s(task_state_);
  for (int b = 1; b < num_problems; b++) {
    weight_.insert(weight_.end(), w.begin(), w.end());
    parameters_.insert(parameters_.end(), p.begin(), p.end());
    task_state_.insert(task_state_.end(), s.begin(), s.end());
  }
  return mjpc_b200_create(model, max_candidates, max_horizon, device, &gpu_);
}

void BatchPlanner::SetTask(int b, const double* weight, const double* parameters, const double* task_state) {
  if (weight) std::copy(weight, weight + nw_, weight_.begin() + (size_t)b * nw_);
  if (parameters) std::copy(parameters, parameters + np_, parameters_.begin() + (size_t)b * np_);
  if (task_state) std::copy(task_state, task_state + nts_, task_state_.begin() + (size_t)b * nts_);
}

int BatchPlanner::SetModels(const mjpc_model_blob* models, int count) {
  if (count != 0 && count != NumProblems())
    return MJPC_B200_ERR_BAD_ARGUMENT;
  // the handles were created from one model, so a variant the rule refuses is refused by the first, before any
  // handle changed
  for (mjpc_b200_t* h : Handles())
    if (int rc = mjpc_b200_set_model_variants(h, models, count)) return rc;
  return 0;
}

int BatchPlanner::SetStateEnsemble(int K, int worst, uint32_t seed) {
  for (int b = 0; b < NumProblems(); b++)
    if (int rc = problem(b).SetStateEnsemble(K, worst, seed)) return rc;
  return 0;
}

TaskRows BatchPlanner::Rows() const {
  TaskRows r;
  r.w = weight_.data(); r.p = parameters_.data(); r.ts = task_state_.data(); r.nw = nw_; r.np = np_; r.nts = nts_;
  return r;
}

// ------------------------------------------------------------------------------------------ Predictive Sampling
int BatchSamplingPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                     int num_spline_points, int interpolation, double exploration, double timestep,
                                     const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device) {
  if (num_problems < 1 || num_trajectory < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * num_trajectory, max_horizon, device)) return rc;
  for (int b = 0; b < num_problems; b++) {
    auto* p = new SamplingPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep,
                               ctrlrange, seeds[b], num_trajectory, max_horizon, device, gpu_))
      return rc;
  }
  return 0;
}

int BatchSamplingPlanner::OptimizePolicy(int horizon) {
  return SamplingPlanner::Iterate(all<SamplingPlanner>(), Rows(), horizon, &launch_);
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
  return CrossEntropyPlanner::Iterate(all<CrossEntropyPlanner>(), Rows(), horizon, &launch_);
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
  return SampleGradientPlanner::Iterate(all<SampleGradientPlanner>(), Rows(), horizon, &launch_);
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
  return RobustPlanner::Iterate(all<RobustPlanner>(), Rows(), horizon, &launch_);
}

// ------------------------------------------------------------------------------------------ Gradient
int BatchGradientPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                     int num_spline_points, int representation, double timestep,
                                     const double* ctrlrange, int max_horizon, int device) {
  if (num_problems < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * std::max(num_trajectory, 1), max_horizon, device)) return rc;
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
  return GradientPlanner::Iterate(all<GradientPlanner>(), Rows(), horizon, &launch_, codes_.data());
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
  return iLQSPlanner::Iterate(all<iLQSPlanner>(), Rows(), horizon, &launch_, &sweeps_, codes_.data());
}

// ------------------------------------------------------------------------------------------ iLQG
int BatchILQGPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_rollouts, int representation,
                                 int max_horizon, int device) {
  if (num_problems < 1 || num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * num_rollouts, max_horizon, device)) return rc;
  for (int b = 0; b < num_problems; b++) {
    auto* p = new iLQGPlanner;
    problems_.emplace_back(p);
    problem_rows_.push_back(b);
    if (int rc = p->Initialize(model, num_rollouts, representation, max_horizon, device, gpu_)) return rc;
  }
  return 0;
}

int BatchILQGPlanner::NominalTrajectory(int horizon) {
  const DifferentiableScope diff(gpu_, planner(0).settings.differentiable != 0);
  return sweeps_.Nominal(all<iLQGPlanner>(), problem_rows_, Rows(), horizon, nullptr);
}

int BatchILQGPlanner::OptimizePolicy(int horizon) {
  std::fill(codes_.begin(), codes_.end(), 0);
  const DifferentiableScope diff(gpu_, planner(0).settings.differentiable != 0);
  const std::vector<iLQGPlanner*> ps = all<iLQGPlanner>();
  if (sweeps_.Nominal(ps, problem_rows_, Rows(), horizon, nullptr)) return -1;
  return sweeps_.Iterate(ps, problem_rows_, Rows(), horizon, codes_.data());
}

}  // namespace mjpc_b200_host


// ------------------------------------------------------------------------------------------ C entry points
// (the batch family of include/mjpc_b200.h: every batch kind's handle is its BatchPlanner base)
using mjpc_b200_host::BatchCrossEntropyPlanner;
using mjpc_b200_host::BatchGradientPlanner;
using mjpc_b200_host::BatchILQGPlanner;
using mjpc_b200_host::BatchILQSPlanner;
using mjpc_b200_host::BatchPlanner;
using mjpc_b200_host::BatchRobustPlanner;
using mjpc_b200_host::BatchSampleGradientPlanner;
using mjpc_b200_host::BatchSamplingPlanner;
using mjpc_b200_host::ToHandle;

namespace {
mjpc_b200_batch_planner_t* batch_handle(BatchPlanner* p) { return reinterpret_cast<mjpc_b200_batch_planner_t*>(p); }
// the batch planner behind a handle if it is a T and `problem` is one of its problems, else nullptr
template <class T>
T* problem_of(mjpc_b200_batch_planner_t* h, int problem) {
  T* bp = dynamic_cast<T*>(reinterpret_cast<BatchPlanner*>(h));
  return bp && problem >= 0 && problem < bp->NumProblems() ? bp : nullptr;
}
template <class T>
int finish_create(T* p, int rc, mjpc_b200_batch_planner_t** out) {
  if (rc) { delete p; return rc; }
  *out = batch_handle(p);
  return 0;
}
}  // namespace

extern "C" {

void mjpc_b200_batch_planner_destroy(mjpc_b200_batch_planner_t* h) { delete reinterpret_cast<BatchPlanner*>(h); }
int mjpc_b200_batch_planner_reset(mjpc_b200_batch_planner_t* h, int problem, int horizon,
                                  const double* initial_repeated_action) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).Reset(horizon, initial_repeated_action);
  return 0;
}
int mjpc_b200_batch_planner_set_state(mjpc_b200_batch_planner_t* h, int problem, const double* state, double time,
                                      const double* mocap) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, problem);
  if (!bp || !state) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).SetState(state, time, mocap);
  return 0;
}
int mjpc_b200_batch_planner_set_task(mjpc_b200_batch_planner_t* h, int problem, const double* weight,
                                     const double* parameters, const double* task_state) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->SetTask(problem, weight, parameters, task_state);
  return 0;
}
int mjpc_b200_batch_planner_set_models(mjpc_b200_batch_planner_t* h, const mjpc_model_blob* models, int count) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, 0);
  if (!bp || count < 0) return MJPC_B200_ERR_BAD_ARGUMENT;
  return bp->SetModels(models, count);
}
int mjpc_b200_batch_planner_set_ensemble(mjpc_b200_batch_planner_t* h, const mjpc_model_blob* models, int K,
                                         int worst) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, 0);
  return bp ? bp->SetEnsemble(models, K, worst) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_batch_planner_set_state_ensemble(mjpc_b200_batch_planner_t* h, int K, int worst, uint32_t seed) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, 0);
  return bp ? bp->SetStateEnsemble(K, worst, seed) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_batch_planner_set_state_covariance(mjpc_b200_batch_planner_t* h, int problem, const double* covariance) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, problem);
  return bp ? bp->SetStateCovariance(problem, covariance) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_batch_planner_optimize_policy(mjpc_b200_batch_planner_t* h, int horizon, int* codes) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, 0);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  const int rc = bp->OptimizePolicy(horizon);
  for (int b = 0; codes && b < bp->NumProblems(); b++) codes[b] = rc < 0 ? 0 : bp->codes()[b];
  return rc;
}
int mjpc_b200_batch_planner_action_from_policy(mjpc_b200_batch_planner_t* h, int problem, double* action,
                                               const double* state, double time, int use_previous) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, problem);
  if (!bp || !action) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).ActionFromPolicy(action, state, time, use_previous != 0);
  return 0;
}
int mjpc_b200_batch_planner_set_fd(mjpc_b200_batch_planner_t* h, double tolerance, int mode, int derivative_skip) {
  BatchPlanner* bp = problem_of<BatchPlanner>(h, 0);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  for (int b = 0; b < bp->NumProblems(); b++)
    if (int rc = bp->problem(b).SetFD(tolerance, mode, derivative_skip)) return rc;   // the kinds without: UNSUPPORTED
  return 0;
}

int mjpc_b200_batch_sampling_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                            int num_spline_points, int interpolation, double exploration,
                                            double timestep, const double* ctrlrange, const uint32_t* seeds,
                                            int max_horizon, int device, mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchSamplingPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation,
                                        exploration, timestep, ctrlrange, seeds, max_horizon, device), out);
}
int mjpc_b200_batch_sampling_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, int* winner,
                                                double* improvement, float* returns, double* knots,
                                                double* knot_times) {
  BatchSamplingPlanner* bp = problem_of<BatchSamplingPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_sampling_planner_get_result(ToHandle(&bp->planner(problem)), winner, improvement, returns, knots,
                                               knot_times);
}

int mjpc_b200_batch_ce_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory, int n_elite,
                                      int num_spline_points, int interpolation, double std_initial, double std_min,
                                      double explore_fraction, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device,
                                      mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 2 || num_spline_points < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchCrossEntropyPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, n_elite, num_spline_points, interpolation,
                                        std_initial, std_min, explore_fraction, timestep, ctrlrange, seeds, max_horizon,
                                        device), out);
}
int mjpc_b200_batch_ce_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, double* improvement,
                                          float* returns, int* order, double* knots, double* knot_times,
                                          double* variance) {
  BatchCrossEntropyPlanner* bp = problem_of<BatchCrossEntropyPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_ce_planner_get_result(ToHandle(&bp->planner(problem)), improvement, returns, order, knots,
                                         knot_times, variance);
}

int mjpc_b200_batch_sg_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                      int num_gradient, int num_spline_points, int interpolation, double exploration,
                                      double gradient_filter, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device,
                                      mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 1 || num_spline_points < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchSampleGradientPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_gradient, num_spline_points,
                                        interpolation, exploration, gradient_filter, timestep, ctrlrange, seeds,
                                        max_horizon, device), out);
}
int mjpc_b200_batch_sg_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, int* winner, int* winner_type,
                                          double* improvement, float* returns, int* order, double* knots,
                                          double* knot_times, double* gradient_knots, double* gradient) {
  BatchSampleGradientPlanner* bp = problem_of<BatchSampleGradientPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_sg_planner_get_result(ToHandle(&bp->planner(problem)), winner, winner_type, improvement, returns,
                                         order, knots, knot_times, gradient_knots, gradient);
}

int mjpc_b200_batch_robust_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                          int num_spline_points, int interpolation, double exploration, double timestep,
                                          const double* ctrlrange, const uint32_t* seeds, int ncandidates,
                                          int nrepetitions, double xfrc_std, double xfrc_rate, int max_horizon,
                                          int device, mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchRobustPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation,
                                        exploration, timestep, ctrlrange, seeds, ncandidates, nrepetitions, xfrc_std,
                                        xfrc_rate, max_horizon, device), out);
}
int mjpc_b200_batch_robust_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, int* winner, double* scores,
                                              float* returns, double* knots, double* knot_times) {
  BatchRobustPlanner* bp = problem_of<BatchRobustPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_robust_planner_get_result(ToHandle(&bp->planner(problem)), winner, scores, returns, knots,
                                             knot_times);
}

int mjpc_b200_batch_gradient_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                            int num_spline_points, int representation, double fd_tolerance,
                                            double timestep, const double* ctrlrange, int max_horizon, int device,
                                            mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !out || num_trajectory < 1 || num_spline_points < 1 || max_horizon < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchGradientPlanner;
  int rc = p->Initialize(model, num_problems, num_trajectory, num_spline_points, representation, timestep, ctrlrange,
                         max_horizon, device);
  if (rc == 0) mjpc_b200_batch_planner_set_fd(batch_handle(p), fd_tolerance, -1, -1);
  return finish_create(p, rc, out);
}
int mjpc_b200_batch_gradient_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, double* scalars,
                                                double* parameters, double* times) {
  BatchGradientPlanner* bp = problem_of<BatchGradientPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_gradient_planner_get_result(ToHandle(&bp->planner(problem)), scalars, parameters, times);
}

int mjpc_b200_batch_ilqs_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                        int num_spline_points, int interpolation, double exploration, double timestep,
                                        const double* ctrlrange, const uint32_t* seeds, int ilqg_num_rollouts,
                                        int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                                        mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out || num_trajectory < 1 || ilqg_num_rollouts < 1 ||
      max_horizon < 2)
    return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchILQSPlanner;
  return finish_create(p, p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation,
                                        exploration, timestep, ctrlrange, seeds, ilqg_num_rollouts, ilqg_representation,
                                        fd_tolerance, max_horizon, device), out);
}
int mjpc_b200_batch_ilqs_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, double* scalars) {
  BatchILQSPlanner* bp = problem_of<BatchILQSPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_ilqs_planner_get_result(ToHandle(&bp->planner(problem)), scalars);
}
int mjpc_b200_batch_ilqs_planner_set_exploration(mjpc_b200_batch_planner_t* h, double exploration) {
  BatchILQSPlanner* bp = problem_of<BatchILQSPlanner>(h, 0);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  for (int b = 0; b < bp->NumProblems(); b++) bp->planner(b).sampling.SetExploration(exploration, 0.0);
  return 0;
}

int mjpc_b200_batch_ilqg_planner_create(const mjpc_model_blob* model, int num_problems, int num_rollouts,
                                        int representation, double fd_tolerance, int max_horizon, int device,
                                        mjpc_b200_batch_planner_t** out) {
  if (!model || !model->data || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchILQGPlanner;
  int rc = p->Initialize(model, num_problems, num_rollouts, representation, max_horizon, device);
  if (rc == 0) mjpc_b200_batch_planner_set_fd(batch_handle(p), fd_tolerance, -1, -1);
  return finish_create(p, rc, out);
}
int mjpc_b200_batch_ilqg_planner_get_result(mjpc_b200_batch_planner_t* h, int problem, double* scalars, float* states,
                                            float* actions, double* times) {
  BatchILQGPlanner* bp = problem_of<BatchILQGPlanner>(h, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_ilqg_planner_get_result(ToHandle(&bp->planner(problem)), scalars, states, actions, times);
}
int mjpc_b200_batch_ilqg_planner_nominal_trajectory(mjpc_b200_batch_planner_t* h, int horizon) {
  BatchILQGPlanner* bp = problem_of<BatchILQGPlanner>(h, 0);
  return bp ? bp->NominalTrajectory(horizon) : MJPC_B200_ERR_BAD_ARGUMENT;
}

}  // extern "C"
