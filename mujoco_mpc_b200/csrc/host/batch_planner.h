// batch_planner.h - several independent planning problems of one planner kind planned together on one engine handle:
// one planner per problem (its own seed, state, mocap, task snapshot, policy and policy lock), and per iteration ONE
// mjpc_b200_rollout_spline_batched launch where each of those planners would make one.  Each planner runs exactly the
// host steps it runs around its own launch (its prepare / install halves), so each problem's result is bitwise the one
// a planner of that kind with the same seed and inputs computes with its own launches.
//   BatchSamplingPlanner       (batch_sampling_planner.h)  B x N candidates
//   BatchCrossEntropyPlanner   B x (N noisy + the nominal)
//   BatchSampleGradientPlanner B x N (nominal, noisy samples, gradient candidates)
//   BatchRobustPlanner         B x N clean, then B x ncandidates x nrepetitions with force noise keyed per problem
//   BatchGradientPlanner       per max_rollout iteration: B nominals, one mjpc_b200_gradient_batched, B x K line search
//   BatchILQSPlanner           B x N sampling; the iLQG halves as batched iLQG sweeps on a second handle of B x K
// Settings (noise, ncandidates, finite differences, ...) are common to a batch.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "batch_ilqg_planner.h"
#include "cross_entropy_planner.h"
#include "gradient_planner.h"
#include "robust_planner.h"
#include "sample_gradient_planner.h"

namespace mjpc_b200_host {

class BatchPlanner {
 public:
  virtual ~BatchPlanner();
  int NumProblems() const { return (int)problems_.size(); }
  Planner& problem(int b) { return *problems_[b]; }
  // Task::weight / parameters / task-state block of problem b; NULL members keep the current value
  void SetTask(int b, const double* weight, const double* parameters, const double* task_state);
  // Planner::OptimizePolicy of every problem
  virtual int OptimizePolicy(int horizon) = 0;

 protected:
  // the task snapshots of num_problems problems, each the model's, and the engine handle of max_candidates (all
  // problems' candidates) x max_horizon
  int Attach(const mjpc_model_blob* model, int num_problems, int max_candidates, int max_horizon, int device);
  // ONE launch on `gpu` of every problem's candidates cands[b] (common N, P and interpolation) from its state, time,
  // mocap and task snapshot; fills returns_, failure_ and order_ [B][N]
  int LaunchSpline(mjpc_b200_t* gpu, const std::vector<const SplineCandidates*>& cands, int horizon);
  // every problem's task snapshot [B][..]; NULL when the model has no such member
  const double* weights() const { return nw_ ? weight_.data() : nullptr; }
  const double* parameters() const { return np_ ? parameters_.data() : nullptr; }
  const double* task_states() const { return nts_ ? task_state_.data() : nullptr; }
  template <class T>
  T& at(int b) { return static_cast<T&>(*problems_[b]); }
  // the planner whose state, time and mocap problem b's spline candidates start from
  virtual const Planner& launcher(int b) const { return *problems_[b]; }
  TaskRows Rows() const;

  mjpc_b200_t* gpu_ = nullptr;
  std::vector<std::unique_ptr<Planner>> problems_;   // borrow gpu_
  std::vector<float> returns_;
  std::vector<uint8_t> failure_;
  std::vector<int> order_;

 private:
  std::vector<double> weight_, parameters_, task_state_;   // [B][num_term], [B][num_parameters], [B][task_state_size]
  int nw_ = 0, np_ = 0, nts_ = 0;
  // launch staging
  std::vector<float> states_, mocaps_, knots_;
  std::vector<double> times_, knot_times_;
};

class BatchCrossEntropyPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int n_elite, int num_spline_points,
                 int interpolation, double std_initial, double std_min, double explore_fraction, double timestep,
                 const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device);
  CrossEntropyPlanner& planner(int b) { return at<CrossEntropyPlanner>(b); }
  int OptimizePolicy(int horizon) override;
};

class BatchSampleGradientPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_gradient,
                 int num_spline_points, int interpolation, double exploration, double gradient_filter, double timestep,
                 const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device);
  SampleGradientPlanner& planner(int b) { return at<SampleGradientPlanner>(b); }
  int OptimizePolicy(int horizon) override;
};

// The noisy re-evaluations run on a second handle, as the single planner's do, so that every problem's clean
// trajectories survive them.
class BatchRobustPlanner : public BatchPlanner {
 public:
  ~BatchRobustPlanner() override;
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate, int max_horizon, int device);
  RobustPlanner& planner(int b) { return at<RobustPlanner>(b); }
  int OptimizePolicy(int horizon) override;

 private:
  mjpc_b200_t* noisy_gpu_ = nullptr;
  std::vector<uint32_t> seeds_;
};

// Each problem's nominal trajectory stays the problem's own; only the derivatives and the gradient recursion of all of
// them run as one device call, whose k and dV0 are bitwise the single planner's host GradientSweep.
class BatchGradientPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int representation, double timestep, const double* ctrlrange, int max_horizon, int device);
  GradientPlanner& planner(int b) { return at<GradientPlanner>(b); }
  int OptimizePolicy(int horizon) override;
  int improved(int b) const { return improved_[b]; }    // GradientPlanner::OptimizePolicy's 1/0; 0 after an error

 private:
  std::vector<int> improved_;
  std::vector<float> x_, u_, mc_, res_;                  // the nominals' trajectories [B][H][..], mocaps [B][7 nmocap]
  std::vector<double> t_, k_, dV0_;
};

// Two handles, as the single iLQS planner has: the sampling halves launch B x N on the base's handle, the iLQG halves
// run the batched iLQG sweeps (ILQGSweeps) on a handle of B x K, each over the problems that need it in that iteration.
// Settings (exploration, finite differences, iLQG settings) are common to the batch; each problem has its own seed.
class BatchILQSPlanner : public BatchPlanner {
 public:
  ~BatchILQSPlanner() override;
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int ilqg_num_rollouts, int ilqg_representation, double fd_tolerance, int max_horizon, int device);
  iLQSPlanner& planner(int b) { return at<iLQSPlanner>(b); }
  int OptimizePolicy(int horizon) override;
  int improved(int b) const { return improved_[b]; }    // iLQSPlanner::OptimizePolicy's 1/0; 0 after an error

 protected:
  const Planner& launcher(int b) const override { return static_cast<const iLQSPlanner&>(*problems_[b]).sampling; }

 private:
  mjpc_b200_t* ilqg_gpu_ = nullptr;
  ILQGSweeps sweeps_;
  std::vector<int> improved_;
};

}  // namespace mjpc_b200_host
