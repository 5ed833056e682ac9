// batch_planner.h - several independent planning problems of one planner kind planned together on one engine handle:
// one planner per problem (its own seed, state, mocap, task snapshot, policy and policy lock), and per iteration the
// kind's own iteration (XPlanner::Iterate, which a single planner runs over itself alone) over all the problems, with
// each problem's task snapshot row.  Each problem's result is therefore bitwise the one a planner of that kind with the
// same seed and inputs computes on its own.
//   BatchSamplingPlanner       B x N candidates
//   BatchCrossEntropyPlanner   B x (N noisy + the nominal)
//   BatchSampleGradientPlanner B x N (nominal, noisy samples, gradient candidates)
//   BatchRobustPlanner         B x N clean, then B x ncandidates x nrepetitions with force noise keyed per problem
//   BatchGradientPlanner       per max_rollout iteration: B nominals, one mjpc_b200_gradient_batched, B x K line search
//   BatchILQSPlanner           B x N sampling; the iLQG halves as batched iLQG sweeps on a second handle of B x K
//   BatchILQGPlanner           the iLQG sweeps (ILQGSweeps) of all B problems, B x K rollouts per feedback launch
// Settings (noise, ncandidates, finite differences, ...) are common to a batch.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "cross_entropy_planner.h"
#include "gradient_planner.h"
#include "ilqg_planner.h"
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
  // Planner::OptimizePolicy of every problem; codes()[b] is then what problem b's returned when it succeeded (the
  // Gradient, iLQG and iLQS 1/0, 0 for the other kinds)
  virtual int OptimizePolicy(int horizon) = 0;
  const std::vector<int>& codes() const { return codes_; }
  // problem b plans on models[b] from now on (mjpc_b200_set_model_variants on every handle the batch owns); count is
  // the number of problems, or 0 to plan every problem on the batch's model again
  int SetModels(const mjpc_model_blob* models, int count);
  // every problem plans on one model ensemble: Planner::SetEnsemble of the problems, which share the batch's handle
  int SetEnsemble(const mjpc_model_blob* models, int K, int worst) { return problem(0).SetEnsemble(models, K, worst); }
  // every problem plans over its own state covariance with the same K, worst and seed (Planner::SetStateEnsemble of
  // each problem; problem 0 first, so a refusal changes nothing); the launch draws problem b with key seed + b
  int SetStateEnsemble(int K, int worst, uint32_t seed);
  int SetStateCovariance(int b, const double* covariance) { return problem(b).SetStateCovariance(covariance); }

 protected:
  // the task snapshots of num_problems problems, each the model's, and the engine handle of max_candidates (all
  // problems' candidates) x max_horizon
  int Attach(const mjpc_model_blob* model, int num_problems, int max_candidates, int max_horizon, int device);
  TaskRows Rows() const;   // every problem's task snapshot, row b problem b's
  template <class T>
  T& at(int b) { return static_cast<T&>(*problems_[b]); }
  template <class T>
  std::vector<T*> all() {
    std::vector<T*> ps;
    for (auto& p : problems_) ps.push_back(static_cast<T*>(p.get()));
    return ps;
  }

  // every engine handle the batch owns: gpu_, and the second handle of the Robust and iLQS batches
  virtual std::vector<mjpc_b200_t*> Handles() const { return {gpu_}; }

  mjpc_b200_t* gpu_ = nullptr;
  std::vector<std::unique_ptr<Planner>> problems_;   // borrow gpu_
  SplineLaunch launch_;
  std::vector<int> codes_;                            // [B], all 0 until a kind's OptimizePolicy fills it

 private:
  std::vector<double> weight_, parameters_, task_state_;   // [B][num_term], [B][num_parameters], [B][task_state_size]
  int nw_ = 0, np_ = 0, nts_ = 0;
};

class BatchSamplingPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int max_horizon, int device);
  SamplingPlanner& planner(int b) { return at<SamplingPlanner>(b); }
  int OptimizePolicy(int horizon) override;
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
  std::vector<mjpc_b200_t*> Handles() const override { return {gpu_, noisy_gpu_}; }
  mjpc_b200_t* noisy_gpu_ = nullptr;
};

class BatchGradientPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int representation, double timestep, const double* ctrlrange, int max_horizon, int device);
  GradientPlanner& planner(int b) { return at<GradientPlanner>(b); }
  int OptimizePolicy(int horizon) override;
};

// Two handles, as the single iLQS planner has: the sampling halves launch B x N on the base's handle, the iLQG halves
// run the iLQG sweeps on a handle of B x K, each over the problems that need it in that iteration.  Each problem has
// its own seed.
class BatchILQSPlanner : public BatchPlanner {
 public:
  ~BatchILQSPlanner() override;
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int ilqg_num_rollouts, int ilqg_representation, double fd_tolerance, int max_horizon, int device);
  iLQSPlanner& planner(int b) { return at<iLQSPlanner>(b); }
  int OptimizePolicy(int horizon) override;

 private:
  std::vector<mjpc_b200_t*> Handles() const override { return {gpu_, ilqg_gpu_}; }
  mjpc_b200_t* ilqg_gpu_ = nullptr;
  ILQGSweeps sweeps_;
};

class BatchILQGPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_rollouts, int representation, int max_horizon,
                 int device);
  iLQGPlanner& planner(int b) { return at<iLQGPlanner>(b); }
  // iLQGPlanner::NominalTrajectory of every problem in one launch; <0 on error
  int NominalTrajectory(int horizon);
  int OptimizePolicy(int horizon) override;

 private:
  ILQGSweeps sweeps_;
  std::vector<int> problem_rows_;   // 0 .. B-1: problem b reads task row b
};

}  // namespace mjpc_b200_host
