// batch_sampling_planner.h - several independent Predictive Sampling problems planned together: one engine handle,
// one SamplingPlanner per problem (its own seed, state, mocap, task snapshot and policy lock), and per iteration ONE
// mjpc_b200_rollout_spline_batched launch for the candidates of all problems.  Each problem's result is bitwise the
// one a SamplingPlanner with the same seed and inputs computes with its own launches.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "sampling_planner.h"

namespace mjpc_b200_host {

class BatchSamplingPlanner {
 public:
  ~BatchSamplingPlanner();
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int max_horizon, int device);
  int NumProblems() const { return (int)problems_.size(); }
  SamplingPlanner& problem(int b) { return *problems_[b]; }
  // Task::weight / parameters / task-state block of problem b; NULL members keep the current value
  void SetTask(int b, const double* weight, const double* parameters, const double* task_state);
  // SamplingPlanner::OptimizePolicy of every problem, with the rollouts of all of them in one launch
  int OptimizePolicy(int horizon);

 private:
  mjpc_b200_t* gpu_ = nullptr;
  std::vector<std::unique_ptr<SamplingPlanner>> problems_;
  int num_trajectory_ = 0, nu_ = 0;
  std::vector<double> weight_, parameters_, task_state_;   // [B][num_term], [B][num_parameters], [B][task_state_size]
  int nw_ = 0, np_ = 0, nts_ = 0;
  // launch staging
  std::vector<float> states_, mocaps_, knots_, returns_;
  std::vector<double> times_, knot_times_;
  std::vector<uint8_t> failure_;
  std::vector<int> order_;
};

}  // namespace mjpc_b200_host
