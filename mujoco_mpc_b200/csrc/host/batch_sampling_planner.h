// batch_sampling_planner.h - several independent Predictive Sampling problems planned together (batch_planner.h): one
// SamplingPlanner per problem and per iteration ONE mjpc_b200_rollout_spline_batched launch for the candidates of all
// problems.  Each problem's result is bitwise the one a SamplingPlanner with the same seed and inputs computes with its
// own launches.
#pragma once
#include <cstdint>

#include "batch_planner.h"

namespace mjpc_b200_host {

class BatchSamplingPlanner : public BatchPlanner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                 int interpolation, double exploration, double timestep, const double* ctrlrange, const uint32_t* seeds,
                 int max_horizon, int device);
  SamplingPlanner& planner(int b) { return at<SamplingPlanner>(b); }
  // SamplingPlanner::OptimizePolicy of every problem, with the rollouts of all of them in one launch
  int OptimizePolicy(int horizon) override;
};

}  // namespace mjpc_b200_host
