// cross_entropy_planner.h - C++ host side of the Cross-Entropy Method planner with the reference's method names
// (mjpc/planners/cross_entropy/planner.h:35-146, planner.cc:38-470).  Same rollout engine call as the sampling
// planner: Rollouts() makes ONE mjpc_b200_rollout_spline call over N noisy candidates + the un-noised nominal
// (candidate N) where the reference schedules N+1 closures on its ThreadPool (planner.cc:414-459).
// Noise comes from the injected Philox stream (sampling_planner.h), counter (iteration, candidate, knot, dof).
#pragma once
#include "sampling_planner.h"

namespace mjpc_b200_host {

class CrossEntropyPlanner : public Planner {
 public:
  // settings the reference reads from <custom> numerics (planner.cc:55-71): sampling_exploration (initial std),
  // std_min, explore_fraction, sampling_trajectories, n_elite (default max(N/10, 2))
  int Initialize(const mjpc_model_blob* model, int num_trajectory, int n_elite, int num_spline_points, int interpolation,
                 double std_initial, double std_min, double explore_fraction, double timestep, const double* ctrlrange,
                 uint32_t seed, int max_horizon, int device);
  void Reset(int horizon, const double* initial_repeated_action) override;   // :121-150 (variance = std_initial^2)
  int OptimizePolicy(int horizon) override;           // :153-292
  int NominalTrajectory(int) override { return 0; }   // not restated: planning disabled leaves the plan as it is
  void ResamplePolicy(int horizon);                   // :343-371
  void AddNoiseToPolicy(int i, double std_min);       // :374-411
  int Rollouts(int num_trajectory, int horizon);      // :414-459
  // :331-340; the policy does not depend on the state
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  const Trajectory* BestTrajectory() override;        // the NOMINAL trajectory (:462-464)

  SamplingPolicy policy, resampled_policy, previous_policy;
  std::vector<SamplingPolicy> candidate_policy;
  std::vector<int> trajectory_order;
  std::vector<double> variance;                       // [P * nu]
  double improvement = 0;
  int iteration = 0;
  int n_elite() const { return n_elite_; }
  const std::vector<float>& returns() const { return returns_; }

 private:
  int num_trajectory_ = 0, n_elite_ = 2, nu_ = 0;
  SplineInterpolation interpolation_ = kCubicSpline;
  double std_initial_ = 0.1, std_min_ = 0.01, explore_fraction_ = 0.0, timestep_ = 0.01;
  uint32_t seed_ = 0x5EED;
  std::vector<double> times_scratch_;
  std::vector<float> knots_, returns_;
  std::vector<uint8_t> failure_;
  std::vector<int> order_all_;
  Trajectory nominal_;
  mutable std::shared_mutex mtx_;
};

}  // namespace mjpc_b200_host
