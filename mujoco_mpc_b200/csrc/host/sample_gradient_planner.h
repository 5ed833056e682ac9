// sample_gradient_planner.h - C++ host side of the Sample Gradient planner with the reference's method names
// (mjpc/planners/sample_gradient/planner.h, planner.cc:43-498).  Rollouts is ONE spline launch
// over all N candidates where the reference schedules N closures on its ThreadPool (planner.cc:358-398):
//   0             the resampled nominal
//   1 .. N-G-1    noisy samples, knot += exploration * z, z from the injected Philox stream (sampling_planner.h),
//                 counter (iteration, candidate, knot, dof); NOT scaled by the control range (planner.cc:346-350)
//   N-G .. N-1    gradient candidates, computed at the end of the previous iteration (GradientCandidates) and
//                 resampled onto this iteration's knot times
// After resampling every candidate has the same knot times, so the launch's single interpolation id fits all of them.
// The gradient arithmetic (about N * P * nu flops) stays on the host in double, as in the reference.
#pragma once
#include "sampling_planner.h"

namespace mjpc_b200_host {

class SampleGradientPlanner : public Planner {
 public:
  enum WinnerType : int { kNominal = 0, kPerturb = 1, kGradient = 2 };
  static constexpr double gradient_max_step_size = 2.0;    // planner.h
  static constexpr double gradient_min_step_size = 1.0e-3;

  // settings the reference reads from <custom> numerics (planner.cc:57-69): sampling_trajectories (N),
  // sampling_exploration, sampling_representation, sample_gradient_trajectories (G), sample_gradient_filter
  int Initialize(const mjpc_model_blob* model, int num_trajectory, int num_gradient, int num_spline_points,
                 int interpolation, double exploration, double gradient_filter, double timestep,
                 const double* ctrlrange, uint32_t seed, int max_horizon, int device, mjpc_b200_t* engine = nullptr);
  void Reset(int horizon, const double* initial_repeated_action) override;   // :121-160
  int OptimizePolicy(int horizon) override;                         // :169-273: Iterate over this planner alone
  // OptimizePolicy of every planner of ps, which plan on one handle: the two halves below around ONE launch of all
  // their candidates; problem b reads task row b of `rows`.  0, or the launch's error code
  static int Iterate(const std::vector<SampleGradientPlanner*>& ps, const TaskRows& rows, int horizon,
                     SplineLaunch* launch);
  // ... before the launch: the resampled nominal, the noisy samples and the resampled gradient candidates (N in all)
  const SplineCandidates& PrepareCandidates(int horizon);
  // ... after it: the launch's horizon, the returns, failure flags and ranking of these N candidates, which it held from
  // flat index `offset` on; the winner, the installed policy, improvement and GradientCandidates
  void InstallRollouts(int horizon, const float* returns, const uint8_t* failure, const int* order, int offset);
  int NominalTrajectory(int horizon) override;                      // :276-287
  // :290-299; the policy does not depend on the state
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  void ResamplePolicy(SamplingPolicy& p, int horizon, int num_spline_points);     // :302-326
  void AddNoiseToPolicy(int i);                                     // :329-355
  void GradientCandidates(int num_trajectory, int num_gradient);    // :401-493
  const Trajectory* BestTrajectory() override;                      // trajectory[winner] (:496-498)
  int SetEnsemble(const mjpc_model_blob* models, int K, int worst) override { return ModelEnsemble(models, K, worst); }
  int SetStateEnsemble(int K, int worst, uint32_t seed) override { return StateEnsemble(K, worst, seed); }
  int SetStateCovariance(const double* covariance) override { return StateCovariance(covariance); }
  uint32_t PlanIteration() const override { return (uint32_t)iteration; }

  SamplingPolicy policy, resampled_policy, previous_policy;
  std::vector<SamplingPolicy> candidate_policy;
  std::vector<int> trajectory_order;
  std::vector<double> noise;                          // [N][P * nu]; slot 0 and the gradient slots stay 0
  std::vector<double> gradient, gradient_previous;    // [P * nu]
  int winner = 0, winner_type = kNominal, iteration = 0;
  double improvement = 0;
  int num_trajectory() const { return num_trajectory_; }
  int num_gradient() const { return num_gradient_; }
  const std::vector<float>& returns() const { return returns_; }

 private:
  int num_trajectory_ = 10, num_gradient_ = 0, nu_ = 0;
  SplineInterpolation interpolation_ = kCubicSpline;
  double noise_exploration_ = 0.1, gradient_filter_ = 1.0, timestep_ = 0.01;
  uint32_t seed_ = 0x5EED;
  std::vector<double> knot_times_;
  std::vector<double> return_weight_, step_size_;   // cached on size, as in the reference; Reset keeps them
  SplineCandidates cands_;                            // of the last launch: the iteration's, or the nominal alone
  std::vector<float> returns_;
  std::vector<uint8_t> failure_;
  Trajectory best_;
  mutable std::shared_mutex mtx_;
};

}  // namespace mjpc_b200_host
