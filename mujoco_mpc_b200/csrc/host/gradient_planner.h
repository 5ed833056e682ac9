// gradient_planner.h - Gradient-descent planner and iLQS planner above the C ABI, with the reference's method names
// (mjpc/planners/gradient/planner.h:39-168, planner.cc:159-383; gradient.cc:44-107; spline_mapping.cc;
//  mjpc/planners/ilqs/planner.h:37-117, planner.cc:60-260).
//
// Every sweep is one call of the ABI: NominalTrajectory / Rollouts -> mjpc_b200_rollout_spline (GradientPolicy::Action
// = FindInterval + Zero/Linear/CubicInterpolation + Clamp, gradient/policy.cc:80-103, which for >= 3 spline points is the
// function TimeSpline::Sample evaluates on the device), ModelDerivatives::Compute -> mjpc_b200_model_derivatives,
// CostDerivatives::Compute -> mjpc_b200_cost_derivatives.  Gradient::Compute (a sequential O(H n^2) recursion) and the
// spline mappings are host arithmetic in double, as in the reference.
#pragma once
#include <memory>
#include <shared_mutex>
#include <vector>

#include "ilqg_planner.h"
#include "sampling_planner.h"

namespace mjpc_b200_host {

// Linear operator "spline parameters at input_times -> actions at output_times" (spline_mapping.cc:35-208).  The
// reference stores its Kronecker product with I_nu; the operator is block diagonal over the action dimension, so only the
// scalar weights W [num_output][num_input] are kept.
void SplineMapping(int representation, const std::vector<double>& input_times, const double* output_times, int num_output,
                   std::vector<double>* W);

// Gradient::Compute (gradient.cc:76-107): k [T][m] (row T-1 repeats row T-2), dV[0] = sum_t k_t . Qu_t.  A [T][n][n],
// B [T][n][m], cx [T][n], cu [T][m] as returned by the ABI (float).
void GradientSweep(const float* A, const float* B, const float* cx, const float* cu, int n, int m, int T,
                   std::vector<double>* k, double* dV0);

struct GradientPlannerSettings {        // gradient/settings.h:21-27
  int max_rollout = 1;
  double min_linesearch_step = 1.0e-8;
  double fd_tolerance = 3.0e-4;   // fp32: centred 3e-4 (ilqg_planner.h); the reference's gradient planner uses 1e-5 one-sided in fp64
  int fd_mode = 1;
  int action_limits = 1;
  int derivative_skip = 0;
  int differentiable = 1;               // agent.cc:158-164
};

struct GradientPolicy {                 // gradient/policy.h:29-68
  std::vector<double> parameters, times, ctrlrange;   // [P][nu], [P], [nu][2]
  int num_spline_points = 0, nu = 0, representation = 1;
  void Action(double* action, double time) const;      // policy.cc:80-103
};

class GradientPlanner : public Planner {
 public:
  int Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int representation,
                 double timestep, const double* ctrlrange, int max_horizon, int device);
  void Reset(int horizon, const double* initial_repeated_action) override;
  int OptimizePolicy(int horizon) override;              // planner.cc:159-330; 1 = improved, 0 = not, <0 error
  int NominalTrajectory(int) override { return 0; }      // not restated: planning disabled leaves the plan as it is
  void ResamplePolicy(int horizon);                      // :356-383
  // the policy does not depend on the state
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  const Trajectory* BestTrajectory() override { return winner >= 0 ? &best_ : nullptr; }

  GradientPlannerSettings settings;
  GradientPolicy policy, previous_policy;
  int winner = -1;
  double action_step = 0, expected = 0, improvement = 0, surprise = 0, total_return = 0;

 private:
  int Rollouts(const std::vector<double>& parameters, int count, int horizon);   // count candidates [count][P][nu]
  int Fetch(int candidate, int horizon, double ret);     // trajectory[0] = trajectory[candidate], never a failure
  int K_ = 32, nu_ = 0, n_ = 0, nr_ = 0, Hmax_ = 0;
  double timestep_ = 0.01;
  GradientPolicy cand_;                                   // candidate_policy[0]
  std::vector<float> A_, B_, C_, D_, cx_, cu_, cxx_, cuu_, cxu_, knots_, ret_;
  std::vector<uint8_t> fail_;
  std::vector<int> order_;
  Trajectory best_;                                       // trajectory[0] / trajectory[winner]
  mutable std::shared_mutex mtx_;
};

// iLQSPlanner: a SamplingPlanner and an iLQGPlanner on the same state (ilqs/planner.cc:87-215)
class iLQSPlanner : public Planner {
 public:
  enum { kSampling = 0, kiLQG = 1 };
  int Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                 double exploration, double timestep, const double* ctrlrange, uint32_t seed, int ilqg_num_rollouts,
                 int ilqg_representation, double fd_tolerance, int max_horizon, int device);
  void Reset(int horizon, const double* initial_repeated_action) override;
  void SetState(const double* state, double time, const double* mocap) override;
  int OptimizePolicy(int horizon) override;
  int NominalTrajectory(int horizon) override;
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  const Trajectory* BestTrajectory() override {
    return active_policy == kSampling ? sampling.BestTrajectory() : ilqg.BestTrajectory();
  }
  std::vector<mjpc_b200_t*> Handles() override { return {sampling.gpu(), ilqg.gpu()}; }
  SamplingPlanner sampling;
  iLQGPlanner ilqg;
  int active_policy = kSampling, previous_active_policy = kSampling;

 private:
  int nu_ = 0;
  double timestep_ = 0.01;
};

}  // namespace mjpc_b200_host
