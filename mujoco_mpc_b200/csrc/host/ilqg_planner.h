// ilqg_planner.h - C++ host side of the iLQG planner with the reference's method names
// (mjpc/planners/ilqg/planner.h, planner.cc:40-740; settings.h:21-36; backward_pass.cc:327-356 regularisation).
// Every sweep is one call of the C ABI: NominalTrajectory / ActionRollouts -> mjpc_b200_rollout_feedback,
// ModelDerivatives::Compute -> mjpc_b200_model_derivatives, CostDerivatives::Compute -> mjpc_b200_cost_derivatives,
// the Riccati loop -> mjpc_b200_backward_pass (the regularisation retry loop, planner.cc:429-520, stays here).
// The host work around each call is split into prepare / install halves, so BatchILQGPlanner (batch_ilqg_planner.h)
// can run the same halves for several planners around one batched call.
#pragma once
#include <cstdint>
#include <shared_mutex>
#include <vector>

#include "../../../include/mjpc_b200.h"
#include "sampling_planner.h"

namespace mjpc_b200_host {

struct iLQGSettings {                    // mjpc/planners/ilqg/settings.h:21-36
  double min_linesearch_step = 1.0e-3;
  // The reference's settings are 1e-6, one-sided, in fp64.  In fp32 that is below the rounding of the states; measured on
  // the device (profiles/fd_gradient_check.py): with 1e-3 one-sided iLQG does not improve the
  // Quadruped return at all, with CENTRED 3e-4 it follows the fp64 reference (0.124 vs 0.115 after 8 iterations from 0.324).
  double fd_tolerance = 3.0e-4;
  double min_regularization = 1.0e-6;
  double max_regularization = 1.0e6;
  int regularization_type = 0;           // 0 control, 1 feedback, 2 value, 3 none
  int max_regularization_iterations = 5;
  int action_limits = 1;
  int nominal_feedback_scaling = 1;
  int fd_mode = 1;                       // ilqg/settings.h:24: 0 one-sided (reference default), 1 centred (default here, see above)
  int derivative_skip = 0;               // planner.h derivative_skip_ (GUI "Deriv. Skip"): interpolate skipped steps
  // Agent::PlanIteration plans gradient-based planners on a "differentiable" model: solimp[0] = 0 for every joint,
  // geom and pair while planning (agent.cc:296-309,346-356; utilities.cc:60-75; default on, agent.cc:158-164)
  int differentiable = 1;
};

// iLQGPolicy::Action (mjpc/planners/ilqg/policy.cc:82-161) on the host: what the physics thread evaluates between plans.
// Interpolates the nominal actions / states / gains at `time` (representation 0 zero-order, 1 linear, 2 cubic with
// finite-difference slopes; mjpc/utilities.cc:303-422), adds feedback_scaling * K (x (-) x_nominal) with the
// tangent-space state difference (StateDiff, utilities.cc:543-553) when a state is given, clamps to ctrlrange.
struct iLQGPolicyModel {       // the few mjModel fields the policy needs, read from the blob
  int nq = 0, nv = 0, nu = 0;
  std::vector<int> jnt_type, jnt_qposadr, jnt_dofadr;
  std::vector<double> ctrlrange;
  int Load(const mjpc_model_blob* blob);
};
void iLQGPolicyAction(const iLQGPolicyModel& m, const float* u_nom, const float* x_nom, const double* t_nom,
                      const float* gains, int horizon, int representation, double feedback_scaling, const double* state,
                      double time, double* action);

class iLQGPlanner : public Planner {
 public:
  // borrowed != nullptr: plan on that engine handle (not owned; it must hold max_horizon and num_rollouts candidates)
  int Initialize(const mjpc_model_blob* model, int num_rollouts, int representation, int max_horizon, int device,
                 mjpc_b200_t* borrowed = nullptr);
  void Reset(int horizon, const double* initial_repeated_action) override;
  int OptimizePolicy(int horizon) override;       // planner.cc:156-165: NominalTrajectory + Iteration; 1 = policy updated
  int NominalTrajectory(int horizon) override;    // :167-223
  int Iteration(int horizon);                     // :377-627
  // ilqg/policy.cc:82-161; there is no previous policy, so use_previous is ignored
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  const Trajectory* BestTrajectory() override { return &best_; }

  iLQGSettings settings;
  // the LIVE policy (iLQGPolicy policy): nominal trajectory, feedback gains, open-loop improvement.  Only written
  // under the unique lock at the end of a successful Iteration (planner.cc:597-605); buffers keep max_horizon rows.
  std::vector<float> states, actions, residual, gains, du;
  std::vector<double> times;
  double total_return = 0, regularization = 1.0, regularization_rate = 1.0, regularization_factor = 2.0;
  double feedback_scaling = 1.0, improvement = 0, expected = 0, surprise = 0;
  int winner = 0;
  int horizon() const { return live_H_; }
  // candidate_policy[0] / the last K rollouts, as iLQSPlanner needs them (ilqs/planner.cc:98-215)
  const std::vector<double>& candidate_times() const { return c_times_; }
  const std::vector<float>& candidate_actions() const { return c_actions_; }
  double candidate_return() const { return c_return_; }
  void SetCandidateTrajectory(const Trajectory& tr);      // candidate_policy[0].trajectory = tr
  float rollout_return(int j) const { return ret_[j]; }   // trajectory[j].total_return of the last K rollouts
  int dim_state() const { return ds_; }
  int dim_action() const { return nu_; }

 private:
  friend class BatchILQGPlanner;
  std::vector<float> StepSizes() const;                                   // LogScale (utilities.cc:819-825) + trailing 0
  static int BestRollout(const float* ret, const uint8_t* fail, int K);  // :727-740
  // candidate_policy[0].trajectory = trajectory[candidate]; candidate is the flat index of the last launch
  int FetchCandidate(int candidate, double ret);
  // NominalTrajectory = PrepareNominal (policy snapshot, staging) + feedback launch + InstallNominal (winner, copy)
  int PrepareNominal(int horizon);
  int InstallNominal(const float* ret, const uint8_t* fail, int cand0);
  // Iteration = PrepareIteration + derivatives + cost derivatives + {BackwardPending -> backward pass ->
  // AfterBackward}* + InstallGains + action rollouts + InstallActions (winner, UpdateRegularization, publish)
  int PrepareIteration(int horizon);
  bool BackwardPending(int status) const { return reg_iter_ < settings.max_regularization_iterations && status == 0; }
  void AfterBackward(int status);
  bool InstallGains(int status);
  int InstallActions(const float* ret, const uint8_t* fail, int cand0);
  void ScaleRegularization(double factor);                                // backward_pass.cc:327-343
  void UpdateRegularization(double z, double s);                          // :345-356
  iLQGPolicyModel pm_;
  mutable std::shared_mutex mtx_;   // the policy is read by the physics thread while a plan installs a new one
  int K_ = 10, representation_ = 1, H_ = 0, Hmax_ = 0, nu_ = 0, ds_ = 0, n_ = 0, nr_ = 0;
  // candidate_policy[0]: the working copy NominalTrajectory / Iteration operate on (planner.cc:190-222,392-560)
  std::vector<float> c_states_, c_actions_, c_residual_, c_gains_, c_du_;
  std::vector<double> c_times_;
  double c_return_ = 0;
  int live_H_ = 0;
  // staged by the prepare halves: the launch inputs of this planner's problem
  std::vector<float> steps_, st_, mc_;
  double previous_return_ = 0;
  int reg_iter_ = 0, iter_H_ = 0;
  float dV_[2] = {0, 0};
  std::vector<float> A_, B_, C_, D_, cx_, cu_, cxx_, cuu_, cxu_, Kbuf_, dubuf_, ret_;
  std::vector<uint8_t> fail_;
  std::vector<int> order_;
  Trajectory best_;
};

}  // namespace mjpc_b200_host
