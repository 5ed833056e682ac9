// agent.h - the plan-side glue of mjpc::Agent above the planners (mjpc/agent.cc:85-107,150-164,283-357):
//   settings     agent_planner / agent_horizon / agent_timestep / agent_integrator / agent_differentiable
//   steps_       = max(min(horizon / timestep + 1, kMaxTrajectoryHorizon), 1), truncated to int (agent.cc:107,292-293)
//   PlanIteration  timestep + integrator override of the planning model, MakeDifferentiable around gradient-based
//                planners, planner.SetState(state), the per-iteration residual snapshot (Task::Residual() ->
//                mjpc_b200_set_task on every engine handle the active planner owns), then OptimizePolicy(steps_) - or
//                NominalTrajectory(steps_) when planning is disabled
// The GUI / estimator / threading of Agent (agent.cc:360-1100) are outside the hot path and stay in the reference.
#pragma once
#include <memory>
#include <vector>

#include "cross_entropy_planner.h"
#include "gradient_planner.h"
#include "ilqg_planner.h"
#include "robust_planner.h"
#include "sample_gradient_planner.h"
#include "sampling_planner.h"

namespace mjpc_b200_host {

enum PlannerType : int {            // mjpc/planners/include.h:26-34
  kSamplingPlanner = 0, kGradientPlanner, kILQGPlanner, kILQSPlanner, kRobustPlanner, kCrossEntropyPlanner,
  kSampleGradientPlanner
};
constexpr int kMaxTrajectoryHorizon = 512;   // mjpc/trajectory.h

struct AgentSettings {              // what the reference reads from the task XML's <custom> numerics
  int planner = kSamplingPlanner;   // agent_planner
  double horizon = 0.5;             // agent_horizon  (agent.cc:100)
  double timestep = 1.0e-2;         // agent_timestep (agent.cc:103)
  int integrator = 0;               // agent_integrator (agent.cc:96-97); only Euler (0) is implemented on the device
  int differentiable = -1;          // agent_differentiable; -1 = default: on for Gradient / iLQG / iLQS (agent.cc:158-164)
  // planner settings (sampling_* / gradient_* / ilqg_* / robust_* numerics)
  int num_trajectory = 10, num_spline_points = 3, representation = 2;
  double exploration = 0.1;
  int ilqg_num_rollouts = 10, ilqg_representation = 1;
  double fd_tolerance = 3.0e-4;     // with centred differences (ilqg_planner.h)
  int n_elite = 0; double std_min = 0.01, explore_fraction = 0.0;
  int robust_candidates = -1, robust_repetitions = 5; double robust_xfrc = 0.1, robust_xfrc_rate = 0.1;
  int num_gradient = 0; double gradient_filter = 1.0;   // sample_gradient_trajectories / sample_gradient_filter
  unsigned seed = 0x5EED;
};

class Agent {
 public:
  int Initialize(const mjpc_model_blob* model, const AgentSettings& s, const double* ctrlrange, int device);
  void Reset(const double* initial_repeated_action);
  void SetState(const double* state, double time, const double* mocap);            // State::CopyTo (state.cc:128-135)
  void SetTask(const mjpc_task_desc* task);                                         // Task::Residual() snapshot source
  int PlanIteration();                                                              // agent.cc:283-357
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false);
  static int Steps(double horizon, double timestep);                                // agent.cc:107
  int steps() const { return steps_; }
  bool plan_enabled = true;
  AgentSettings settings;

 private:
  int steps_ = 1, differentiable_ = 0;
  std::unique_ptr<Planner> planner_;
  std::vector<double> state_, mocap_, weight_, parameters_, task_state_;
  double time_ = 0, risk_ = 0;
  bool have_task_ = false;
  mjpc_b200_info info_{};
};

}  // namespace mjpc_b200_host
