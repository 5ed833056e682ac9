// agent.cc - see agent.h
#include "agent.h"

#include <algorithm>
#include <cmath>

namespace mjpc_b200_host {

int Agent::Steps(double horizon, double timestep) {
  // steps_ = mju_max(mju_min(horizon_ / timestep_ + 1, kMaxTrajectoryHorizon), 1): a double truncated on assignment to int
  return (int)std::max(std::min(horizon / timestep + 1, (double)kMaxTrajectoryHorizon), 1.0);
}

int Agent::Initialize(const mjpc_model_blob* model, const AgentSettings& s, const double* ctrlrange, int device) {
  settings = s;
  steps_ = Steps(s.horizon, s.timestep);
  const bool gradient_planner = s.planner == kGradientPlanner || s.planner == kILQGPlanner || s.planner == kILQSPlanner;
  differentiable_ = s.differentiable < 0 ? (gradient_planner ? 1 : 0) : (s.differentiable != 0);
  const int Hmax = std::max(steps_, 2);
  int rc = 0;
  switch (s.planner) {
    case kSamplingPlanner: {
      auto* p = new SamplingPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.num_trajectory, s.num_spline_points, s.representation, s.exploration, 0.0, s.timestep,
                         ctrlrange, s.seed, s.num_trajectory, Hmax, device);
      break;
    }
    case kGradientPlanner: {
      auto* p = new GradientPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.num_trajectory, s.num_spline_points, s.representation, s.timestep, ctrlrange, Hmax, device);
      if (!rc) { p->settings.fd_tolerance = s.fd_tolerance; p->settings.differentiable = 0; }   // the Agent owns the switch
      break;
    }
    case kILQGPlanner: {
      auto* p = new iLQGPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.ilqg_num_rollouts, s.ilqg_representation, Hmax, device);
      if (!rc) { p->settings.fd_tolerance = s.fd_tolerance; p->settings.differentiable = 0; }
      break;
    }
    case kILQSPlanner: {
      auto* p = new iLQSPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.num_trajectory, s.num_spline_points, s.representation, s.exploration, s.timestep, ctrlrange,
                         s.seed, s.ilqg_num_rollouts, s.ilqg_representation, s.fd_tolerance, Hmax, device);
      if (!rc) p->ilqg.settings.differentiable = 0;
      break;
    }
    case kRobustPlanner: {
      std::unique_ptr<SamplingPlanner> d(new SamplingPlanner);
      rc = d->Initialize(model, s.num_trajectory, s.num_spline_points, s.representation, s.exploration, 0.0, s.timestep, ctrlrange,
                         s.seed, s.num_trajectory, Hmax, device);
      if (rc) break;
      const int reps = s.robust_repetitions > 0 ? s.robust_repetitions : 5;
      const int ncand = s.robust_candidates > 0 ? s.robust_candidates : std::max(s.num_trajectory / reps, 1);
      auto* p = new RobustPlanner;
      planner_.reset(p);
      rc = p->Initialize(std::move(d), model, ncand * reps, Hmax, device);
      if (!rc) p->Configure(s.num_trajectory, ncand, reps, s.robust_xfrc, s.robust_xfrc_rate, s.seed);
      break;
    }
    case kCrossEntropyPlanner: {
      auto* p = new CrossEntropyPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.num_trajectory, s.n_elite > 0 ? s.n_elite : std::max(s.num_trajectory / 10, 2),
                         s.num_spline_points, s.representation, s.exploration, s.std_min, s.explore_fraction, s.timestep,
                         ctrlrange, s.seed, Hmax, device);
      break;
    }
    case kSampleGradientPlanner: {   // not gradient-based for MakeDifferentiable (agent.cc:155-163)
      auto* p = new SampleGradientPlanner;
      planner_.reset(p);
      rc = p->Initialize(model, s.num_trajectory, s.num_gradient, s.num_spline_points, s.representation, s.exploration,
                         s.gradient_filter, s.timestep, ctrlrange, s.seed, Hmax, device);
      break;
    }
    default:
      return MJPC_B200_ERR_UNSUPPORTED;
  }
  if (rc) return rc;
  std::vector<mjpc_b200_t*> hs = planner_->Handles();
  mjpc_b200_get_info(hs[0], &info_);
  state_.assign(info_.dim_state, 0.0); mocap_.assign(7 * info_.nmocap, 0.0);
  // model_->opt.timestep = timestep_; model_->opt.integrator = integrator_ (agent.cc:288-289) on every planning model
  for (mjpc_b200_t* h : hs)
    if (int orc = mjpc_b200_set_options(h, s.timestep, s.integrator)) return orc;
  return 0;
}

void Agent::Reset(const double* a) { planner_->Reset(steps_, a); }

void Agent::SetState(const double* state, double time, const double* mocap) {
  std::copy(state, state + state_.size(), state_.begin());
  if (!mocap_.empty() && mocap) std::copy(mocap, mocap + mocap_.size(), mocap_.begin());
  time_ = time;
}

void Agent::SetTask(const mjpc_task_desc* task) {
  if (!task) return;
  if (task->weight) weight_.assign(task->weight, task->weight + info_.num_term);
  if (task->parameters) parameters_.assign(task->parameters, task->parameters + info_.num_parameters);
  if (task->task_state) task_state_.assign(task->task_state, task->task_state + info_.task_state_size);
  risk_ = task->risk;
  have_task_ = true;
}

int Agent::PlanIteration() {
  steps_ = Steps(settings.horizon, settings.timestep);
  std::vector<mjpc_b200_t*> hs = planner_->Handles();
  for (mjpc_b200_t* h : hs) {
    if (int rc = mjpc_b200_set_options(h, settings.timestep, settings.integrator)) return rc;
    mjpc_b200_set_differentiable(h, differentiable_);                      // MakeDifferentiable (agent.cc:296-309)
  }
  planner_->SetState(state_.data(), time_, mocap_.empty() ? nullptr : mocap_.data());   // ActivePlanner().SetState(state)
  if (have_task_) {   // residual_fn_ = ActiveTask()->Residual(): the snapshot stays constant during planning (agent.cc:316-319)
    mjpc_task_desc td{weight_.empty() ? nullptr : weight_.data(), parameters_.empty() ? nullptr : parameters_.data(),
                      task_state_.empty() ? nullptr : task_state_.data(), risk_};
    for (mjpc_b200_t* h : hs)
      if (int rc = mjpc_b200_set_task(h, &td)) return rc;
  }
  const int rc = plan_enabled ? planner_->OptimizePolicy(steps_) : planner_->NominalTrajectory(steps_);
  for (mjpc_b200_t* h : hs) mjpc_b200_set_differentiable(h, 0);            // restore solimp defaults (agent.cc:346-356)
  return rc;
}

void Agent::ActionFromPolicy(double* action, const double* state, double time, bool use_previous) {
  planner_->ActionFromPolicy(action, state, time, use_previous);
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::Agent;
using mjpc_b200_host::AgentSettings;

extern "C" {

int mjpc_b200_agent_steps(double horizon, double timestep) { return Agent::Steps(horizon, timestep); }

// settings[20] = {planner, horizon, timestep, integrator, differentiable (-1 default), num_trajectory, num_spline_points,
//                 representation, exploration, ilqg_num_rollouts, ilqg_representation, fd_tolerance, n_elite, std_min,
//                 explore_fraction, robust_candidates, robust_repetitions, robust_xfrc, robust_xfrc_rate, seed}
// settings[22] for the Sample Gradient planner (planner 6): settings[20] = sample_gradient_trajectories,
//                 settings[21] = sample_gradient_filter; read only for planner 6, so the other planners may pass 20
int mjpc_b200_agent_create(const mjpc_model_blob* model, const double* settings, const double* ctrlrange, int device, void** out) {
  if (!model || !settings || !ctrlrange || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  AgentSettings s;
  s.planner = (int)settings[0]; s.horizon = settings[1]; s.timestep = settings[2]; s.integrator = (int)settings[3];
  s.differentiable = (int)settings[4]; s.num_trajectory = (int)settings[5]; s.num_spline_points = (int)settings[6];
  s.representation = (int)settings[7]; s.exploration = settings[8]; s.ilqg_num_rollouts = (int)settings[9];
  s.ilqg_representation = (int)settings[10]; s.fd_tolerance = settings[11]; s.n_elite = (int)settings[12];
  s.std_min = settings[13]; s.explore_fraction = settings[14]; s.robust_candidates = (int)settings[15];
  s.robust_repetitions = (int)settings[16]; s.robust_xfrc = settings[17]; s.robust_xfrc_rate = settings[18];
  s.seed = (unsigned)settings[19];
  if (s.planner == mjpc_b200_host::kSampleGradientPlanner) { s.num_gradient = (int)settings[20]; s.gradient_filter = settings[21]; }
  auto* a = new Agent;
  int rc = a->Initialize(model, s, ctrlrange, device);
  if (rc) { delete a; *out = nullptr; return rc; }
  *out = a;
  return 0;
}
void mjpc_b200_agent_destroy(void* a) { delete (Agent*)a; }
void mjpc_b200_agent_reset(void* a, const double* initial_repeated_action) { ((Agent*)a)->Reset(initial_repeated_action); }
void mjpc_b200_agent_set_state(void* a, const double* state, double time, const double* mocap) { ((Agent*)a)->SetState(state, time, mocap); }
void mjpc_b200_agent_set_task(void* a, const mjpc_task_desc* task) { ((Agent*)a)->SetTask(task); }
void mjpc_b200_agent_set_plan_enabled(void* a, int on) { ((Agent*)a)->plan_enabled = on != 0; }
int mjpc_b200_agent_plan_iteration(void* a) { return ((Agent*)a)->PlanIteration(); }
int mjpc_b200_agent_get_steps(void* a) { return ((Agent*)a)->steps(); }
void mjpc_b200_agent_action_from_policy(void* a, double* action, const double* state, double time, int use_previous) {
  ((Agent*)a)->ActionFromPolicy(action, state, time, use_previous != 0);
}

}  // extern "C"
