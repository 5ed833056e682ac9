// planner.h - the interface every host planner implements (the reference's virtual Planner,
// mjpc/planners/planner.h:33-77, limited to what exists here) and the engine plumbing they share: the engine handle,
// the planning state, the spline launch and the trajectory fetch.
#pragma once
#include <cstdint>
#include <vector>

#include "../../../include/mjpc_b200.h"

namespace mjpc_b200_host {

struct Trajectory {                                   // mjpc/trajectory.h:74-86 (device arithmetic: float)
  int horizon = 0, dim_state = 0, dim_action = 0, dim_residual = 0, dim_trace = 0;
  std::vector<float> states, actions, residual, costs, trace;
  std::vector<double> times;
  double total_return = 0;
  bool failure = false;
};

// FindInterval (mjpc/utilities.cc:303-330): the indices of the entries of a non-decreasing sequence around `value`,
// clamped to the sequence
void FindInterval(int* bounds, const double* sequence, double value, int length);

// MakeDifferentiable while planning, restored afterwards (agent.cc:296-309,346-356)
struct DifferentiableScope {
  mjpc_b200_t* g; bool on;
  DifferentiableScope(mjpc_b200_t* g_, bool on_) : g(g_), on(on_) { if (on) mjpc_b200_set_differentiable(g, 1); }
  ~DifferentiableScope() { if (on) mjpc_b200_set_differentiable(g, 0); }
};

class Planner {
 public:
  virtual ~Planner();
  virtual void Reset(int horizon, const double* initial_repeated_action) = 0;
  // State::CopyTo (state.cc:128-135); a NULL mocap keeps the previous one
  virtual void SetState(const double* state, double time, const double* mocap);
  virtual int OptimizePolicy(int horizon) = 0;
  virtual int NominalTrajectory(int horizon) = 0;
  virtual void ActionFromPolicy(double* action, const double* state, double time, bool use_previous) = 0;
  virtual const Trajectory* BestTrajectory() = 0;
  // every engine handle the planner plans on: Agent applies the planning-model options and the task snapshot to each
  virtual std::vector<mjpc_b200_t*> Handles() { return {gpu_}; }
  mjpc_b200_t* gpu() { return gpu_; }

 protected:
  // borrowed != nullptr: plan on that handle (not owned); otherwise create one for max_candidates x max_horizon.
  // Sizes state_ and mocap_ from the handle's model.
  int AttachEngine(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                   mjpc_b200_t* borrowed = nullptr);
  // mjpc_b200_rollout_spline from state_, time_ and mocap_ with the handle's task snapshot; sets horizon_
  int RolloutSpline(const float* knots, const double* knot_times, int interpolation, int P, int N, int horizon,
                    float* returns, uint8_t* failure, int* order);
  // sizes *out to `horizon` rows and fetches trajectory `candidate` (flat index) of the handle's last launch into it;
  // total_return and failure are the caller's
  int FetchTrajectory(int candidate, int horizon, Trajectory* out);

  mjpc_b200_t* gpu_ = nullptr;
  bool owns_gpu_ = false;
  mjpc_b200_info info_{};
  std::vector<double> state_, mocap_;
  double time_ = 0;
  int horizon_ = 0;                                   // of the last spline launch: the rows a fetch fills
};

}  // namespace mjpc_b200_host
