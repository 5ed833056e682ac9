// planner.h - the interface every host planner implements (the reference's virtual Planner,
// mjpc/planners/planner.h:33-77, limited to what exists here) and the engine plumbing they share: the engine handle,
// the planning state, the spline launch and the trajectory fetch.  Also the host maths the planners share: the Cholesky
// factor, FindInterval and the host model's state difference.
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

// the candidates of one spline launch of one planning problem: knots [N][P][nu], knot times [P] (absolute)
struct SplineCandidates {
  int N = 0, P = 0, interpolation = 0;
  std::vector<float> knots;
  std::vector<double> knot_times;
  void Resize(int n, int p, int nu) { N = n; P = p; knots.resize((size_t)n * p * nu); knot_times.resize(p); }
};

// the task snapshots of the problems of a launch: rows [..][nw], [..][np], [..][nts].  Empty (no rows): every problem
// reads the handle's set_task snapshot, as the engine does for NULL task arrays
struct TaskRows {
  const double *w = nullptr, *p = nullptr, *ts = nullptr;
  int nw = 0, np = 0, nts = 0;
};

class Planner;

// The staging and the results of one mjpc_b200_rollout_spline_batched launch.  Run launches, on the handle of from[0],
// the candidates cands[b] (common N, P and interpolation) of problem b from planner from[b]'s state, time and mocap with
// task row b of `rows`; every planner of from plans on that handle.  Fills returns, failure and order [B][N].
class SplineLaunch {
 public:
  int Run(const std::vector<const Planner*>& from, const std::vector<const SplineCandidates*>& cands,
          const TaskRows& rows, int horizon);
  std::vector<float> returns;
  std::vector<uint8_t> failure;
  std::vector<int> order;

 private:
  std::vector<float> states_, mocaps_, knots_;
  std::vector<double> times_, knot_times_, covariances_;
};

// mju_cholFactor: in-place lower Cholesky factor of the row-major n x n matrix M (upper triangle left as it was); a
// pivot below mindiag is raised to mindiag.  Returns the rank, the number of pivots that were not raised.
int CholFactor(double* M, int n, double mindiag);

// FindInterval (mjpc/utilities.cc:303-330): the indices of the entries of a non-decreasing sequence around `value`,
// clamped to the sequence
void FindInterval(int* bounds, const double* sequence, double value, int length);

struct HostModel {             // the few mjModel fields the host-side state arithmetic needs, read from the blob
  int nq = 0, nv = 0, nu = 0;
  std::vector<int> jnt_type, jnt_qposadr, jnt_dofadr;
  std::vector<double> ctrlrange;
  int Load(const mjpc_model_blob* blob);
};
// StateDiff (utilities.cc:543-553): dx [2 nv] = x_to (-) x_from, positions in the tangent space (mj_differentiatePos)
void StateDiff(const HostModel& m, double* dx, const double* x_to, const double* x_from);

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
  // finite-difference settings of the planners that take derivatives (SetFiniteDifferences); the others:
  // MJPC_B200_ERR_UNSUPPORTED
  virtual int SetFD(double tolerance, int mode, int derivative_skip) { return MJPC_B200_ERR_UNSUPPORTED; }
  // plan on a model ensemble (mjpc_b200_set_model_ensemble on the planner's handle): the planners whose iteration ranks
  // by SplineLaunch's returns, which are then the scores; the others: MJPC_B200_ERR_UNSUPPORTED
  virtual int SetEnsemble(const mjpc_model_blob* models, int K, int worst) { return MJPC_B200_ERR_UNSUPPORTED; }
  // plan over the state covariance (mjpc_b200_planner_set_state_ensemble / _set_state_covariance): SplineLaunch then
  // runs mjpc_b200_rollout_spline_belief_batched; the planners whose iteration ranks by its returns, the others:
  // MJPC_B200_ERR_UNSUPPORTED
  virtual int SetStateEnsemble(int K, int worst, uint32_t seed) { return MJPC_B200_ERR_UNSUPPORTED; }
  virtual int SetStateCovariance(const double* covariance) { return MJPC_B200_ERR_UNSUPPORTED; }
  // the counter of the planner's iterations, which its state-ensemble draws take (0 for the kinds without them)
  virtual uint32_t PlanIteration() const { return 0; }
  int state_members() const { return state_members_; }
  int state_worst() const { return state_worst_; }
  uint32_t state_seed() const { return state_seed_; }
  const std::vector<double>& state_covariance() const { return state_cov_; }
  // every engine handle the planner plans on: Agent applies the planning-model options and the task snapshot to each
  virtual std::vector<mjpc_b200_t*> Handles() { return {gpu_}; }
  mjpc_b200_t* gpu() const { return gpu_; }
  const std::vector<double>& state() const { return state_; }
  const std::vector<double>& mocap() const { return mocap_; }
  double time() const { return time_; }

 protected:
  // borrowed != nullptr: plan on that handle (not owned); otherwise create one for max_candidates x max_horizon.
  // Sizes state_ and mocap_ from the handle's model.
  int AttachEngine(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                   mjpc_b200_t* borrowed = nullptr);
  // sizes *out to `horizon` rows and fetches trajectory `candidate` of the handle's last launch into it (flat index
  // launch_offset_ + candidate); total_return and failure are the caller's
  int FetchTrajectory(int candidate, int horizon, Trajectory* out);
  // SetEnsemble / SetStateEnsemble / SetStateCovariance of the kinds that support them: a model ensemble and a state
  // ensemble exclude each other (MJPC_B200_ERR_UNSUPPORTED)
  int ModelEnsemble(const mjpc_model_blob* models, int K, int worst);
  int StateEnsemble(int K, int worst, uint32_t seed);
  int StateCovariance(const double* covariance);

  mjpc_b200_t* gpu_ = nullptr;
  bool owns_gpu_ = false;
  mjpc_b200_info info_{};
  std::vector<double> state_, mocap_;
  double time_ = 0;
  int horizon_ = 0;                                   // of the last spline launch: the rows a fetch fills
  int launch_offset_ = 0;                             // flat index of this planner's candidate 0 in that launch
  SplineLaunch launch_;                               // of the spline launches the planner makes when it plans alone
  bool model_ensemble_ = false;                       // SetEnsemble set one
  int state_members_ = 0, state_worst_ = 0;           // SetStateEnsemble (0: none)
  uint32_t state_seed_ = 0;
  std::vector<double> state_cov_;                     // [2 nv][2 nv], zero until SetStateCovariance
};

// SetFD for a settings struct with fd_tolerance, fd_mode and derivative_skip: tolerance <= 0, mode < 0 and
// derivative_skip < 0 keep the current value
template <class Settings>
int SetFiniteDifferences(Settings* s, double tolerance, int mode, int derivative_skip) {
  if (tolerance > 0) s->fd_tolerance = tolerance;
  if (mode >= 0) s->fd_mode = mode ? 1 : 0;
  if (derivative_skip >= 0) s->derivative_skip = derivative_skip;
  return 0;
}

// mjpc_b200_planner_t* is the Planner base of the planner, whatever its kind
inline mjpc_b200_planner_t* ToHandle(Planner* p) { return reinterpret_cast<mjpc_b200_planner_t*>(p); }
// the planner behind a handle if it is a T, else nullptr (a NULL handle, or one of another kind)
template <class T>
T* PlannerOf(mjpc_b200_planner_t* h) { return dynamic_cast<T*>(reinterpret_cast<Planner*>(h)); }

}  // namespace mjpc_b200_host
