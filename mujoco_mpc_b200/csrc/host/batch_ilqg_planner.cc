// batch_ilqg_planner.cc - see batch_ilqg_planner.h.  Compiled into libmjpc_b200.so next to the engine.
#include "batch_ilqg_planner.h"

#include <algorithm>
#include <exception>

#include "../dev_model.h"   // Blob reader (plain C++)

namespace mjpc_b200_host {

namespace {
// dst[j] = the first `per` values of row(idx[j]), back to back
template <class T, class F>
void gather(std::vector<T>& dst, const std::vector<int>& idx, size_t per, F row) {
  dst.resize(idx.size() * per);
  for (size_t j = 0; j < idx.size(); j++) {
    const T* src = row(idx[j]);
    std::copy(src, src + per, dst.begin() + j * per);
  }
}
}  // namespace

BatchILQGPlanner::~BatchILQGPlanner() {
  problems_.clear();   // the planners borrow the handle
  if (gpu_) mjpc_b200_destroy(gpu_);
}

int BatchILQGPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_rollouts, int representation,
                                 int max_horizon, int device) {
  if (num_problems < 1 || num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  // every problem's task snapshot starts as the model's
  try {
    mjpc_dev::Blob blob(model->data, model->nbytes);
    weight_ = blob.reals("task_weight"); parameters_ = blob.reals("task_parameters"); task_state_ = blob.reals("task_state");
  } catch (const std::exception&) {
    return MJPC_B200_ERR_BAD_BLOB;
  }
  nw_ = (int)weight_.size(); np_ = (int)parameters_.size(); nts_ = (int)task_state_.size();
  std::vector<double> w(weight_), p(parameters_), s(task_state_);
  for (int b = 1; b < num_problems; b++) {
    weight_.insert(weight_.end(), w.begin(), w.end());
    parameters_.insert(parameters_.end(), p.begin(), p.end());
    task_state_.insert(task_state_.end(), s.begin(), s.end());
  }
  K_ = num_rollouts;
  representation_ = representation;
  if (int rc = mjpc_b200_create(model, num_problems * num_rollouts, max_horizon, device, &gpu_)) return rc;
  mjpc_b200_info info;
  mjpc_b200_get_info(gpu_, &info);
  nu_ = info.nu; ds_ = info.dim_state; n_ = info.dim_dstate; nr_ = info.num_residual; nmocap7_ = 7 * info.nmocap;
  for (int b = 0; b < num_problems; b++) {
    problems_.emplace_back(new iLQGPlanner);
    if (int rc = problems_.back()->Initialize(model, num_rollouts, representation, max_horizon, device, gpu_)) return rc;
  }
  return 0;
}

void BatchILQGPlanner::SetTask(int b, const double* weight, const double* parameters, const double* task_state) {
  if (weight) std::copy(weight, weight + nw_, weight_.begin() + (size_t)b * nw_);
  if (parameters) std::copy(parameters, parameters + np_, parameters_.begin() + (size_t)b * np_);
  if (task_state) std::copy(task_state, task_state + nts_, task_state_.begin() + (size_t)b * nts_);
}

// one rollout_feedback_batched launch of the candidate policies of the problems `idx`, as each iLQGPlanner makes it
int BatchILQGPlanner::FeedbackLaunch(const std::vector<int>& idx, int horizon, bool with_du, int mode) {
  const size_t H = horizon, J = idx.size();
  auto pl = [&](int b) -> iLQGPlanner& { return *problems_[b]; };
  gather(st_, idx, ds_, [&](int b) { return pl(b).st_.data(); });
  gather(mc_, idx, nmocap7_, [&](int b) { return pl(b).mc_.data(); });
  gather(times_, idx, 1, [&](int b) { return &pl(b).time_; });
  gather(u_, idx, H * nu_, [&](int b) { return pl(b).c_actions_.data(); });
  gather(x_, idx, H * ds_, [&](int b) { return pl(b).c_states_.data(); });
  gather(t_, idx, H, [&](int b) { return pl(b).c_times_.data(); });
  gather(g_, idx, H * nu_ * n_, [&](int b) { return pl(b).c_gains_.data(); });
  if (with_du) gather(du_, idx, H * nu_, [&](int b) { return pl(b).c_du_.data(); });
  gather(steps_, idx, K_, [&](int b) { return pl(b).steps_.data(); });
  gather(w_, idx, nw_, [&](int b) { return weight_.data() + (size_t)b * nw_; });
  gather(p_, idx, np_, [&](int b) { return parameters_.data() + (size_t)b * np_; });
  gather(ts_, idx, nts_, [&](int b) { return task_state_.data() + (size_t)b * nts_; });
  ret_.resize(J * K_); fail_.resize(J * K_); order_.resize(J * K_);
  return mjpc_b200_rollout_feedback_batched(gpu_, (int)J, st_.data(), times_.data(), nmocap7_ ? mc_.data() : nullptr,
                                            nw_ ? w_.data() : nullptr, np_ ? p_.data() : nullptr,
                                            nts_ ? ts_.data() : nullptr, u_.data(), x_.data(), t_.data(), g_.data(),
                                            with_du ? du_.data() : nullptr, steps_.data(), mode, K_, horizon,
                                            ret_.data(), fail_.data(), order_.data());
}

int BatchILQGPlanner::Nominal(int horizon) {
  const int B = NumProblems();
  std::vector<int> all(B);
  for (int b = 0; b < B; b++) {
    all[b] = b;
    problems_[b]->settings = settings;
    if (problems_[b]->PrepareNominal(horizon)) return -1;
  }
  if (FeedbackLaunch(all, horizon, false, representation_)) return -1;
  for (int b = 0; b < B; b++)
    if (problems_[b]->InstallNominal(ret_.data() + (size_t)b * K_, fail_.data() + (size_t)b * K_, b * K_) < 0) return -1;
  return 0;
}

int BatchILQGPlanner::Iterate(int horizon, int* updated) {
  const int B = NumProblems();
  const size_t H = horizon, n = n_, m = nu_, nr = nr_;
  std::vector<int> all(B);
  for (int b = 0; b < B; b++) {
    all[b] = b;
    if (updated) updated[b] = 0;
    if (problems_[b]->PrepareIteration(horizon)) return -1;
  }
  auto pl = [&](int b) -> iLQGPlanner& { return *problems_[b]; };
  // derivatives and cost derivatives of every problem (ModelDerivatives / CostDerivatives::Compute)
  gather(x_, all, H * ds_, [&](int b) { return pl(b).c_states_.data(); });
  gather(u_, all, H * m, [&](int b) { return pl(b).c_actions_.data(); });
  gather(t_, all, H, [&](int b) { return pl(b).c_times_.data(); });
  gather(mc_, all, nmocap7_, [&](int b) { return pl(b).mc_.data(); });
  gather(res_, all, H * nr, [&](int b) { return pl(b).c_residual_.data(); });
  A_.resize(B * H * n * n); B_.resize(B * H * n * m); C_.resize(B * H * nr * n); D_.resize(B * H * nr * m);
  cx_.resize(B * H * n); cu_.resize(B * H * m); cxx_.resize(B * H * n * n); cuu_.resize(B * H * m * m);
  cxu_.resize(B * H * n * m);
  if (mjpc_b200_model_derivatives_batched(gpu_, B, x_.data(), u_.data(), t_.data(), nmocap7_ ? mc_.data() : nullptr,
                                          nw_ ? weight_.data() : nullptr, np_ ? parameters_.data() : nullptr,
                                          nts_ ? task_state_.data() : nullptr, horizon, settings.derivative_skip,
                                          (float)settings.fd_tolerance, settings.fd_mode, A_.data(), B_.data(),
                                          C_.data(), D_.data()))
    return -1;
  if (mjpc_b200_cost_derivatives_batched(gpu_, B, nw_ ? weight_.data() : nullptr, res_.data(), C_.data(), D_.data(),
                                         horizon, cx_.data(), cu_.data(), cxx_.data(), cuu_.data(), cxu_.data()))
    return -1;
  // backward passes: round r holds the problems whose pass has not succeeded and whose retry budget is not spent,
  // each at its own regularisation - every problem follows its own iLQGPlanner retry loop
  status_.assign(B, 0);
  for (;;) {
    std::vector<int> act;
    for (int b = 0; b < B; b++) if (pl(b).BackwardPending(status_[b])) act.push_back(b);
    if (act.empty()) break;
    const size_t J = act.size();
    auto row = [&](std::vector<float>& v, size_t per) { return [&v, per](int b) { return v.data() + (size_t)b * per; }; };
    gather(sA_, act, H * n * n, row(A_, H * n * n));
    gather(sB_, act, H * n * m, row(B_, H * n * m));
    gather(scx_, act, H * n, row(cx_, H * n));
    gather(scu_, act, H * m, row(cu_, H * m));
    gather(scxx_, act, H * n * n, row(cxx_, H * n * n));
    gather(scxu_, act, H * n * m, row(cxu_, H * n * m));
    gather(scuu_, act, H * m * m, row(cuu_, H * m * m));
    gather(sact_, act, H * m, [&](int b) { return pl(b).c_actions_.data(); });
    mu_.resize(J);
    for (size_t j = 0; j < J; j++) mu_[j] = (float)pl(act[j]).regularization;
    K_out_.resize(J * H * m * n); du_out_.resize(J * H * m); dV_out_.resize(2 * J);
    std::vector<int> st(J, 0);
    if (mjpc_b200_backward_pass_batched(gpu_, (int)J, sA_.data(), sB_.data(), scx_.data(), scu_.data(), scxx_.data(),
                                        scxu_.data(), scuu_.data(), sact_.data(), horizon, mu_.data(),
                                        settings.regularization_type, settings.action_limits, K_out_.data(),
                                        du_out_.data(), dV_out_.data(), nullptr, nullptr, st.data()))
      return -1;
    for (size_t j = 0; j < J; j++) {
      iLQGPlanner& p = pl(act[j]);
      std::copy(K_out_.begin() + j * H * m * n, K_out_.begin() + (j + 1) * H * m * n, p.Kbuf_.begin());
      std::copy(du_out_.begin() + j * H * m, du_out_.begin() + (j + 1) * H * m, p.dubuf_.begin());
      p.dV_[0] = dV_out_[2 * j]; p.dV_[1] = dV_out_[2 * j + 1];
      status_[act[j]] = st[j];
      p.AfterBackward(st[j]);
    }
  }
  // action rollouts of the problems whose backward pass succeeded; the others are left untouched
  std::vector<int> ok;
  for (int b = 0; b < B; b++) if (pl(b).InstallGains(status_[b])) ok.push_back(b);
  if (ok.empty()) return 0;
  if (FeedbackLaunch(ok, horizon, true, 3)) return -1;
  for (size_t j = 0; j < ok.size(); j++) {
    const int r = pl(ok[j]).InstallActions(ret_.data() + j * K_, fail_.data() + j * K_, (int)j * K_);
    if (r < 0) return -1;
    if (updated) updated[ok[j]] = r;
  }
  return 0;
}

int BatchILQGPlanner::NominalTrajectory(int horizon) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  return Nominal(horizon);
}

int BatchILQGPlanner::OptimizePolicy(int horizon, int* updated) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  if (Nominal(horizon)) return -1;
  return Iterate(horizon, updated);
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::BatchILQGPlanner;

namespace {
BatchILQGPlanner* ilqg_problem_of(void* p, int problem) {
  auto* bp = (BatchILQGPlanner*)p;
  return bp && problem >= 0 && problem < bp->NumProblems() ? bp : nullptr;
}
}  // namespace

extern "C" {

int mjpc_b200_batch_ilqg_planner_create(const mjpc_model_blob* model, int num_problems, int num_rollouts, int representation,
                                        double fd_tolerance, int max_horizon, int device, void** out) {
  if (!model || !model->data || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchILQGPlanner;
  int rc = p->Initialize(model, num_problems, num_rollouts, representation, max_horizon, device);
  if (rc) { delete p; return rc; }
  if (fd_tolerance > 0) p->settings.fd_tolerance = fd_tolerance;
  *out = p;
  return 0;
}
void mjpc_b200_batch_ilqg_planner_destroy(void* p) { delete (BatchILQGPlanner*)p; }
void mjpc_b200_batch_ilqg_planner_set_fd(void* p, double tolerance, int mode, int derivative_skip) {
  if (!p) return;
  auto& s = ((BatchILQGPlanner*)p)->settings;
  if (tolerance > 0) s.fd_tolerance = tolerance;
  if (mode >= 0) s.fd_mode = mode ? 1 : 0;
  if (derivative_skip >= 0) s.derivative_skip = derivative_skip;
}
int mjpc_b200_batch_ilqg_planner_reset(void* p, int problem, int horizon, const double* initial_repeated_action) {
  BatchILQGPlanner* bp = ilqg_problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).Reset(horizon, initial_repeated_action);
  return 0;
}
int mjpc_b200_batch_ilqg_planner_set_state(void* p, int problem, const double* state, double time, const double* mocap) {
  BatchILQGPlanner* bp = ilqg_problem_of(p, problem);
  if (!bp || !state) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).SetState(state, time, mocap);
  return 0;
}
int mjpc_b200_batch_ilqg_planner_set_task(void* p, int problem, const double* weight, const double* parameters,
                                          const double* task_state) {
  BatchILQGPlanner* bp = ilqg_problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->SetTask(problem, weight, parameters, task_state);
  return 0;
}
int mjpc_b200_batch_ilqg_planner_nominal_trajectory(void* p, int horizon) {
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  return ((BatchILQGPlanner*)p)->NominalTrajectory(horizon);
}
int mjpc_b200_batch_ilqg_planner_optimize_policy(void* p, int horizon, int* updated) {
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  return ((BatchILQGPlanner*)p)->OptimizePolicy(horizon, updated);
}
int mjpc_b200_batch_ilqg_planner_action_from_policy(void* p, int problem, double* action, const double* state,
                                                    double time) {
  BatchILQGPlanner* bp = ilqg_problem_of(p, problem);
  if (!bp || !action) return MJPC_B200_ERR_BAD_ARGUMENT;
  bp->problem(problem).ActionFromPolicy(action, state, time, false);
  return 0;
}
int mjpc_b200_batch_ilqg_planner_get_result(void* p, int problem, double* scalars, float* states, float* actions,
                                            double* times) {
  BatchILQGPlanner* bp = ilqg_problem_of(p, problem);
  if (!bp) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_ilqg_planner_get_result(mjpc_b200_host::ToHandle(&bp->problem(problem)), scalars, states, actions,
                                           times);
}

}  // extern "C"
