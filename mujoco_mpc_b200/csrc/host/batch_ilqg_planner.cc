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

void ILQGSweeps::Attach(mjpc_b200_t* gpu, int num_rollouts, int representation) {
  gpu_ = gpu; K_ = num_rollouts; representation_ = representation;
  mjpc_b200_info info;
  mjpc_b200_get_info(gpu_, &info);
  nu_ = info.nu; ds_ = info.dim_state; n_ = info.dim_dstate; nr_ = info.num_residual; nmocap7_ = 7 * info.nmocap;
}

// one rollout_feedback_batched launch of the candidate policies of ps, as each iLQGPlanner makes it
int ILQGSweeps::FeedbackLaunch(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                               int horizon, bool with_du, int mode) {
  const size_t H = horizon, J = ps.size();
  std::vector<int> idx(J);
  for (size_t j = 0; j < J; j++) idx[j] = (int)j;
  auto pl = [&](int j) -> iLQGPlanner& { return *ps[j]; };
  gather(st_, idx, ds_, [&](int j) { return pl(j).st_.data(); });
  gather(mc_, idx, nmocap7_, [&](int j) { return pl(j).mc_.data(); });
  gather(times_, idx, 1, [&](int j) { return &pl(j).time_; });
  gather(u_, idx, H * nu_, [&](int j) { return pl(j).c_actions_.data(); });
  gather(x_, idx, H * ds_, [&](int j) { return pl(j).c_states_.data(); });
  gather(t_, idx, H, [&](int j) { return pl(j).c_times_.data(); });
  gather(g_, idx, H * nu_ * n_, [&](int j) { return pl(j).c_gains_.data(); });
  if (with_du) gather(du_, idx, H * nu_, [&](int j) { return pl(j).c_du_.data(); });
  gather(steps_, idx, K_, [&](int j) { return pl(j).steps_.data(); });
  gather(w_, task, rows.nw, [&](int r) { return rows.w + (size_t)r * rows.nw; });
  gather(p_, task, rows.np, [&](int r) { return rows.p + (size_t)r * rows.np; });
  gather(ts_, task, rows.nts, [&](int r) { return rows.ts + (size_t)r * rows.nts; });
  ret_.resize(J * K_); fail_.resize(J * K_); order_.resize(J * K_);
  return mjpc_b200_rollout_feedback_batched(gpu_, (int)J, st_.data(), times_.data(), nmocap7_ ? mc_.data() : nullptr,
                                            rows.nw ? w_.data() : nullptr, rows.np ? p_.data() : nullptr,
                                            rows.nts ? ts_.data() : nullptr, u_.data(), x_.data(), t_.data(), g_.data(),
                                            with_du ? du_.data() : nullptr, steps_.data(), mode, K_, horizon,
                                            ret_.data(), fail_.data(), order_.data());
}

int ILQGSweeps::Nominal(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                        int horizon) {
  for (iLQGPlanner* p : ps)
    if (p->PrepareNominal(horizon)) return -1;
  if (FeedbackLaunch(ps, task, rows, horizon, false, representation_)) return -1;
  for (size_t j = 0; j < ps.size(); j++)
    if (ps[j]->InstallNominal(ret_.data() + j * K_, fail_.data() + j * K_, (int)j * K_) < 0) return -1;
  return 0;
}

int ILQGSweeps::Iterate(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                        int horizon, int* updated) {
  const int J = (int)ps.size();
  const size_t H = horizon, n = n_, m = nu_, nr = nr_;
  const iLQGSettings& settings = ps[0]->settings;
  std::vector<int> all(J);
  for (int j = 0; j < J; j++) {
    all[j] = j;
    if (updated) updated[j] = 0;
    if (ps[j]->PrepareIteration(horizon)) return -1;
  }
  auto pl = [&](int j) -> iLQGPlanner& { return *ps[j]; };
  // derivatives and cost derivatives of every problem (ModelDerivatives / CostDerivatives::Compute)
  gather(x_, all, H * ds_, [&](int j) { return pl(j).c_states_.data(); });
  gather(u_, all, H * m, [&](int j) { return pl(j).c_actions_.data(); });
  gather(t_, all, H, [&](int j) { return pl(j).c_times_.data(); });
  gather(mc_, all, nmocap7_, [&](int j) { return pl(j).mc_.data(); });
  gather(res_, all, H * nr, [&](int j) { return pl(j).c_residual_.data(); });
  gather(w_, task, rows.nw, [&](int r) { return rows.w + (size_t)r * rows.nw; });
  gather(p_, task, rows.np, [&](int r) { return rows.p + (size_t)r * rows.np; });
  gather(ts_, task, rows.nts, [&](int r) { return rows.ts + (size_t)r * rows.nts; });
  A_.resize(J * H * n * n); B_.resize(J * H * n * m); C_.resize(J * H * nr * n); D_.resize(J * H * nr * m);
  cx_.resize(J * H * n); cu_.resize(J * H * m); cxx_.resize(J * H * n * n); cuu_.resize(J * H * m * m);
  cxu_.resize(J * H * n * m);
  if (mjpc_b200_model_derivatives_batched(gpu_, J, x_.data(), u_.data(), t_.data(), nmocap7_ ? mc_.data() : nullptr,
                                          rows.nw ? w_.data() : nullptr, rows.np ? p_.data() : nullptr,
                                          rows.nts ? ts_.data() : nullptr, horizon, settings.derivative_skip,
                                          (float)settings.fd_tolerance, settings.fd_mode, A_.data(), B_.data(),
                                          C_.data(), D_.data()))
    return -1;
  if (mjpc_b200_cost_derivatives_batched(gpu_, J, rows.nw ? w_.data() : nullptr, res_.data(), C_.data(), D_.data(),
                                         horizon, cx_.data(), cu_.data(), cxx_.data(), cuu_.data(), cxu_.data()))
    return -1;
  // backward passes: round r holds the problems whose pass has not succeeded and whose retry budget is not spent,
  // each at its own regularisation - every problem follows its own iLQGPlanner retry loop
  status_.assign(J, 0);
  for (;;) {
    std::vector<int> act;
    for (int j = 0; j < J; j++) if (pl(j).BackwardPending(status_[j])) act.push_back(j);
    if (act.empty()) break;
    const size_t JA = act.size();
    auto row = [&](std::vector<float>& v, size_t per) { return [&v, per](int j) { return v.data() + (size_t)j * per; }; };
    gather(sA_, act, H * n * n, row(A_, H * n * n));
    gather(sB_, act, H * n * m, row(B_, H * n * m));
    gather(scx_, act, H * n, row(cx_, H * n));
    gather(scu_, act, H * m, row(cu_, H * m));
    gather(scxx_, act, H * n * n, row(cxx_, H * n * n));
    gather(scxu_, act, H * n * m, row(cxu_, H * n * m));
    gather(scuu_, act, H * m * m, row(cuu_, H * m * m));
    gather(sact_, act, H * m, [&](int j) { return pl(j).c_actions_.data(); });
    mu_.resize(JA);
    for (size_t a = 0; a < JA; a++) mu_[a] = (float)pl(act[a]).regularization;
    K_out_.resize(JA * H * m * n); du_out_.resize(JA * H * m); dV_out_.resize(2 * JA);
    std::vector<int> st(JA, 0);
    if (mjpc_b200_backward_pass_batched(gpu_, (int)JA, sA_.data(), sB_.data(), scx_.data(), scu_.data(), scxx_.data(),
                                        scxu_.data(), scuu_.data(), sact_.data(), horizon, mu_.data(),
                                        settings.regularization_type, settings.action_limits, K_out_.data(),
                                        du_out_.data(), dV_out_.data(), nullptr, nullptr, st.data()))
      return -1;
    for (size_t a = 0; a < JA; a++) {
      iLQGPlanner& p = pl(act[a]);
      std::copy(K_out_.begin() + a * H * m * n, K_out_.begin() + (a + 1) * H * m * n, p.Kbuf_.begin());
      std::copy(du_out_.begin() + a * H * m, du_out_.begin() + (a + 1) * H * m, p.dubuf_.begin());
      p.dV_[0] = dV_out_[2 * a]; p.dV_[1] = dV_out_[2 * a + 1];
      status_[act[a]] = st[a];
      p.AfterBackward(st[a]);
    }
  }
  // action rollouts of the problems whose backward pass succeeded; the others are left untouched
  std::vector<iLQGPlanner*> okp;
  std::vector<int> ok, okt;
  for (int j = 0; j < J; j++)
    if (pl(j).InstallGains(status_[j])) { ok.push_back(j); okp.push_back(ps[j]); okt.push_back(task[j]); }
  if (ok.empty()) return 0;
  if (FeedbackLaunch(okp, okt, rows, horizon, true, 3)) return -1;
  for (size_t j = 0; j < ok.size(); j++) {
    const int r = okp[j]->InstallActions(ret_.data() + j * K_, fail_.data() + j * K_, (int)j * K_);
    if (r < 0) return -1;
    if (updated) updated[ok[j]] = r;
  }
  return 0;
}

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
  if (int rc = mjpc_b200_create(model, num_problems * num_rollouts, max_horizon, device, &gpu_)) return rc;
  sweeps_.Attach(gpu_, num_rollouts, representation);
  for (int b = 0; b < num_problems; b++) {
    problems_.emplace_back(new iLQGPlanner);
    all_.push_back(problems_.back().get()); all_idx_.push_back(b);
    if (int rc = problems_.back()->Initialize(model, num_rollouts, representation, max_horizon, device, gpu_)) return rc;
  }
  return 0;
}

void BatchILQGPlanner::SetTask(int b, const double* weight, const double* parameters, const double* task_state) {
  if (weight) std::copy(weight, weight + nw_, weight_.begin() + (size_t)b * nw_);
  if (parameters) std::copy(parameters, parameters + np_, parameters_.begin() + (size_t)b * np_);
  if (task_state) std::copy(task_state, task_state + nts_, task_state_.begin() + (size_t)b * nts_);
}

TaskRows BatchILQGPlanner::Rows() const {
  TaskRows r;
  r.w = weight_.data(); r.p = parameters_.data(); r.ts = task_state_.data(); r.nw = nw_; r.np = np_; r.nts = nts_;
  return r;
}

int BatchILQGPlanner::Nominal(int horizon) {
  for (auto& p : problems_) p->settings = settings;
  return sweeps_.Nominal(all_, all_idx_, Rows(), horizon);
}

int BatchILQGPlanner::NominalTrajectory(int horizon) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  return Nominal(horizon);
}

int BatchILQGPlanner::OptimizePolicy(int horizon, int* updated) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  if (Nominal(horizon)) return -1;
  return sweeps_.Iterate(all_, all_idx_, Rows(), horizon, updated);
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
