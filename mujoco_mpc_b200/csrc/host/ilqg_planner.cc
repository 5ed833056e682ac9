// ilqg_planner.cc - see ilqg_planner.h.  Reference: mjpc/planners/ilqg/planner.cc.
#include "ilqg_planner.h"

#include <algorithm>
#include <cmath>
#include <mutex>

namespace mjpc_b200_host {

// ------------------------------------------------------------------------------------------ iLQGPolicy::Action
namespace {
double FdSlope(double x, const double* xs, const float* ys, int dim, int length, int i) {   // utilities.cc:333-365
  int b[2];
  FindInterval(b, xs, x, length);
  auto Y = [&](int k) { return (double)ys[(size_t)dim * k + i]; };
  if (b[0] == 0 && b[1] == 0) return length > 2 ? (Y(b[1] + 1) - Y(b[1])) / (xs[b[1] + 1] - xs[b[1]]) : 0.0;
  if (b[0] == length - 1 && b[1] == length - 1) return length > 2 ? (Y(b[0]) - Y(b[0] - 1)) / (xs[b[0]] - xs[b[0] - 1]) : 0.0;
  if (b[0] == 0) return (Y(b[1]) - Y(b[0])) / (xs[b[1]] - xs[b[0]]);
  return 0.5 * (Y(b[1]) - Y(b[0])) / (xs[b[1]] - xs[b[0]]) + 0.5 * (Y(b[0]) - Y(b[0] - 1)) / (xs[b[0]] - xs[b[0] - 1]);
}
void Interpolate(double* out, double x, const double* xs, const float* ys, int dim, int length, int rep) {
  int b[2];
  FindInterval(b, xs, x, length);
  if (rep == 0 || b[0] == b[1]) { for (int i = 0; i < dim; i++) out[i] = ys[(size_t)dim * b[0] + i]; return; }
  const double t = (x - xs[b[0]]) / (xs[b[1]] - xs[b[0]]);
  if (rep == 1) {
    for (int i = 0; i < dim; i++) out[i] = ys[(size_t)dim * b[0] + i] * (1 - t) + ys[(size_t)dim * b[1] + i] * t;
    return;
  }
  const double dt = xs[b[1]] - xs[b[0]];
  const double c0 = 2 * t * t * t - 3 * t * t + 1, c1 = (t * t * t - 2 * t * t + t) * dt, c2 = -2 * t * t * t + 3 * t * t,
               c3 = (t * t * t - t * t) * dt;
  for (int i = 0; i < dim; i++)
    out[i] = c0 * ys[(size_t)b[0] * dim + i] + c1 * FdSlope(xs[b[0]], xs, ys, dim, length, i) +
             c2 * ys[(size_t)b[1] * dim + i] + c3 * FdSlope(xs[b[1]], xs, ys, dim, length, i);
}
void NormalizeQuat(double* q) {
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < 1e-15) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  for (int k = 0; k < 4; k++) q[k] /= n;
}
}  // namespace

void iLQGPolicyAction(const HostModel& m, const float* u_nom, const float* x_nom, const double* t_nom,
                      const float* gains, int H, int representation, double feedback_scaling, const double* state,
                      double time, double* action) {
  const int ds = m.nq + m.nv, n = 2 * m.nv, nu = m.nu;
  int b[2];
  FindInterval(b, t_nom, time, H);
  const int rep = (b[0] == b[1]) ? 0 : representation;
  Interpolate(action, time, t_nom, u_nom, nu, H - 1, rep);
  if (state) {
    std::vector<double> xi(ds), K((size_t)nu * n), dx(n);
    Interpolate(xi.data(), time, t_nom, x_nom, ds, H, rep);
    if (rep != 0)
      for (size_t j = 0; j < m.jnt_type.size(); j++) {
        if (m.jnt_type[j] == 0) NormalizeQuat(&xi[m.jnt_qposadr[j] + 3]);
        else if (m.jnt_type[j] == 1) NormalizeQuat(&xi[m.jnt_qposadr[j]]);
      }
    Interpolate(K.data(), time, t_nom, gains, nu * n, H - 1, rep);
    // StateDiff(model, dx, x_interp, state, 1): tangent-space difference state (-) x_interp
    StateDiff(m, dx.data(), state, xi.data());
    for (int i = 0; i < nu; i++) {
      double a = 0;
      for (int j = 0; j < n; j++) a += K[(size_t)i * n + j] * dx[j];
      action[i] += feedback_scaling * a;
    }
  }
  for (int i = 0; i < nu; i++) action[i] = std::max(m.ctrlrange[2 * i], std::min(m.ctrlrange[2 * i + 1], action[i]));
}

int iLQGPlanner::Initialize(const mjpc_model_blob* model, int num_rollouts, int representation, int max_horizon, int device,
                            mjpc_b200_t* borrowed) {
  K_ = std::max(num_rollouts, 1);
  if (int rc = AttachEngine(model, K_, max_horizon, device, borrowed)) return rc;
  nu_ = info_.nu; ds_ = info_.dim_state; n_ = info_.dim_dstate; nr_ = info_.num_residual;
  Hmax_ = info_.max_horizon;
  representation_ = representation;
  if (int prc = pm_.Load(model)) return prc;
  Reset(max_horizon, nullptr);
  return 0;
}

// all trajectory-shaped buffers are allocated at max_horizon once (the reference allocates kMaxTrajectoryHorizon):
// a later call with a larger horizon <= max_horizon never reads past the end
void iLQGPlanner::Reset(int horizon, const double* a) {
  H_ = live_H_ = std::min(std::max(horizon, 1), Hmax_);
  const size_t H = Hmax_;
  const std::unique_lock<std::shared_mutex> lock(mtx_);
  states.assign(H * ds_, 0.f); times.assign(H, 0.0); residual.assign(H * nr_, 0.f);
  actions.assign(H * nu_, 0.f);
  if (a) for (size_t t = 0; t < H; t++) for (int i = 0; i < nu_; i++) actions[t * nu_ + i] = (float)a[i];
  gains.assign(H * nu_ * n_, 0.f); du.assign(H * nu_, 0.f);
  c_states_ = states; c_actions_ = actions; c_times_ = times; c_residual_ = residual; c_gains_ = gains; c_du_ = du;
  total_return = c_return_ = 0; regularization = 1.0; regularization_rate = 1.0; regularization_factor = 2.0;
  feedback_scaling = 1.0; winner = 0; improvement = expected = surprise = 0;
  ret_.assign(K_, 0.f); fail_.assign(K_, 0);
}

std::vector<float> iLQGPlanner::StepSizes() const {
  std::vector<float> s(K_, 0.f);
  const int steps = K_ - 1;
  if (steps > 0) {
    std::vector<double> d(steps);
    LogScale(d.data(), 1.0, settings.min_linesearch_step, steps);
    for (int i = 0; i < steps; i++) s[i] = (float)d[i];
  }
  s[K_ - 1] = 0.f;
  return s;
}

int iLQGPlanner::BestRollout(const float* ret, const uint8_t* fail, int K) {
  int best = -1;
  float best_ret = 0;
  for (int j = K - 1; j >= 0; j--) {
    if (fail[j]) continue;
    if (best == -1 || ret[j] < best_ret) { best_ret = ret[j]; best = j; }
  }
  return best;
}

// candidate_policy[0].trajectory = trajectory[candidate] (planner.cc:214,560): the first H rows of the working copy
int iLQGPlanner::FetchCandidate(int candidate, double ret) {
  if (FetchTrajectory(candidate, H_, &best_)) return -1;
  std::copy(best_.states.begin(), best_.states.end(), c_states_.begin());
  std::copy(best_.actions.begin(), best_.actions.end(), c_actions_.begin());
  std::copy(best_.times.begin(), best_.times.end(), c_times_.begin());
  std::copy(best_.residual.begin(), best_.residual.end(), c_residual_.begin());
  c_return_ = ret;
  best_.total_return = ret; best_.failure = false;
  return 0;
}

// planner.cc:167-223.  Works on candidate_policy[0] (a copy of the live policy); the live policy - what
// ActionFromPolicy evaluates concurrently - is not touched.  `feedback_scaling` is the winning line-search scale
// (a planner diagnostic, planner.cc:217); the live policy keeps its own feedback_scaling of 1.
int iLQGPlanner::PrepareNominal(int horizon) {
  if (horizon < 1 || horizon > Hmax_) return -1;
  H_ = horizon;
  steps_ = StepSizes();
  st_.assign(state_.begin(), state_.end()); mc_.assign(mocap_.begin(), mocap_.end());
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  c_states_ = states; c_actions_ = actions; c_times_ = times; c_residual_ = residual; c_gains_ = gains; c_du_ = du;
  c_return_ = total_return;
  return 0;
}

// ret / fail: this problem's K rollouts, the first of which has the flat index cand0 in the last launch
int iLQGPlanner::InstallNominal(const float* ret, const uint8_t* fail, int cand0) {
  std::copy(ret, ret + K_, ret_.begin());
  std::copy(fail, fail + K_, fail_.begin());
  const int best = BestRollout(ret_.data(), fail_.data(), K_);
  if (best == -1) { feedback_scaling = 0.0; return 0; }   // candidate_policy[0] keeps the live trajectory (:203-211)
  if (FetchCandidate(cand0 + best, ret_[best])) return -1;
  feedback_scaling = steps_[best];
  return 1;
}

int iLQGPlanner::NominalTrajectory(int horizon) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  int found = 0;
  return sweeps_.Nominal({this}, {0}, TaskRows(), horizon, &found) ? -1 : found;
}

void iLQGPlanner::ScaleRegularization(double factor) {
  if (factor > 1) regularization_rate = std::max(regularization_rate * factor, factor);
  else regularization_rate = std::min(regularization_rate * factor, factor);
  regularization = std::min(std::max(regularization * regularization_rate, settings.min_regularization),
                            settings.max_regularization);
}

void iLQGPlanner::UpdateRegularization(double z, double s) {
  const double f = regularization_factor;
  if (!(std::isfinite(z) && std::isfinite(s))) ScaleRegularization(f * f);
  else if (z > 0.5 || s > 0.3) ScaleRegularization(1.0 / f);
  else if (z < 0.1 || s < 0.06) ScaleRegularization(f);
}

int iLQGPlanner::PrepareIteration(int horizon) {
  if (horizon < 2 || horizon > Hmax_) return -1;
  const size_t H = horizon, n = n_, m = nu_;
  iter_H_ = horizon;
  previous_return_ = c_return_;
  steps_ = StepSizes();
  Kbuf_.resize(H * m * n); dubuf_.resize(H * m);
  st_.assign(state_.begin(), state_.end()); mc_.assign(mocap_.begin(), mocap_.end());
  reg_iter_ = 0;
  dV_[0] = dV_[1] = 0;
  return 0;
}

// one step of the regularisation retry loop (planner.cc:429-520) after a backward pass with `status`
void iLQGPlanner::AfterBackward(int status) {
  if (status == 0 && regularization <= settings.max_regularization) {
    ScaleRegularization(regularization_factor);
    reg_iter_++;
  }
}

// false: backward-pass failure, the live policy is untouched (planner.cc:523-531).  Otherwise candidate_policy[j] =
// candidate_policy[0] with the new gains / improvement (:536-540): staged, not published
bool iLQGPlanner::InstallGains(int status) {
  if (status == 0) return false;
  std::copy(Kbuf_.begin(), Kbuf_.end(), c_gains_.begin());
  std::copy(dubuf_.begin(), dubuf_.end(), c_du_.begin());
  return true;
}

int iLQGPlanner::InstallActions(const float* ret, const uint8_t* fail, int cand0) {
  const size_t H = iter_H_, m = nu_, n = n_, nr = nr_;
  std::copy(ret, ret + K_, ret_.begin());
  std::copy(fail, fail + K_, fail_.begin());
  const int best = BestRollout(ret_.data(), fail_.data(), K_);
  if (best == -1) return 0;    // every rollout failed: nothing is published (:548-550)
  winner = best;
  const double action_step = steps_[best];
  // policy.CopyFrom(candidate_policy[winner]) (:597-605).  ActionRollouts left candidate j's nominal ACTIONS at
  // old + step_j * du with the OLD nominal states (:639-643); only candidate 0's trajectory was then replaced by the
  // winning rollout (:560) - restated literally: the closed-loop trajectory is published only when the winner is 0.
  std::vector<float> old_actions(c_actions_.begin(), c_actions_.begin() + H * m);
  std::vector<float> old_states(c_states_.begin(), c_states_.begin() + H * ds_), old_residual(c_residual_.begin(), c_residual_.begin() + H * nr);
  std::vector<double> old_times(c_times_.begin(), c_times_.begin() + H);
  if (FetchCandidate(cand0 + best, ret_[best])) return -1;      // candidate_policy[0].trajectory = trajectory[winner]
  expected = -1.0 * action_step * ((double)dV_[0] + action_step * (double)dV_[1]) + 1.0e-16;
  improvement = previous_return_ - c_return_;
  surprise = std::min(std::max(0.0, improvement / expected), 2.0);
  UpdateRegularization(surprise, action_step);
  {
    const std::unique_lock<std::shared_mutex> lock(mtx_);
    if (best == 0) {
      std::copy(c_states_.begin(), c_states_.begin() + H * ds_, states.begin());
      std::copy(c_actions_.begin(), c_actions_.begin() + H * m, actions.begin());
      std::copy(c_times_.begin(), c_times_.begin() + H, times.begin());
      std::copy(c_residual_.begin(), c_residual_.begin() + H * nr, residual.begin());
    } else {
      std::copy(old_states.begin(), old_states.end(), states.begin());
      for (size_t k = 0; k < H * m; k++) actions[k] = old_actions[k] + (float)action_step * c_du_[k];
      std::copy(old_times.begin(), old_times.end(), times.begin());
      std::copy(old_residual.begin(), old_residual.end(), residual.begin());
    }
    std::copy(c_gains_.begin(), c_gains_.begin() + H * m * n, gains.begin());
    std::copy(c_du_.begin(), c_du_.begin() + H * m, du.begin());
    total_return = c_return_;
    live_H_ = iter_H_;
  }
  return 1;
}

void iLQGPlanner::SetCandidateTrajectory(const Trajectory& tr) {
  const size_t H = std::min<size_t>(tr.horizon, Hmax_);
  H_ = (int)H;
  std::copy(tr.states.begin(), tr.states.begin() + H * ds_, c_states_.begin());
  std::copy(tr.actions.begin(), tr.actions.begin() + H * nu_, c_actions_.begin());
  std::copy(tr.times.begin(), tr.times.begin() + H, c_times_.begin());
  std::copy(tr.residual.begin(), tr.residual.begin() + H * nr_, c_residual_.begin());
  c_return_ = tr.total_return;
}

int iLQGPlanner::OptimizePolicy(int horizon) {
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  int updated = 0;
  if (sweeps_.Nominal({this}, {0}, TaskRows(), horizon, nullptr) ||
      sweeps_.Iterate({this}, {0}, TaskRows(), horizon, &updated))
    return -1;
  return updated;
}

void iLQGPlanner::ActionFromPolicy(double* action, const double* state, double time, bool) {
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  // the live policy's own feedback_scaling is always 1 (planner.cc:603)
  iLQGPolicyAction(pm_, actions.data(), states.data(), times.data(), gains.data(), live_H_, representation_, 1.0,
                   state, time, action);
}

// ------------------------------------------------------------------------------------------ ILQGSweeps
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

// one rollout_feedback_batched launch of the candidate policies of ps, as each iLQGPlanner makes it
int ILQGSweeps::FeedbackLaunch(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                               int horizon, bool with_du, int mode) {
  const iLQGPlanner& p0 = *ps[0];
  const size_t H = horizon, J = ps.size(), K = p0.K_, ds = p0.ds_, nu = p0.nu_, n = p0.n_, nm = p0.mocap_.size();
  std::vector<int> idx(J);
  for (size_t j = 0; j < J; j++) idx[j] = (int)j;
  auto pl = [&](int j) -> iLQGPlanner& { return *ps[j]; };
  gather(st_, idx, ds, [&](int j) { return pl(j).st_.data(); });
  gather(mc_, idx, nm, [&](int j) { return pl(j).mc_.data(); });
  gather(times_, idx, 1, [&](int j) { return &pl(j).time_; });
  gather(u_, idx, H * nu, [&](int j) { return pl(j).c_actions_.data(); });
  gather(x_, idx, H * ds, [&](int j) { return pl(j).c_states_.data(); });
  gather(t_, idx, H, [&](int j) { return pl(j).c_times_.data(); });
  gather(g_, idx, H * nu * n, [&](int j) { return pl(j).c_gains_.data(); });
  if (with_du) gather(du_, idx, H * nu, [&](int j) { return pl(j).c_du_.data(); });
  gather(steps_, idx, K, [&](int j) { return pl(j).steps_.data(); });
  gather(w_, task, rows.nw, [&](int r) { return rows.w + (size_t)r * rows.nw; });
  gather(p_, task, rows.np, [&](int r) { return rows.p + (size_t)r * rows.np; });
  gather(ts_, task, rows.nts, [&](int r) { return rows.ts + (size_t)r * rows.nts; });
  ret_.resize(J * K); fail_.resize(J * K); order_.resize(J * K);
  // with model variants, sweep problem j runs on the variant of the problem it plans (its task row)
  if (int rc = mjpc_b200_select_model_variants(p0.gpu_, task.data(), (int)J)) return rc;
  return mjpc_b200_rollout_feedback_batched(p0.gpu_, (int)J, st_.data(), times_.data(), nm ? mc_.data() : nullptr,
                                            rows.nw ? w_.data() : nullptr, rows.np ? p_.data() : nullptr,
                                            rows.nts ? ts_.data() : nullptr, u_.data(), x_.data(), t_.data(), g_.data(),
                                            with_du ? du_.data() : nullptr, steps_.data(), mode, (int)K, horizon,
                                            ret_.data(), fail_.data(), order_.data());
}

int ILQGSweeps::Nominal(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                        int horizon, int* found) {
  for (iLQGPlanner* p : ps)
    if (p->PrepareNominal(horizon)) return -1;
  if (FeedbackLaunch(ps, task, rows, horizon, false, ps[0]->representation_)) return -1;
  const int K = ps[0]->K_;
  for (size_t j = 0; j < ps.size(); j++) {
    const int r = ps[j]->InstallNominal(ret_.data() + j * K, fail_.data() + j * K, (int)j * K);
    if (r < 0) return -1;
    if (found) found[j] = r;
  }
  return 0;
}

int ILQGSweeps::Iterate(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                        int horizon, int* updated) {
  const int J = (int)ps.size();
  const iLQGPlanner& p0 = *ps[0];
  const iLQGSettings& settings = p0.settings;
  const size_t H = horizon, n = p0.n_, m = p0.nu_, nr = p0.nr_, ds = p0.ds_, nm = p0.mocap_.size();
  std::vector<int> all(J);
  for (int j = 0; j < J; j++) {
    all[j] = j;
    if (updated) updated[j] = 0;
    if (ps[j]->PrepareIteration(horizon)) return -1;
  }
  auto pl = [&](int j) -> iLQGPlanner& { return *ps[j]; };
  // derivatives and cost derivatives of every problem (ModelDerivatives / CostDerivatives::Compute)
  gather(x_, all, H * ds, [&](int j) { return pl(j).c_states_.data(); });
  gather(u_, all, H * m, [&](int j) { return pl(j).c_actions_.data(); });
  gather(t_, all, H, [&](int j) { return pl(j).c_times_.data(); });
  gather(mc_, all, nm, [&](int j) { return pl(j).mc_.data(); });
  gather(res_, all, H * nr, [&](int j) { return pl(j).c_residual_.data(); });
  gather(w_, task, rows.nw, [&](int r) { return rows.w + (size_t)r * rows.nw; });
  gather(p_, task, rows.np, [&](int r) { return rows.p + (size_t)r * rows.np; });
  gather(ts_, task, rows.nts, [&](int r) { return rows.ts + (size_t)r * rows.nts; });
  A_.resize(J * H * n * n); B_.resize(J * H * n * m); C_.resize(J * H * nr * n); D_.resize(J * H * nr * m);
  cx_.resize(J * H * n); cu_.resize(J * H * m); cxx_.resize(J * H * n * n); cuu_.resize(J * H * m * m);
  cxu_.resize(J * H * n * m);
  if (mjpc_b200_select_model_variants(p0.gpu_, task.data(), J) ||
      mjpc_b200_model_derivatives_batched(p0.gpu_, J, x_.data(), u_.data(), t_.data(), nm ? mc_.data() : nullptr,
                                          rows.nw ? w_.data() : nullptr, rows.np ? p_.data() : nullptr,
                                          rows.nts ? ts_.data() : nullptr, horizon, settings.derivative_skip,
                                          (float)settings.fd_tolerance, settings.fd_mode, A_.data(), B_.data(),
                                          C_.data(), D_.data()))
    return -1;
  if (mjpc_b200_cost_derivatives_batched(p0.gpu_, J, rows.nw ? w_.data() : nullptr, res_.data(), C_.data(), D_.data(),
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
    // the rows of the round's problems; when every problem is in the round they are the arrays themselves
    auto rows_of = [&](std::vector<float>& v, std::vector<float>& sub, size_t per) -> const float* {
      if (JA == (size_t)J) return v.data();
      gather(sub, act, per, [&v, per](int j) { return v.data() + (size_t)j * per; });
      return sub.data();
    };
    const float *rA = rows_of(A_, sA_, H * n * n), *rB = rows_of(B_, sB_, H * n * m), *rcx = rows_of(cx_, scx_, H * n),
                *rcu = rows_of(cu_, scu_, H * m), *rcxx = rows_of(cxx_, scxx_, H * n * n),
                *rcxu = rows_of(cxu_, scxu_, H * n * m), *rcuu = rows_of(cuu_, scuu_, H * m * m);
    gather(sact_, act, H * m, [&](int j) { return pl(j).c_actions_.data(); });
    mu_.resize(JA);
    for (size_t a = 0; a < JA; a++) mu_[a] = (float)pl(act[a]).regularization;
    K_out_.resize(JA * H * m * n); du_out_.resize(JA * H * m); dV_out_.resize(2 * JA);
    std::vector<int> st(JA, 0);
    if (mjpc_b200_backward_pass_batched(p0.gpu_, (int)JA, rA, rB, rcx, rcu, rcxx, rcxu, rcuu, sact_.data(), horizon,
                                        mu_.data(), settings.regularization_type, settings.action_limits,
                                        K_out_.data(), du_out_.data(), dV_out_.data(), nullptr, nullptr, st.data()))
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
  const int K = p0.K_;
  for (size_t j = 0; j < ok.size(); j++) {
    const int r = okp[j]->InstallActions(ret_.data() + j * K, fail_.data() + j * K, (int)j * K);
    if (r < 0) return -1;
    if (updated) updated[ok[j]] = r;
  }
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::iLQGPlanner;
using mjpc_b200_host::PlannerOf;

extern "C" {

int mjpc_b200_ilqg_planner_create(const mjpc_model_blob* model, int num_rollouts, int representation, double fd_tolerance,
                                  int max_horizon, int device, mjpc_b200_planner_t** out) {
  if (!model || !out || num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new iLQGPlanner;
  int rc = p->Initialize(model, num_rollouts, representation, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  p->SetFD(fd_tolerance, -1, -1);
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
// stateless form of iLQGPolicy::Action (host only, no device): u_nom [H][nu], x_nom [H][dim_state], t_nom [H],
// gains [H][nu][2nv]; state may be NULL (open loop)
int mjpc_b200_host_ilqg_policy_action(const mjpc_model_blob* model, const float* u_nom, const float* x_nom,
                                      const double* t_nom, const float* gains, int horizon, int representation,
                                      double feedback_scaling, const double* state, double time, double* action) {
  if (!model || !u_nom || !x_nom || !t_nom || !gains || !action || horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  mjpc_b200_host::HostModel pm;
  if (int rc = pm.Load(model)) return rc;
  mjpc_b200_host::iLQGPolicyAction(pm, u_nom, x_nom, t_nom, gains, horizon, representation, feedback_scaling, state, time,
                                   action);
  return 0;
}
// scalars[6] = {total_return, regularization, improvement, expected, surprise, winner}; nominal states [H][dim_state],
// actions [H][nu], times [H]; any pointer may be NULL
int mjpc_b200_ilqg_planner_get_result(mjpc_b200_planner_t* h, double* scalars, float* states, float* actions,
                                      double* times) {
  auto* p = PlannerOf<iLQGPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (scalars) {
    scalars[0] = p->total_return; scalars[1] = p->regularization; scalars[2] = p->improvement;
    scalars[3] = p->expected; scalars[4] = p->surprise; scalars[5] = p->winner;
  }
  const int H = p->horizon();
  if (states) std::copy(p->states.begin(), p->states.begin() + (size_t)H * p->dim_state(), states);
  if (actions) std::copy(p->actions.begin(), p->actions.begin() + (size_t)H * p->dim_action(), actions);
  if (times) std::copy(p->times.begin(), p->times.begin() + H, times);
  return H;
}

}  // extern "C"
