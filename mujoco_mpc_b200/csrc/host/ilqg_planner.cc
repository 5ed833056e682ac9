// ilqg_planner.cc - see ilqg_planner.h.  Reference: mjpc/planners/ilqg/planner.cc.
#include "ilqg_planner.h"

#include <algorithm>
#include <cmath>
#include <mutex>

#include "../dev_model.h"   // Blob reader (plain C++)

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
void SubQuat(double* res, const double* qa, const double* qb) {   // qb * quat(res) = qa  (mju_subQuat)
  const double n[4] = {qb[0], -qb[1], -qb[2], -qb[3]};
  const double d[4] = {n[0] * qa[0] - n[1] * qa[1] - n[2] * qa[2] - n[3] * qa[3],
                       n[0] * qa[1] + n[1] * qa[0] + n[2] * qa[3] - n[3] * qa[2],
                       n[0] * qa[2] - n[1] * qa[3] + n[2] * qa[0] + n[3] * qa[1],
                       n[0] * qa[3] + n[1] * qa[2] - n[2] * qa[1] + n[3] * qa[0]};
  double axis[3] = {d[1], d[2], d[3]};
  const double s = std::sqrt(axis[0] * axis[0] + axis[1] * axis[1] + axis[2] * axis[2]);
  if (s < 1e-15) { axis[0] = 1; axis[1] = axis[2] = 0; } else { for (double& a : axis) a /= s; }
  double speed = 2 * std::atan2(s, d[0]);
  if (speed > M_PI) speed -= 2 * M_PI;
  for (int c = 0; c < 3; c++) res[c] = axis[c] * speed;
}
}  // namespace

int iLQGPolicyModel::Load(const mjpc_model_blob* blob) {
  try {
    mjpc_dev::Blob b(blob->data, blob->nbytes);
    nq = b.i("nq"); nv = b.i("nv"); nu = b.i("nu");
    jnt_type = b.ints("jnt_type"); jnt_qposadr = b.ints("jnt_qposadr"); jnt_dofadr = b.ints("jnt_dofadr");
    ctrlrange = b.reals("actuator_ctrlrange");
  } catch (const std::exception&) {
    return MJPC_B200_ERR_BAD_BLOB;
  }
  return 0;
}

void iLQGPolicyAction(const iLQGPolicyModel& m, const float* u_nom, const float* x_nom, const double* t_nom,
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
    for (size_t j = 0; j < m.jnt_type.size(); j++) {
      const int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
      if (m.jnt_type[j] == 0) {
        for (int c = 0; c < 3; c++) dx[da + c] = state[qa + c] - xi[qa + c];
        SubQuat(&dx[da + 3], state + qa + 3, &xi[qa + 3]);
      } else if (m.jnt_type[j] == 1) {
        SubQuat(&dx[da], state + qa, &xi[qa]);
      } else {
        dx[da] = state[qa] - xi[qa];
      }
    }
    for (int i = 0; i < m.nv; i++) dx[m.nv + i] = state[m.nq + i] - xi[m.nq + i];
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
  ret_.assign(K_, 0.f); fail_.assign(K_, 0); order_.assign(K_, 0);
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
  if (ret != ret_.data()) std::copy(ret, ret + K_, ret_.begin());
  if (fail != fail_.data()) std::copy(fail, fail + K_, fail_.begin());
  const int best = BestRollout(ret_.data(), fail_.data(), K_);
  if (best == -1) { feedback_scaling = 0.0; return 0; }   // candidate_policy[0] keeps the live trajectory (:203-211)
  if (FetchCandidate(cand0 + best, ret_[best])) return -1;
  feedback_scaling = steps_[best];
  return 1;
}

int iLQGPlanner::NominalTrajectory(int horizon) {
  if (PrepareNominal(horizon)) return -1;
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  const int rc = mjpc_b200_rollout_feedback(gpu_, st_.data(), time_, mc_.empty() ? nullptr : mc_.data(), nullptr, c_actions_.data(),
                                            c_states_.data(), c_times_.data(), c_gains_.data(), nullptr, steps_.data(),
                                            representation_, K_, horizon, ret_.data(), fail_.data(), order_.data());
  if (rc) return -1;
  return InstallNominal(ret_.data(), fail_.data(), 0);
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
  const size_t H = horizon, n = n_, m = nu_, nr = nr_;
  iter_H_ = horizon;
  previous_return_ = c_return_;
  steps_ = StepSizes();
  A_.resize(H * n * n); B_.resize(H * n * m); C_.resize(H * nr * n); D_.resize(H * nr * m);
  cx_.resize(H * n); cu_.resize(H * m); cxx_.resize(H * n * n); cuu_.resize(H * m * m); cxu_.resize(H * n * m);
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
  if (ret != ret_.data()) std::copy(ret, ret + K_, ret_.begin());
  if (fail != fail_.data()) std::copy(fail, fail + K_, fail_.begin());
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

int iLQGPlanner::Iteration(int horizon) {
  if (PrepareIteration(horizon)) return -1;
  const DifferentiableScope diff(gpu_, settings.differentiable != 0);
  const float* mc = mc_.empty() ? nullptr : mc_.data();
  if (mjpc_b200_model_derivatives(gpu_, c_states_.data(), c_actions_.data(), c_times_.data(), mc, horizon,
                                  settings.derivative_skip, (float)settings.fd_tolerance, settings.fd_mode,
                                  A_.data(), B_.data(), C_.data(), D_.data()))
    return -1;
  if (mjpc_b200_cost_derivatives(gpu_, c_residual_.data(), C_.data(), D_.data(), horizon, cx_.data(), cu_.data(),
                                 cxx_.data(), cuu_.data(), cxu_.data()))
    return -1;
  int status = 0;
  while (BackwardPending(status)) {
    if (mjpc_b200_backward_pass(gpu_, A_.data(), B_.data(), cx_.data(), cu_.data(), cxx_.data(), cxu_.data(),
                                cuu_.data(), c_actions_.data(), horizon, (float)regularization, settings.regularization_type,
                                settings.action_limits, Kbuf_.data(), dubuf_.data(), dV_, nullptr, nullptr, &status))
      return -1;
    AfterBackward(status);
  }
  if (!InstallGains(status)) return 0;
  if (mjpc_b200_rollout_feedback(gpu_, st_.data(), time_, mc, nullptr, c_actions_.data(), c_states_.data(),
                                 c_times_.data(), c_gains_.data(), c_du_.data(), steps_.data(), 3, K_, horizon,
                                 ret_.data(), fail_.data(), order_.data()))
    return -1;
  return InstallActions(ret_.data(), fail_.data(), 0);
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
  if (NominalTrajectory(horizon) < 0) return -1;
  return Iteration(horizon);
}

void iLQGPlanner::ActionFromPolicy(double* action, const double* state, double time, bool) {
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  // the live policy's own feedback_scaling is always 1 (planner.cc:603)
  iLQGPolicyAction(pm_, actions.data(), states.data(), times.data(), gains.data(), live_H_, representation_, 1.0,
                   state, time, action);
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::iLQGPlanner;

extern "C" {

int mjpc_b200_ilqg_planner_create(const mjpc_model_blob* model, int num_rollouts, int representation, double fd_tolerance,
                                  int max_horizon, int device, void** out) {
  if (!model || !out || num_rollouts < 1 || max_horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new iLQGPlanner;
  int rc = p->Initialize(model, num_rollouts, representation, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  if (fd_tolerance > 0) p->settings.fd_tolerance = fd_tolerance;
  *out = p;
  return 0;
}
void mjpc_b200_ilqg_planner_destroy(void* p) { delete (iLQGPlanner*)p; }
void mjpc_b200_ilqg_planner_set_fd(void* p, double tolerance, int mode, int derivative_skip) {
  auto& s = ((iLQGPlanner*)p)->settings;
  if (tolerance > 0) s.fd_tolerance = tolerance;
  if (mode >= 0) s.fd_mode = mode ? 1 : 0;
  if (derivative_skip >= 0) s.derivative_skip = derivative_skip;
}
void mjpc_b200_ilqg_planner_reset(void* p, int horizon, const double* initial_repeated_action) {
  ((iLQGPlanner*)p)->Reset(horizon, initial_repeated_action);
}
void mjpc_b200_ilqg_planner_set_state(void* p, const double* state, double time, const double* mocap) {
  ((iLQGPlanner*)p)->SetState(state, time, mocap);
}
int mjpc_b200_ilqg_planner_nominal_trajectory(void* p, int horizon) { return ((iLQGPlanner*)p)->NominalTrajectory(horizon); }
int mjpc_b200_ilqg_planner_optimize_policy(void* p, int horizon) { return ((iLQGPlanner*)p)->OptimizePolicy(horizon); }
void mjpc_b200_ilqg_planner_action_from_policy(void* p, double* action, const double* state, double time) {
  ((iLQGPlanner*)p)->ActionFromPolicy(action, state, time, false);
}
// stateless form of iLQGPolicy::Action (host only, no device): u_nom [H][nu], x_nom [H][dim_state], t_nom [H],
// gains [H][nu][2nv]; state may be NULL (open loop)
int mjpc_b200_host_ilqg_policy_action(const mjpc_model_blob* model, const float* u_nom, const float* x_nom,
                                      const double* t_nom, const float* gains, int horizon, int representation,
                                      double feedback_scaling, const double* state, double time, double* action) {
  if (!model || !u_nom || !x_nom || !t_nom || !gains || !action || horizon < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  mjpc_b200_host::iLQGPolicyModel pm;
  if (int rc = pm.Load(model)) return rc;
  mjpc_b200_host::iLQGPolicyAction(pm, u_nom, x_nom, t_nom, gains, horizon, representation, feedback_scaling, state, time,
                                   action);
  return 0;
}
// scalars[6] = {total_return, regularization, improvement, expected, surprise, winner}; nominal states [H][dim_state],
// actions [H][nu], times [H]; any pointer may be NULL
int mjpc_b200_ilqg_planner_get_result(void* pv, double* scalars, float* states, float* actions, double* times) {
  auto* p = (iLQGPlanner*)pv;
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
