// planner.cc - see planner.h.
#include "planner.h"

#include <cmath>

#include <algorithm>

#include "../dev_model.h"   // Blob reader (plain C++)

namespace mjpc_b200_host {

namespace {
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

int HostModel::Load(const mjpc_model_blob* blob) {
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

void StateDiff(const HostModel& m, double* dx, const double* x_to, const double* x_from) {
  for (size_t j = 0; j < m.jnt_type.size(); j++) {
    const int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
    if (m.jnt_type[j] == 0) {
      for (int c = 0; c < 3; c++) dx[da + c] = x_to[qa + c] - x_from[qa + c];
      SubQuat(&dx[da + 3], x_to + qa + 3, &x_from[qa + 3]);
    } else if (m.jnt_type[j] == 1) {
      SubQuat(&dx[da], x_to + qa, &x_from[qa]);
    } else {
      dx[da] = x_to[qa] - x_from[qa];
    }
  }
  for (int i = 0; i < m.nv; i++) dx[m.nv + i] = x_to[m.nq + i] - x_from[m.nq + i];
}

void FindInterval(int* b, const double* seq, double value, int length) {
  int upper = 0;
  while (upper < length && !(value < seq[upper])) upper++;
  const int lower = upper - 1;
  if (lower < 0) b[0] = b[1] = 0;
  else if (lower > length - 1) b[0] = b[1] = length - 1;
  else { b[0] = std::max(lower, 0); b[1] = std::min(upper, length - 1); }
}

Planner::~Planner() {
  if (gpu_ && owns_gpu_) mjpc_b200_destroy(gpu_);
}

int Planner::AttachEngine(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                          mjpc_b200_t* borrowed) {
  owns_gpu_ = borrowed == nullptr;
  if (borrowed) gpu_ = borrowed;
  else if (int rc = mjpc_b200_create(model, max_candidates, max_horizon, device, &gpu_)) return rc;
  mjpc_b200_get_info(gpu_, &info_);
  state_.assign(info_.dim_state, 0.0); mocap_.assign(7 * info_.nmocap, 0.0);
  state_cov_.assign((size_t)info_.dim_dstate * info_.dim_dstate, 0.0);
  return 0;
}

int Planner::ModelEnsemble(const mjpc_model_blob* models, int K, int worst) {
  const bool set = K > 0 && models;
  if (set && state_members_) return MJPC_B200_ERR_UNSUPPORTED;
  if (int rc = mjpc_b200_set_model_ensemble(gpu_, models, K, worst)) return rc;
  model_ensemble_ = set;
  return 0;
}

int Planner::StateEnsemble(int K, int worst, uint32_t seed) {
  if (K < 0 || K > 32) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (K == 0) { state_members_ = state_worst_ = 0; return 0; }
  if (worst < 1 || worst > K) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (model_ensemble_) return MJPC_B200_ERR_UNSUPPORTED;
  state_members_ = K; state_worst_ = worst; state_seed_ = seed;
  return 0;
}

int Planner::StateCovariance(const double* covariance) {
  if (!covariance) { std::fill(state_cov_.begin(), state_cov_.end(), 0.0); return 0; }
  for (size_t e = 0; e < state_cov_.size(); e++)
    if (!std::isfinite(covariance[e])) return MJPC_B200_ERR_BAD_ARGUMENT;
  std::copy(covariance, covariance + state_cov_.size(), state_cov_.begin());
  return 0;
}

void Planner::SetState(const double* state, double time, const double* mocap) {
  std::copy(state, state + state_.size(), state_.begin());
  if (mocap && !mocap_.empty()) std::copy(mocap, mocap + mocap_.size(), mocap_.begin());
  time_ = time;
}

int SplineLaunch::Run(const std::vector<const Planner*>& from, const std::vector<const SplineCandidates*>& cands,
                      const TaskRows& rows, int horizon) {
  const size_t B = from.size(), N = cands[0]->N, P = cands[0]->P, nk = cands[0]->knots.size();   // nk = N P nu
  const int interp = cands[0]->interpolation;
  for (const SplineCandidates* c : cands)
    if (c->N != (int)N || c->P != (int)P || c->interpolation != interp) return MJPC_B200_ERR_BAD_ARGUMENT;
  const size_t ds = from[0]->state().size(), nm = from[0]->mocap().size();
  states_.resize(B * ds); mocaps_.resize(B * nm); times_.resize(B);
  knots_.resize(B * nk); knot_times_.resize(B * P);
  for (size_t b = 0; b < B; b++) {
    std::copy(cands[b]->knots.begin(), cands[b]->knots.begin() + nk, knots_.begin() + b * nk);
    std::copy(cands[b]->knot_times.begin(), cands[b]->knot_times.begin() + P, knot_times_.begin() + b * P);
    std::copy(from[b]->state().begin(), from[b]->state().end(), states_.begin() + b * ds);
    std::copy(from[b]->mocap().begin(), from[b]->mocap().end(), mocaps_.begin() + b * nm);
    times_[b] = from[b]->time();
  }
  returns.resize(B * N); failure.resize(B * N); order.resize(B * N);
  const Planner& p0 = *from[0];
  if (p0.state_members()) {   // problem b's members from planner b's covariance, the draws on problem 0's counter
    const size_t nn = p0.state_covariance().size();
    covariances_.resize(B * nn);
    for (size_t b = 0; b < B; b++)
      std::copy(from[b]->state_covariance().begin(), from[b]->state_covariance().end(), covariances_.begin() + b * nn);
    return mjpc_b200_rollout_spline_belief_batched(
        p0.gpu(), (int)B, p0.state_members(), p0.state_worst(), p0.state_seed(), p0.PlanIteration(), states_.data(),
        covariances_.data(), times_.data(), nm ? mocaps_.data() : nullptr, rows.nw ? rows.w : nullptr,
        rows.np ? rows.p : nullptr, rows.nts ? rows.ts : nullptr, knots_.data(), knot_times_.data(), interp, (int)P,
        (int)N, horizon, returns.data(), failure.data(), order.data());
  }
  return mjpc_b200_rollout_spline_batched(from[0]->gpu(), (int)B, states_.data(), times_.data(),
                                          nm ? mocaps_.data() : nullptr, rows.nw ? rows.w : nullptr,
                                          rows.np ? rows.p : nullptr, rows.nts ? rows.ts : nullptr, knots_.data(),
                                          knot_times_.data(), interp, (int)P, (int)N, horizon, returns.data(),
                                          failure.data(), order.data());
}

int Planner::FetchTrajectory(int candidate, int horizon, Trajectory* t) {
  const size_t H = horizon;
  t->horizon = horizon; t->dim_state = info_.dim_state; t->dim_action = info_.nu; t->dim_residual = info_.num_residual;
  t->dim_trace = 3 * info_.num_trace;
  t->states.resize(H * t->dim_state); t->actions.resize(H * t->dim_action); t->times.resize(H);
  t->residual.resize(H * t->dim_residual); t->costs.resize(H); t->trace.resize(H * t->dim_trace);
  return mjpc_b200_fetch_trajectory(gpu_, launch_offset_ + candidate, t->states.data(), t->actions.data(), t->times.data(),
                                    t->residual.data(), t->costs.data(), t->trace.data());
}

int CholFactor(double* M, int n, double mindiag) {
  int rank = 0;
  for (int j = 0; j < n; j++) {
    for (int k = 0; k < j; k++) M[(size_t)j * n + j] -= M[(size_t)j * n + k] * M[(size_t)j * n + k];
    double d = M[(size_t)j * n + j];
    if (d < mindiag) d = mindiag; else rank++;
    M[(size_t)j * n + j] = std::sqrt(d);
    for (int i = j + 1; i < n; i++) {
      for (int k = 0; k < j; k++) M[(size_t)i * n + j] -= M[(size_t)i * n + k] * M[(size_t)j * n + k];
      M[(size_t)i * n + j] /= M[(size_t)j * n + j];
    }
  }
  return rank;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
// (the generic planner family of include/mjpc_b200.h: every kind's handle, a NULL one refused)
using mjpc_b200_host::Planner;
using mjpc_b200_host::PlannerOf;

extern "C" {

int mjpc_b200_planner_destroy(mjpc_b200_planner_t* h) {
  Planner* p = PlannerOf<Planner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  delete p;
  return 0;
}
int mjpc_b200_planner_reset(mjpc_b200_planner_t* h, int horizon, const double* initial_repeated_action) {
  Planner* p = PlannerOf<Planner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  p->Reset(horizon, initial_repeated_action);
  return 0;
}
int mjpc_b200_planner_set_state(mjpc_b200_planner_t* h, const double* state, double time, const double* mocap) {
  Planner* p = PlannerOf<Planner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  p->SetState(state, time, mocap);
  return 0;
}
int mjpc_b200_planner_optimize_policy(mjpc_b200_planner_t* h, int horizon) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->OptimizePolicy(horizon) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_nominal_trajectory(mjpc_b200_planner_t* h, int horizon) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->NominalTrajectory(horizon) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_action_from_policy(mjpc_b200_planner_t* h, double* action, const double* state, double time,
                                         int use_previous) {
  Planner* p = PlannerOf<Planner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  p->ActionFromPolicy(action, state, time, use_previous != 0);
  return 0;
}
int mjpc_b200_planner_set_fd(mjpc_b200_planner_t* h, double tolerance, int mode, int derivative_skip) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->SetFD(tolerance, mode, derivative_skip) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_set_ensemble(mjpc_b200_planner_t* h, const mjpc_model_blob* models, int K, int worst) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->SetEnsemble(models, K, worst) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_set_state_ensemble(mjpc_b200_planner_t* h, int K, int worst, uint32_t seed) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->SetStateEnsemble(K, worst, seed) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_set_state_covariance(mjpc_b200_planner_t* h, const double* covariance) {
  Planner* p = PlannerOf<Planner>(h);
  return p ? p->SetStateCovariance(covariance) : MJPC_B200_ERR_BAD_ARGUMENT;
}
int mjpc_b200_planner_set_task(mjpc_b200_planner_t* h, const mjpc_task_desc* task) {
  Planner* p = PlannerOf<Planner>(h);
  if (!p || !task) return MJPC_B200_ERR_BAD_ARGUMENT;
  for (mjpc_b200_t* g : p->Handles())
    if (int rc = mjpc_b200_set_task(g, task)) return rc;
  return 0;
}

}  // extern "C"
