// TEST INFRASTRUCTURE - CPU oracle (see oracle/model.h header).
// capi.cc: plain-C entry points so tests/ and bench.py's cpu_baseline can drive the oracle through
// ctypes.  All array arguments are double regardless of the oracle's compute precision
// (precision 64 = semantics reference, 32 = same arithmetic width as the CUDA kernels).
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "ilqg.h"
#include "rollout.h"
#include "threadpool.h"

using namespace oracle;

namespace {

template <class T>
struct Engine {
  Model<T> model;
  CostSpec<T> cost;
  std::vector<std::unique_ptr<Data<T>>> data;  // one per worker (Planner::ResizeMjData, planners/planner.cc:23-33)
  std::unique_ptr<ThreadPool> pool;
  XfrcNoise noise;                              // applied by rollout_spline / rollout_feedback when std > 0
  std::vector<double> solimp0;                  // the blob's solimp[0] values (oracle_set_differentiable)
  Engine(const void* blob, size_t n) : model(blob, n), cost(model) {}
  void resize(int nthreads) {
    if (!pool || pool->NumThreads() != nthreads) pool.reset(new ThreadPool(nthreads));
    while ((int)data.size() < nthreads) data.emplace_back(new Data<T>(model));
  }
};

struct Handle {
  int precision;
  std::unique_ptr<Engine<double>> e64;
  std::unique_ptr<Engine<float>> e32;
};

template <class T> std::vector<T> conv(const double* p, size_t n) {
  std::vector<T> v(n);
  for (size_t i = 0; i < n; i++) v[i] = (T)p[i];
  return v;
}

template <class T>
void set_task(Engine<T>& e, const double* weight, const double* parameters, const double* task_state, double risk) {
  if (weight) for (size_t i = 0; i < e.cost.weight.size(); i++) e.model.weight[i] = e.cost.weight[i] = (T)weight[i];
  if (parameters) for (size_t i = 0; i < e.model.parameters.size(); i++) e.model.parameters[i] = (T)parameters[i];
  if (task_state) for (size_t i = 0; i < e.model.task_state.size(); i++) e.model.task_state[i] = (T)task_state[i];
  e.model.risk = e.cost.risk = (T)risk;
}

template <class T>
void copy_out(const Trajectory<T>& tr, int H, int i, int ds, int nu, int nr, int ntr, double* states, double* actions,
              double* times, double* residual, double* costs, double* trace) {
  if (states) for (int k = 0; k < H * ds; k++) states[(size_t)i * H * ds + k] = tr.states[k];
  if (actions) for (int k = 0; k < H * nu; k++) actions[(size_t)i * H * nu + k] = tr.actions[k];
  if (times) for (int k = 0; k < H; k++) times[(size_t)i * H + k] = tr.times[k];
  if (residual) for (int k = 0; k < H * nr; k++) residual[(size_t)i * H * nr + k] = tr.residual[k];
  if (costs) for (int k = 0; k < H; k++) costs[(size_t)i * H + k] = tr.costs[k];
  if (trace) for (int k = 0; k < H * ntr; k++) trace[(size_t)i * H * ntr + k] = tr.trace[k];
}

// SamplingPlanner::Rollouts (planners/sampling/planner.cc:355-393) with injected candidate knots
template <class T>
int rollout_spline(Engine<T>& e, const double* state, double time, const double* mocap, const double* userdata,
                   const double* knots, const double* knot_times, int interp, int P, int N, int H, int nthreads,
                   double* returns, uint8_t* failure, double* states, double* actions, double* times,
                   double* residual, double* costs, double* trace) {
  const Model<T>& m = e.model;
  int ds = m.nq + m.nv + m.na, nu = m.nu, nr = m.num_residual, ntr = 3 * m.num_trace;
  e.resize(nthreads);
  auto st = conv<T>(state, ds);
  auto mc = conv<T>(mocap, 7 * m.nmocap);
  auto ud = conv<T>(userdata, m.nuserdata);
  auto kn = conv<T>(knots, (size_t)N * P * nu);
  auto kt = conv<T>(knot_times, P);
  std::vector<Trajectory<T>> trs(N);
  int before = e.pool->GetCount();
  for (int i = 0; i < N; i++) {
    e.pool->Schedule([&, i]() {
      Trajectory<T>& tr = trs[i];
      tr.Initialize(ds, nu, nr, m.num_trace, H);
      tr.Allocate(H);
      Data<T>& d = *e.data[ThreadPool::WorkerId()];
      auto pol = spline_policy<T>(m, kn.data() + (size_t)i * P * nu, kt.data(), P, interp);
      XfrcNoise nz = e.noise; nz.stream = (uint32_t)i;
      rollout<T>(tr, pol, m, e.cost, d, st.data(), (T)time, mc.data(), ud.data(), H, nz);
    });
  }
  e.pool->WaitCount(before + N);
  e.pool->ResetCount();
  for (int i = 0; i < N; i++) {
    returns[i] = trs[i].total_return;
    failure[i] = trs[i].failure;
    copy_out(trs[i], H, i, ds, nu, nr, ntr, states, actions, times, residual, costs, trace);
  }
  return 0;
}

// K line-search rollouts with the iLQG policy (ilqg/planner.cc:630-724)
template <class T>
int rollout_feedback(Engine<T>& e, const double* state, double time, const double* mocap, const double* userdata,
                     const double* u_nom, const double* x_nom, const double* t_nom, const double* gains,
                     const double* du, const double* step_sizes, int mode, int K, int H, int nthreads,
                     double* returns, uint8_t* failure, double* states, double* actions, double* times,
                     double* residual, double* costs, double* trace) {
  const Model<T>& m = e.model;
  int ds = m.nq + m.nv + m.na, nu = m.nu, nr = m.num_residual, ntr = 3 * m.num_trace, n = 2 * m.nv + m.na;
  e.resize(nthreads);
  auto st = conv<T>(state, ds);
  auto mc = conv<T>(mocap, 7 * m.nmocap);
  auto ud = conv<T>(userdata, m.nuserdata);
  ILQGPolicyData<T> pd;
  pd.H = H;
  pd.u = conv<T>(u_nom, (size_t)H * nu); pd.x = conv<T>(x_nom, (size_t)H * ds); pd.t = conv<T>(t_nom, H);
  pd.K = conv<T>(gains, (size_t)H * nu * n);
  pd.du = du ? conv<T>(du, (size_t)H * nu) : std::vector<T>((size_t)H * nu, 0);
  std::vector<Trajectory<T>> trs(K);
  int before = e.pool->GetCount();
  for (int i = 0; i < K; i++) {
    e.pool->Schedule([&, i]() {
      Trajectory<T>& tr = trs[i];
      tr.Initialize(ds, nu, nr, m.num_trace, H);
      tr.Allocate(H);
      Data<T>& d = *e.data[ThreadPool::WorkerId()];
      auto pol = ilqg_policy<T>(m, pd, (T)step_sizes[i], mode);
      rollout<T>(tr, pol, m, e.cost, d, st.data(), (T)time, mc.data(), ud.data(), H);
    });
  }
  e.pool->WaitCount(before + K);
  e.pool->ResetCount();
  for (int i = 0; i < K; i++) {
    returns[i] = trs[i].total_return;
    failure[i] = trs[i].failure;
    copy_out(trs[i], H, i, ds, nu, nr, ntr, states, actions, times, residual, costs, trace);
  }
  return 0;
}

// one mj_forward at (qpos, qvel, ctrl): exposes internals for per-stage parity tests
template <class T>
int forward_debug(Engine<T>& e, const double* qpos, const double* qvel, const double* ctrl, const double* mocap,
                  double time, const double* warmstart, double* qacc, double* qM, double* qfrc_bias,
                  double* qfrc_smooth_out, double* residual, double* efc_force, int* nefc, int* ncon, int* niter,
                  double* xpos, double* subtree_com, double* contact_out, double* qfrc_constraint,
                  double* next_qpos, double* next_qvel) {
  const Model<T>& m = e.model;
  e.resize(1);
  Data<T>& d = *e.data[0];
  for (int i = 0; i < m.nq; i++) d.qpos[i] = (T)qpos[i];
  for (int i = 0; i < m.nv; i++) d.qvel[i] = (T)qvel[i];
  for (int i = 0; i < m.nu; i++) d.ctrl[i] = (T)ctrl[i];
  for (int i = 0; i < m.nmocap; i++) {
    for (int c = 0; c < 3; c++) d.mocap_pos[3 * i + c] = (T)mocap[7 * i + c];
    for (int c = 0; c < 4; c++) d.mocap_quat[4 * i + c] = (T)mocap[7 * i + 3 + c];
  }
  for (int i = 0; i < m.nv; i++) d.qacc_warmstart[i] = warmstart ? (T)warmstart[i] : 0;
  d.time = (T)time;
  d.warning = false;
  forward<T>(m, d, residual_by_id<T>(m.residual_id));
  for (int i = 0; i < m.nv; i++) {
    qacc[i] = d.qacc[i]; qfrc_bias[i] = d.qfrc_bias[i]; qfrc_smooth_out[i] = d.qfrc_smooth[i];
    qfrc_constraint[i] = d.qfrc_constraint[i];
  }
  for (int i = 0; i < m.nv * m.nv; i++) qM[i] = d.qM[i];
  for (int i = 0; i < m.num_residual; i++) residual[i] = d.residual[i];
  for (int i = 0; i < d.nefc && i < 256; i++) efc_force[i] = d.efc_force[i];
  *nefc = d.nefc; *ncon = d.ncon; *niter = d.solver_niter;
  for (int i = 0; i < 3 * m.nbody; i++) { xpos[i] = d.xpos[i]; subtree_com[i] = d.subtree_com[i]; }
  for (int i = 0; i < d.ncon && i < 64; i++) {
    contact_out[8 * i] = d.contact[i].dist;
    for (int c = 0; c < 3; c++) { contact_out[8 * i + 1 + c] = d.contact[i].pos[c]; contact_out[8 * i + 4 + c] = d.contact[i].frame[c]; }
    contact_out[8 * i + 7] = d.contact[i].dim;
  }
  d.qacc_warmstart = d.qacc;
  euler<T>(m, d);
  for (int i = 0; i < m.nq; i++) next_qpos[i] = d.qpos[i];
  for (int i = 0; i < m.nv; i++) next_qvel[i] = d.qvel[i];
  return d.warning ? 1 : 0;
}

// one mj_forward at (qpos, qvel, ctrl), then the constraint problem the solver was given and its answer: the
// independent restatement of the convex problem (tests/test_constraint_solve_cpu.py) reads these.  Rows past
// cap_efc and contacts past cap_con are not written (the counts are).
//   rows      [nefc]: J [nv], type, id, pos, margin, diagApprox, R, D, aref, force, state, frictionloss
//   contacts  [ncon]: efc_address, dim, geom1, geom2, mu, friction [5], frame [9], dist, pos [3]
//   counts    {nefc, ncon, niter, warning}
template <class T>
int forward_debug_efc(Engine<T>& e, const double* qpos, const double* qvel, const double* ctrl, const double* mocap,
                      double time, const double* warmstart, int cap_efc, int cap_con, double* qacc, double* qacc_smooth,
                      double* qfrc_smooth, double* qM, double* efc_J, int* efc_type, int* efc_id, double* efc_row,
                      int* con_int, double* con_real, int* counts) {
  const Model<T>& m = e.model;
  e.resize(1);
  Data<T>& d = *e.data[0];
  for (int i = 0; i < m.nq; i++) d.qpos[i] = (T)qpos[i];
  for (int i = 0; i < m.nv; i++) d.qvel[i] = (T)qvel[i];
  for (int i = 0; i < m.nu; i++) d.ctrl[i] = (T)ctrl[i];
  for (int i = 0; i < m.nmocap; i++) {
    for (int c = 0; c < 3; c++) d.mocap_pos[3 * i + c] = (T)mocap[7 * i + c];
    for (int c = 0; c < 4; c++) d.mocap_quat[4 * i + c] = (T)mocap[7 * i + 3 + c];
  }
  for (int i = 0; i < m.nv; i++) d.qacc_warmstart[i] = warmstart ? (T)warmstart[i] : 0;
  d.time = (T)time;
  d.warning = false;
  forward<T>(m, d, residual_by_id<T>(m.residual_id));
  const int nv = m.nv;
  for (int i = 0; i < nv; i++) { qacc[i] = d.qacc[i]; qacc_smooth[i] = d.qacc_smooth[i]; qfrc_smooth[i] = d.qfrc_smooth[i]; }
  for (int i = 0; i < nv * nv; i++) qM[i] = d.qM[i];
  for (int r = 0; r < d.nefc && r < cap_efc; r++) {
    for (int i = 0; i < nv; i++) efc_J[(size_t)r * nv + i] = d.efc_J[(size_t)r * nv + i];
    efc_type[r] = d.efc_type[r]; efc_id[r] = d.efc_id[r];
    const T row[10] = {d.efc_pos[r], d.efc_margin[r], d.efc_diagApprox[r], d.efc_R[r], d.efc_D[r], d.efc_aref[r],
                       d.efc_force[r], (T)d.efc_state[r], d.efc_frictionloss[r], d.efc_vel[r]};
    for (int k = 0; k < 10; k++) efc_row[10 * r + k] = row[k];
  }
  for (int ci = 0; ci < d.ncon && ci < cap_con; ci++) {
    const Contact<T>& c = d.contact[ci];
    con_int[4 * ci] = c.efc_address; con_int[4 * ci + 1] = c.dim; con_int[4 * ci + 2] = c.geom1; con_int[4 * ci + 3] = c.geom2;
    double* o = con_real + 19 * ci;
    o[0] = c.mu;
    for (int k = 0; k < 5; k++) o[1 + k] = c.friction[k];
    for (int k = 0; k < 9; k++) o[6 + k] = c.frame[k];
    o[15] = c.dist;
    for (int k = 0; k < 3; k++) o[16 + k] = c.pos[k];
  }
  counts[0] = d.nefc; counts[1] = d.ncon; counts[2] = d.solver_niter; counts[3] = d.warning ? 1 : 0;
  return d.warning ? 1 : 0;
}

// B independent single steps (mj_step, trajectory.cc:158) from given (qpos, qvel, ctrl, warm start, time): the CPU
// side of the teacher-forced per-step parity tests.  counts [B][4] = {ncon, nefc, Newton iterations, warning}.
template <class T>
int step_batch(Engine<T>& e, int B, const double* qpos, const double* qvel, const double* ctrl, const double* warmstart,
               const double* mocap, const double* times, int nthreads, double* qacc, double* next_qpos,
               double* next_qvel, double* residual, double* cost, int* counts) {
  const Model<T>& m = e.model;
  e.resize(nthreads);
  const int nq = m.nq, nv = m.nv, nu = m.nu, nr = m.num_residual;
  const int before = e.pool->GetCount();
  for (int w = 0; w < nthreads; w++) {
    e.pool->Schedule([&, w]() {
      Data<T>& d = *e.data[w];
      for (int b = w; b < B; b += nthreads) {
        for (int i = 0; i < nq; i++) d.qpos[i] = (T)qpos[(size_t)b * nq + i];
        for (int i = 0; i < nv; i++) d.qvel[i] = (T)qvel[(size_t)b * nv + i];
        for (int i = 0; i < nu; i++) d.ctrl[i] = (T)ctrl[(size_t)b * nu + i];
        for (int i = 0; i < m.nmocap; i++) {
          for (int c = 0; c < 3; c++) d.mocap_pos[3 * i + c] = (T)mocap[7 * i + c];
          for (int c = 0; c < 4; c++) d.mocap_quat[4 * i + c] = (T)mocap[7 * i + 3 + c];
        }
        for (int i = 0; i < nv; i++) d.qacc_warmstart[i] = warmstart ? (T)warmstart[(size_t)b * nv + i] : (T)0;
        std::fill(d.xfrc_applied.begin(), d.xfrc_applied.end(), (T)0);
        d.xfrc_active = false;
        d.time = (T)times[b];
        d.warning = false;
        forward<T>(m, d, residual_by_id<T>(m.residual_id));
        if (bad(d.qacc)) d.warning = true;
        if (qacc) for (int i = 0; i < nv; i++) qacc[(size_t)b * nv + i] = d.qacc[i];
        if (residual) for (int i = 0; i < nr; i++) residual[(size_t)b * nr + i] = d.residual[i];
        if (cost) cost[b] = CostValue(e.cost, d.residual.data());
        if (counts) { counts[4 * b] = d.ncon; counts[4 * b + 1] = d.nefc; counts[4 * b + 2] = d.solver_niter; counts[4 * b + 3] = d.warning; }
        d.qacc_warmstart = d.qacc;
        euler<T>(m, d);
        if (next_qpos) for (int i = 0; i < nq; i++) next_qpos[(size_t)b * nq + i] = d.qpos[i];
        if (next_qvel) for (int i = 0; i < nv; i++) next_qvel[(size_t)b * nv + i] = d.qvel[i];
      }
    });
  }
  e.pool->WaitCount(before + nthreads);
  e.pool->ResetCount();
  return 0;
}

}  // namespace

#define DISPATCH(h, call) ((h)->precision == 64 ? call(*(h)->e64) : call(*(h)->e32))

extern "C" {

void* oracle_create(const void* blob, size_t nbytes, int precision) {
  try {
    auto* h = new Handle;
    h->precision = precision;
    if (precision == 64) h->e64.reset(new Engine<double>(blob, nbytes));
    else h->e32.reset(new Engine<float>(blob, nbytes));
    return h;
  } catch (const std::exception&) {
    return nullptr;
  }
}
void oracle_destroy(void* hv) { delete (Handle*)hv; }
// MakeDifferentiable (mjpc/utilities.cc:60-75): solimp[0] = 0 for joints and geoms; on = 0 restores the blob's values
int oracle_set_differentiable(void* hv, int on) {
  Handle* h = (Handle*)hv;
  auto apply = [&](auto& e) {
    auto& m = e.model;
    if (e.solimp0.empty()) {
      for (int i = 0; i < m.njnt; i++) e.solimp0.push_back((double)m.jnt_solimp[5 * i]);
      for (int i = 0; i < m.ngeom; i++) e.solimp0.push_back((double)m.geom_solimp[5 * i]);
    }
    for (int i = 0; i < m.njnt; i++) m.jnt_solimp[5 * i] = on ? 0 : e.solimp0[i];
    for (int i = 0; i < m.ngeom; i++) m.geom_solimp[5 * i] = on ? 0 : e.solimp0[m.njnt + i];
  };
  if (h->precision == 64) apply(*h->e64); else apply(*h->e32);
  return 0;
}
int oracle_step_batch(void* hv, int B, const double* qpos, const double* qvel, const double* ctrl, const double* warmstart,
                      const double* mocap, const double* times, int nthreads, double* qacc, double* next_qpos,
                      double* next_qvel, double* residual, double* cost, int* counts) {
  Handle* h = (Handle*)hv;
#define CALL(e) step_batch(e, B, qpos, qvel, ctrl, warmstart, mocap, times, nthreads, qacc, next_qpos, next_qvel, residual, cost, counts)
  return DISPATCH(h, CALL);
#undef CALL
}
// diagnostics: Newton iterations per solve since the last reset (64 bins)
void oracle_solver_hist(long* out, int reset) {
  for (int i = 0; i < 64; i++) { out[i] = solver_hist()[i].load(); if (reset) solver_hist()[i] = 0; }
}

int oracle_set_task(void* hv, const double* weight, const double* parameters, const double* task_state, double risk) {
  auto* h = (Handle*)hv;
  if (h->precision == 64) set_task(*h->e64, weight, parameters, task_state, risk);
  else set_task(*h->e32, weight, parameters, task_state, risk);
  return 0;
}

int oracle_rollout_spline(void* hv, const double* state, double time, const double* mocap, const double* userdata,
                          const double* knots, const double* knot_times, int interp, int P, int N, int H,
                          int nthreads, double* returns, uint8_t* failure, double* states, double* actions,
                          double* times, double* residual, double* costs, double* trace) {
  auto* h = (Handle*)hv;
  if (h->precision == 64)
    return rollout_spline(*h->e64, state, time, mocap, userdata, knots, knot_times, interp, P, N, H, nthreads, returns,
                          failure, states, actions, times, residual, costs, trace);
  return rollout_spline(*h->e32, state, time, mocap, userdata, knots, knot_times, interp, P, N, H, nthreads, returns,
                        failure, states, actions, times, residual, costs, trace);
}

// iLQGPolicy::Action of the oracle (mode 0/1/2 time-indexed, feedback scaled by `step`), exported for the host-policy test
int oracle_ilqg_policy_action(void* hv, const double* u_nom, const double* x_nom, const double* t_nom, const double* gains,
                              int H, int mode, double step, const double* state, double time, double* action) {
  auto* h = (Handle*)hv;
  const Model<double>& m = h->e64->model;
  const int ds = m.nq + m.nv + m.na, nu = m.nu, n = 2 * m.nv + m.na;
  ILQGPolicyData<double> pd;
  pd.H = H;
  pd.u.assign(u_nom, u_nom + (size_t)H * nu); pd.x.assign(x_nom, x_nom + (size_t)H * ds); pd.t.assign(t_nom, t_nom + H);
  pd.K.assign(gains, gains + (size_t)H * nu * n); pd.du.assign((size_t)H * nu, 0.0);
  auto pol = ilqg_policy<double>(m, pd, step, mode);
  pol(action, state, time, 0);
  return 0;
}

// interpolation helpers of the iLQG policy (mjpc/utilities.cc:303-422), exported for the golden tests
void oracle_find_interval(const double* seq, double value, int length, int* bounds) {
  find_interval<double>(bounds, seq, value, length);
}
void oracle_interpolate(double* out, double x, const double* xs, const double* ys, int dim, int length, int rep) {
  interpolate<double>(out, x, xs, ys, dim, length, rep);
}

// NoisyRollout settings for the following rollout_spline calls (std 0 switches the noise off)
void oracle_set_xfrc_noise(void* hv, double std, double rate, uint32_t seed) {
  auto* h = (Handle*)hv;
  if (h->e64) { h->e64->noise.std = std; h->e64->noise.rate = rate; h->e64->noise.seed = seed; }
  if (h->e32) { h->e32->noise.std = std; h->e32->noise.rate = rate; h->e32->noise.seed = seed; }
}

int oracle_rollout_feedback(void* hv, const double* state, double time, const double* mocap, const double* userdata,
                            const double* u_nom, const double* x_nom, const double* t_nom, const double* gains,
                            const double* du, const double* step_sizes, int mode, int K, int H, int nthreads,
                            double* returns, uint8_t* failure, double* states, double* actions, double* times,
                            double* residual, double* costs, double* trace) {
  auto* h = (Handle*)hv;
  if (h->precision == 64)
    return rollout_feedback(*h->e64, state, time, mocap, userdata, u_nom, x_nom, t_nom, gains, du, step_sizes, mode,
                            K, H, nthreads, returns, failure, states, actions, times, residual, costs, trace);
  return rollout_feedback(*h->e32, state, time, mocap, userdata, u_nom, x_nom, t_nom, gains, du, step_sizes, mode, K,
                          H, nthreads, returns, failure, states, actions, times, residual, costs, trace);
}

int oracle_forward_debug(void* hv, const double* qpos, const double* qvel, const double* ctrl, const double* mocap,
                         double time, const double* warmstart, double* qacc, double* qM, double* qfrc_bias,
                         double* qfrc_smooth, double* residual, double* efc_force, int* nefc, int* ncon, int* niter,
                         double* xpos, double* subtree_com, double* contact_out, double* qfrc_constraint,
                         double* next_qpos, double* next_qvel) {
  auto* h = (Handle*)hv;
  if (h->precision == 64)
    return forward_debug(*h->e64, qpos, qvel, ctrl, mocap, time, warmstart, qacc, qM, qfrc_bias, qfrc_smooth, residual,
                         efc_force, nefc, ncon, niter, xpos, subtree_com, contact_out, qfrc_constraint, next_qpos,
                         next_qvel);
  return forward_debug(*h->e32, qpos, qvel, ctrl, mocap, time, warmstart, qacc, qM, qfrc_bias, qfrc_smooth, residual,
                       efc_force, nefc, ncon, niter, xpos, subtree_com, contact_out, qfrc_constraint, next_qpos,
                       next_qvel);
}

int oracle_forward_debug_efc(void* hv, const double* qpos, const double* qvel, const double* ctrl, const double* mocap,
                             double time, const double* warmstart, int cap_efc, int cap_con, double* qacc,
                             double* qacc_smooth, double* qfrc_smooth, double* qM, double* efc_J, int* efc_type,
                             int* efc_id, double* efc_row, int* con_int, double* con_real, int* counts) {
  auto* h = (Handle*)hv;
#define CALL(e) forward_debug_efc(e, qpos, qvel, ctrl, mocap, time, warmstart, cap_efc, cap_con, qacc, qacc_smooth, \
                                  qfrc_smooth, qM, efc_J, efc_type, efc_id, efc_row, con_int, con_real, counts)
  return DISPATCH(h, CALL);
#undef CALL
}

// ---- exact operation count of one spline rollout batch (instrumented scalar, oracle/counted.h)
// returns the number of arithmetic operations per simulated env-step averaged over the N x H batch
double oracle_count_flops(const void* blob, size_t nbytes, const double* state, double time, const double* mocap,
                          const double* knots, const double* knot_times, int interp, int P, int N, int H,
                          double* returns_out) {
  using T = Counted;
  Model<T> m(blob, nbytes);
  CostSpec<T> cost(m);
  Data<T> d(m);
  const int ds = m.nq + m.nv, nu = m.nu;
  std::vector<T> st(ds), mc(7 * m.nmocap), ud(m.nuserdata + 1), kt(P);
  for (int i = 0; i < ds; i++) st[i] = state[i];
  for (int i = 0; i < 7 * m.nmocap; i++) mc[i] = mocap[i];
  for (int i = 0; i < P; i++) kt[i] = knot_times[i];
  Counted::flops = 0;
  for (int i = 0; i < N; i++) {
    std::vector<T> kn((size_t)P * nu);
    for (size_t k = 0; k < kn.size(); k++) kn[k] = knots[(size_t)i * P * nu + k];
    Trajectory<T> tr;
    tr.Initialize(ds, nu, m.num_residual, m.num_trace, H);
    tr.Allocate(H);
    auto pol = spline_policy<T>(m, kn.data(), kt.data(), P, interp);
    rollout<T>(tr, pol, m, cost, d, st.data(), T(time), mc.data(), ud.data(), H);
    if (returns_out) returns_out[i] = (double)tr.total_return;
  }
  return (double)Counted::flops / ((double)N * H);
}

// ---- stand-alone pieces pinned against the reference's known-answer tests
double oracle_norm(double* g, double* H, const double* x, const double* params, int n, int type) {
  return Norm<double>(g, H, x, params, n, type);
}
void oracle_spline_sample(double* out, const double* times, const double* values, int P, int dim, int interp,
                          double time) {
  spline_sample<double>(out, times, values, P, dim, interp, time);
}
double oracle_cost_value(void* hv, const double* residual, double* terms) {
  auto* h = (Handle*)hv;
  if (h->precision != 64) return 0;
  if (terms) CostTerms(h->e64->cost, terms, residual, true);
  return CostValue(h->e64->cost, residual);
}

// ---- iLQG pieces (oracle/ilqg.h)
int oracle_model_derivatives(void* hv, const double* states, const double* actions, const double* times,
                             const double* mocap, int H, double tol, double* A, double* B, double* C, double* D, int skip,
                             int mode, int nthreads) {
  auto* h = (Handle*)hv;
  if (h->precision == 64) return model_derivatives(h->e64->model, states, actions, times, mocap, H, tol, A, B, C, D, skip, mode, nthreads);
  return model_derivatives(h->e32->model, states, actions, times, mocap, H, tol, A, B, C, D, skip, mode, nthreads);
}
int oracle_cost_derivatives(void* hv, const double* residual, const double* C, const double* D, int H, int n, int m,
                            double* cx, double* cu, double* cxx, double* cuu, double* cxu) {
  auto* h = (Handle*)hv;
  if (h->precision != 64) return -1;
  cost_derivatives<double>(h->e64->cost, residual, C, D, H, n, m, cx, cu, cxx, cuu, cxu);
  return 0;
}
int oracle_backward_pass(const double* A, const double* B, const double* cx, const double* cu, const double* cxx,
                         const double* cxu, const double* cuu, const double* actions, const double* ctrlrange,
                         int n, int m, int H, double mu, int reg_type, int limits, double* Vx, double* Vxx,
                         double* du, double* K, double* dV, double* Qx, double* Qu, double* Qxx, double* Qxu,
                         double* Quu) {
  return backward_pass<double>(A, B, cx, cu, cxx, cxu, cuu, actions, ctrlrange, n, m, H, mu, reg_type, limits, Vx,
                               Vxx, du, K, dV, Qx, Qu, Qxx, Qxu, Quu);
}

}  // extern "C"
