// TEST INFRASTRUCTURE - CPU oracle (see oracle/model.h header).
// rollout.h: Trajectory + the per-candidate rollout loops.
//   Trajectory fields / Reset      <- mjpc/trajectory.h:74-86, trajectory.cc:62-89
//   NoisyRollout (xfrc_std = 0)    <- mjpc/trajectory.cc:92-210   (time-indexed policy)
//   RolloutDiscrete                <- mjpc/trajectory.cc:213-309  (step-indexed policy)
//   UpdateReturn                   <- mjpc/trajectory.cc:312-326
//   GetTraces                      <- mjpc/utilities.cc:268-285
#pragma once
#include <cmath>
#include <cstdint>
#include <functional>
#include <vector>

#include "residuals.h"
#include "task.h"

namespace oracle {

constexpr double kMaxReturnValue = 1.0e6;  // trajectory.cc:29

template <class T>
struct Trajectory {
  int horizon = 0, dim_state = 0, dim_action = 0, dim_residual = 0, dim_trace = 0;
  std::vector<T> states, actions, times, residual, costs, trace;
  T total_return = 0;
  bool failure = false;

  void Initialize(int ds, int da, int dr, int num_trace, int H) {
    horizon = H; dim_state = ds; dim_action = da; dim_residual = dr; dim_trace = 3 * num_trace; failure = false;
  }
  void Allocate(int Tn) {
    states.assign(dim_state * Tn, 0); actions.assign(dim_action * Tn, 0); costs.assign(Tn, 0);
    residual.assign(dim_residual * Tn, 0); times.assign(Tn, 0); trace.assign(dim_trace * Tn, 0);
  }
  void Reset(int Tn, const T* initial_repeated_action) {
    std::fill(states.begin(), states.begin() + dim_state * Tn, (T)0);
    for (int i = 0; i < Tn; i++)
      for (int k = 0; k < dim_action; k++) actions[i * dim_action + k] = initial_repeated_action ? initial_repeated_action[k] : 0;
    std::fill(times.begin(), times.begin() + Tn, (T)0);
    std::fill(costs.begin(), costs.begin() + Tn, (T)0);
    std::fill(residual.begin(), residual.begin() + dim_residual * Tn, (T)0);
    std::fill(trace.begin(), trace.begin() + dim_trace * Tn, (T)0);
    total_return = 0; failure = false;
  }
};

template <class T>
void get_traces(T* out, const Model<T>& m, const Data<T>& d) {
  for (int k = 0; k < m.num_trace; k++) {
    int id = m.trace_objid[k];
    const T* src = m.trace_objtype[k] == OBJ_SITE ? &d.site_xpos[3 * id]
                   : m.trace_objtype[k] == OBJ_GEOM ? &d.geom_xpos[3 * id]
                   : m.trace_objtype[k] == OBJ_XBODY ? &d.xpos[3 * id] : &d.xipos[3 * id];
    for (int c = 0; c < 3; c++) out[3 * k + c] = src[c];
  }
}

template <class T>
void update_return(Trajectory<T>& tr, const CostSpec<T>& cost) {
  tr.total_return = 0;
  for (int t = 0; t < tr.horizon; t++) {
    tr.costs[t] = CostValue(cost, &tr.residual[t * tr.dim_residual]);
    tr.total_return += tr.costs[t];
  }
  tr.total_return /= (T)mm::max(tr.horizon, 1);
}

// policy(action, state, time, step_index)
template <class T> using Policy = std::function<void(T*, const T*, T, int)>;

// Injected noise source of NoisyRollout (the reference's absl::BitGen is unseedable): Philox4x32-10, key (seed, 1),
// counter (step, stream, element, 'XFRC'), Box-Muller on the first two words.  Same definition on the device.
inline void philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]}, k0 = key[0], k1 = key[1];
  for (int r = 0; r < 10; r++) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t n[4] = {(uint32_t)(p1 >> 32) ^ c[1] ^ k0, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c[3] ^ k1, (uint32_t)p0};
    for (int i = 0; i < 4; i++) c[i] = n[i];
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  for (int i = 0; i < 4; i++) out[i] = c[i];
}
inline double xfrc_normal(uint32_t seed, uint32_t step, uint32_t stream, uint32_t element) {
  const uint32_t ctr[4] = {step, stream, element, 0x58465243u}, key[2] = {seed, 1u};
  uint32_t r[4];
  philox4x32(ctr, key, r);
  const double u1 = ((double)r[0] + 0.5) / 4294967296.0, u2 = ((double)r[1] + 0.5) / 4294967296.0;
  return std::sqrt(-2.0 * std::log(u1)) * std::cos(2.0 * M_PI * u2);
}
struct XfrcNoise { double std = 0, rate = 1; uint32_t seed = 0, stream = 0; };

template <class T>
void rollout(Trajectory<T>& tr, const Policy<T>& policy, const Model<T>& m, const CostSpec<T>& cost, Data<T>& d,
             const T* state, T time, const T* mocap, const T* userdata, int steps, const XfrcNoise& noise = XfrcNoise()) {
  ResidualCallback<T> cb = residual_by_id<T>(m.residual_id);
  int nq = m.nq, nv = m.nv, nu = m.nu, ds = tr.dim_state, nr = tr.dim_residual;
  tr.failure = false;
  tr.horizon = steps;
  d.warning = false;
  for (int i = 0; i < m.nmocap; i++) {
    for (int c = 0; c < 3; c++) d.mocap_pos[3 * i + c] = mocap[7 * i + c];
    for (int c = 0; c < 4; c++) d.mocap_quat[4 * i + c] = mocap[7 * i + 3 + c];
  }
  for (int i = 0; i < m.nuserdata; i++) d.userdata[i] = userdata[i];
  for (int i = 0; i < ds; i++) tr.states[i] = state[i];
  for (int i = 0; i < nq; i++) d.qpos[i] = state[i];
  for (int i = 0; i < nv; i++) d.qvel[i] = state[nq + i];
  tr.times[0] = time;
  d.time = time;
  // the reference leaves mjData::qacc_warmstart as the worker thread last left it; we define it as zero
  std::fill(d.qacc_warmstart.begin(), d.qacc_warmstart.end(), (T)0);
  // ... and mjData::xfrc_applied likewise: defined as zero at the start of a noisy rollout
  std::fill(d.xfrc_applied.begin(), d.xfrc_applied.end(), (T)0);
  d.xfrc_active = noise.std > 0;
  for (int t = 0; t < steps - 1; t++) {
    policy(&tr.actions[t * nu], &tr.states[t * ds], d.time, t);
    for (int i = 0; i < nu; i++) d.ctrl[i] = tr.actions[t * nu + i];
    if (noise.std > 0) {   // Ornstein-Uhlenbeck perturbation in discrete time (trajectory.cc:147-155)
      // as 1 + expm1 and sqrt(-expm1), the device's ou_coefficients: 1 - rate^2 cancels in fp32 for rate >> timestep
      const T x = -m.timestep / (T)noise.rate;
      const T rate = 1 + mm::expm1(x);
      const T scale = (T)noise.std * mm::sqrt(-mm::expm1(2 * x));
      for (int i = 0; i < 6 * m.nbody; i++)
        d.xfrc_applied[i] = rate * d.xfrc_applied[i] + scale * (T)xfrc_normal(noise.seed, (uint32_t)t, noise.stream, (uint32_t)i);
    }
    step(m, d, cb);
    for (int i = 0; i < nr; i++) tr.residual[t * nr + i] = d.residual[i];
    get_traces(&tr.trace[t * tr.dim_trace], m, d);
    if (d.warning) { tr.failure = true; tr.total_return = (T)kMaxReturnValue; d.warning = false; return; }
    for (int i = 0; i < nq; i++) tr.states[(t + 1) * ds + i] = d.qpos[i];
    for (int i = 0; i < nv; i++) tr.states[(t + 1) * ds + nq + i] = d.qvel[i];
    tr.times[t + 1] = d.time;
  }
  if (steps > 1) for (int i = 0; i < nu; i++) tr.actions[(steps - 1) * nu + i] = tr.actions[(steps - 2) * nu + i];
  else for (int i = 0; i < nu; i++) tr.actions[i] = 0;
  forward(m, d, cb);
  for (int i = 0; i < nr; i++) tr.residual[(steps - 1) * nr + i] = d.residual[i];
  get_traces(&tr.trace[(steps - 1) * tr.dim_trace], m, d);
  if (d.warning) { tr.failure = true; tr.total_return = (T)kMaxReturnValue; d.warning = false; return; }
  update_return(tr, cost);
}

// SamplingPolicy::Action (sampling/policy.cc:52-59)
template <class T>
Policy<T> spline_policy(const Model<T>& m, const T* knots, const T* knot_times, int P, int interp) {
  return [&m, knots, knot_times, P, interp](T* action, const T*, T time, int) {
    spline_sample(action, knot_times, knots, P, m.nu, interp, time);
    clamp_ctrl(action, m.actuator_ctrlrange.data(), m.nu);
  };
}

// StateDiff (utilities.cc:543-553): ds = (s2 (-) s1) / h in the tangent space
template <class T>
void state_diff(const Model<T>& m, T* ds, const T* s1, const T* s2, T h) {
  int nq = m.nq, nv = m.nv;
  for (int j = 0; j < m.njnt; j++) {
    int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
    switch (m.jnt_type[j]) {
      case JNT_FREE:
        for (int c = 0; c < 3; c++) ds[da + c] = (s2[qa + c] - s1[qa + c]) / h;
        sub_quat(ds + da + 3, s2 + qa + 3, s1 + qa + 3);
        for (int c = 0; c < 3; c++) ds[da + 3 + c] /= h;
        break;
      case JNT_BALL:
        sub_quat(ds + da, s2 + qa, s1 + qa);
        for (int c = 0; c < 3; c++) ds[da + c] /= h;
        break;
      default: ds[da] = (s2[qa] - s1[qa]) / h;
    }
  }
  for (int i = 0; i < nv; i++) ds[nv + i] = (s2[nq + i] - s1[nq + i]) / h;
}

}  // namespace oracle
