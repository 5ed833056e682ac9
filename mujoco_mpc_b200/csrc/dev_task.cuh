// dev_task.cuh - task side of a rollout step on the device: policy evaluation, residual plug-ins, norms,
// cost.  Reference semantics:
//   spline policy      mjpc/planners/sampling/policy.cc:52-59, mjpc/spline/spline.cc:103-156,250-287
//   iLQG policy        mjpc/planners/ilqg/policy.cc:82-161, mjpc/planners/ilqg/planner.cc:630-692
//   residual registry  mjpc/tasks/tasks.cc:46-73 (Name() -> device function id)
//   quadruped residual mjpc/tasks/quadruped/quadruped.cc:33-226, 609-720; Ground mjpc/utilities.cc:556-574
//   norms / cost       mjpc/norm.cc:50-210, mjpc/task.cc:71-110
#pragma once
#include "dev_data.cuh"

namespace mjpc_dev {

enum { kNull = -1, kQuadratic = 0, kL22 = 1, kL2 = 2, kCosh = 3, kPowerLoss = 5, kSmoothAbsLoss = 6,
       kSmoothAbs2Loss = 7, kRectifyLoss = 8 };
// task_state / task_ids layouts (mujoco_mpc_b200/task.py)
enum { QS_MODE = 0, QS_MODE_START_TIME = 1, QS_POSITION = 2, QS_HEADING = 5, QS_SPEED = 7, QS_ANGVEL = 8, QS_GROUND = 9,
       QS_ORIENTATION = 10, QS_GAIT = 14, QS_PHASE_START = 15, QS_PHASE_START_TIME = 16, QS_PHASE_VELOCITY = 17,
       QS_JUMP_VEL = 18, QS_FLIGHT_TIME = 19, QS_JUMP_ACC = 20, QS_CROUCH_TIME = 21, QS_LEAP_TIME = 22,
       QS_JUMP_TIME = 23, QS_CROUCH_VEL = 24, QS_LAND_TIME = 25, QS_LAND_ACC = 26, QS_FLIGHT_ROT_VEL = 27,
       QS_JUMP_ROT_VEL = 28, QS_JUMP_ROT_ACC = 29, QS_LAND_ROT_ACC = 30 };
enum { QI_TORSO_BODY = 0, QI_HEAD_SITE = 1, QI_GOAL_MOCAP = 2, QI_FOOT_GEOM = 3, QI_PARAM_GAIT = 7,
       QI_PARAM_BIPED_TYPE = 8, QI_PARAM_CADENCE = 9, QI_PARAM_AMPLITUDE = 10, QI_PARAM_DUTY = 11,
       QI_PARAM_ARM_POSTURE = 12, QI_PARAM_HEADING = 13, QI_PARAM_FLIP_DIR = 14, QI_KEY_HOME = 15, QI_KEY_CROUCH = 16 };
enum { kModeQuadruped = 0, kModeBiped, kModeWalk, kModeScramble, kModeFlip };
enum { kFootFL = 0, kFootHL, kFootFR, kFootHR };

// ------------------------------------------------------------------------------------------ norms (value)
// Rectify: p * softplus(x / p), written so that no intermediate overflows.  log(1 + e^z) = max(z, 0) + log1p(e^-|z|);
// the naive form's e^z is inf in fp32 above z ~ 88.7 where the fp64 reference is still finite (e.g. p = 0.01, x = 1)
__device__ __forceinline__ float softplus_stable(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }

__device__ __forceinline__ float norm_value(const float* x, const float* params, int n, int type) {
  float y = 0;
  const float p = params[0], q = params[1];
  switch (type) {
    case kNull: y = x[0]; break;
    case kQuadratic:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += x[i] * x[i];
      y *= 0.5f;
      break;
    case kL22: {
      float cc = 0;
      MJPC_ROLL
      for (int i = 0; i < n; i++) cc += x[i] * x[i];
      const float a = powf(cc, q / 2) + powf(p, q);
      y = powf(a, 1 / q) - p;
      break;
    }
    case kL2: {
      float s = 0;
      MJPC_ROLL
      for (int i = 0; i < n; i++) s += x[i] * x[i];
      y = sqrtf(s + p * p) - p;
      break;
    }
    case kCosh:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += p * p * (coshf(x[i] / p) - 1);
      break;
    case kPowerLoss:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += powf(fabsf(x[i]), p);
      break;
    case kSmoothAbsLoss:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += sqrtf(x[i] * x[i] + p * p) - p;
      break;
    case kSmoothAbs2Loss:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += powf(powf(fabsf(x[i]), q) + powf(p, q), 1 / q) - p;
      break;
    case kRectifyLoss:
      MJPC_ROLL
      for (int i = 0; i < n; i++) y += p > 0 ? p * softplus_stable(x[i] / p) : fmaxf(x[i], 0.f);
      break;
  }
  return y;
}

// CostValue of the residual in shared memory; warp-uniform result. Terms are evaluated one per lane and
// summed in term order (same association as the scalar reference loop).
template <class SP>
__device__ __noinline__ float k_cost_value(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  const int *dimr = MI(task_dim_norm_residual), *ntype = MI(task_norm), *npar = MI(task_num_norm_parameter);
  const float *w = MF(task_weight), *prm = MF(task_norm_parameter), *res = DF(residual);
  float cost = 0;
  for (int base = 0; base < M.num_term; base += 32) {
    const int k = base + lane;
    float term = 0;
    if (k < M.num_term) {
      int f = 0, p = 0;
      MJPC_ROLL
      for (int q = 0; q < k; q++) { f += dimr[q]; p += npar[q]; }
      float pr[2] = {npar[k] > 0 ? prm[p] : 0.f, npar[k] > 1 ? prm[p + 1] : 0.f};
      term = w[k] * norm_value(res + f, pr, dimr[k], ntype[k]);
    }
    const int cnt = min(32, M.num_term - base);
    MJPC_ROLL
    for (int q = 0; q < cnt; q++) cost += __shfl_sync(kFull, term, q);
  }
  if (fabsf(CM(c).risk) < 1e-6f) return cost;
  // expm1f, not expf(.) - 1: near zero cost the difference cancels (fast-math expf is good to ~1e-7 absolute near 1,
  // an O(1) relative error once |risk * cost| ~ 1e-7).  -use_fast_math does not remap expm1f.
  return expm1f(CM(c).risk * cost) / CM(c).risk;
}

// ------------------------------------------------------------------------------------------ spline policy
__device__ __forceinline__ float spline_slope(const float* times, const float* values, int P, int dim, int node, int k) {
  if (node == 0) return (values[dim + k] - values[k]) / (times[1] - times[0]);
  if (node == P - 1) return (values[node * dim + k] - values[(node - 1) * dim + k]) / (times[node] - times[node - 1]);
  return 0.5f * (values[(node + 1) * dim + k] - values[node * dim + k]) / (times[node + 1] - times[node]) +
         0.5f * (values[node * dim + k] - values[(node - 1) * dim + k]) / (times[node] - times[node - 1]);
}
__device__ __forceinline__ float spline_sample1(const float* times, const float* values, int P, int dim, int interp,
                                                float time, int i) {
  if (P == 0) return 0.f;
  int upper = 0;
  while (upper < P && !(time < times[upper])) upper++;
  if (upper == P) return values[(P - 1) * dim + i];
  if (upper == 0) return values[i];
  const int lower = upper - 1;
  const float t = (time - times[lower]) / (times[upper] - times[lower]);
  if (interp == 0) return values[lower * dim + i];
  if (interp == 1) return values[lower * dim + i] * (1 - t) + values[upper * dim + i] * t;
  const float dt = times[upper] - times[lower];
  const float c0 = 2 * t * t * t - 3 * t * t + 1, c1 = (t * t * t - 2 * t * t + t) * dt, c2 = -2 * t * t * t + 3 * t * t,
              c3 = (t * t * t - t * t) * dt;
  const float p0 = values[lower * dim + i], p1 = values[upper * dim + i];
  const float m0 = spline_slope(times, values, P, dim, lower, i), m1 = spline_slope(times, values, P, dim, upper, i);
  return c0 * p0 + c1 * m0 + c2 * p1 + c3 * m1;
}
// ctrl <- clamp(spline(time)); one actuator per lane
// (out of line: the main warp and the task warp of a rollout CTA must evaluate it with the very same instructions)
template <class SP>
__device__ __noinline__ void k_policy_spline(Ctx& c, int P, int interp) {
  auto&& M = SP::model(c);
  const float* range = MF(actuator_ctrlrange);
  for (int i = c.lane; i < M.nu; i += 32) {
    float a = spline_sample1(DF(knot_times), DF(knots), P, M.nu, interp, c.time, i);
    DF(ctrl)[i] = fmaxf(range[2 * i], fminf(range[2 * i + 1], a));
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------ iLQG policy
// FindInterval (mjpc/utilities.h:125-144).  Rollout time is accumulated in fp32 on the device while the nominal
// times arrive as (double - time0): a sample that is meant to coincide with a node may land one ulp below it, which
// would shift a zero-order hold by a whole step.  Nodes within 1e-5 s above the query therefore count as reached.
__device__ __forceinline__ void find_interval(int* b, const float* seq, float value, int length) {
  int upper = 0;
  value += 1e-5f;
  while (upper < length && !(value < seq[upper])) upper++;
  const int lower = upper - 1;
  if (lower < 0) { b[0] = b[1] = 0; }
  else if (lower > length - 1) { b[0] = b[1] = length - 1; }
  else { b[0] = max(lower, 0); b[1] = min(upper, length - 1); }
}
__device__ __forceinline__ float fd_slope(float x, const float* xs, const float* ys, int dim, int length, int i) {
  int b[2];
  find_interval(b, xs, x, length);
  if (b[0] == 0 && b[1] == 0) {
    if (length > 2) return (ys[dim * (b[1] + 1) + i] - ys[dim * b[1] + i]) / (xs[b[1] + 1] - xs[b[1]]);
    return 0;
  } else if (b[0] == length - 1 && b[1] == length - 1) {
    if (length > 2) return (ys[dim * b[0] + i] - ys[dim * (b[0] - 1) + i]) / (xs[b[0]] - xs[b[0] - 1]);
    return 0;
  } else if (b[0] == 0) {
    return (ys[dim * b[1] + i] - ys[dim * b[0] + i]) / (xs[b[1]] - xs[b[0]]);
  }
  return 0.5f * (ys[dim * b[1] + i] - ys[dim * b[0] + i]) / (xs[b[1]] - xs[b[0]]) +
         0.5f * (ys[dim * b[0] + i] - ys[dim * (b[0] - 1) + i]) / (xs[b[0]] - xs[b[0] - 1]);
}
__device__ __forceinline__ float interp1(float x, const float* xs, const float* ys, int dim, int length, int rep, int i) {
  int b[2];
  find_interval(b, xs, x, length);
  if (rep == 0 || b[0] == b[1]) return ys[dim * b[0] + i];
  const float t = (x - xs[b[0]]) / (xs[b[1]] - xs[b[0]]);
  if (rep == 1) return ys[dim * b[0] + i] * (1 - t) + ys[dim * b[1] + i] * t;
  const float dt = xs[b[1]] - xs[b[0]];
  const float c0 = 2 * t * t * t - 3 * t * t + 1, c1 = (t * t * t - 2 * t * t + t) * dt, c2 = -2 * t * t * t + 3 * t * t,
              c3 = (t * t * t - t * t) * dt;
  const float p0 = ys[b[0] * dim + i], p1 = ys[b[1] * dim + i];
  return c0 * p0 + c1 * fd_slope(xs[b[0]], xs, ys, dim, length, i) + c2 * p1 + c3 * fd_slope(xs[b[1]], xs, ys, dim, length, i);
}
__device__ __forceinline__ void sub_quat(float* res, const float* qa, const float* qb) {
  float qneg[4] = {qb[0], -qb[1], -qb[2], -qb[3]}, qd[4];
  quat_mul(qd, qneg, qa);
  float axis[3] = {qd[1], qd[2], qd[3]};
  const float s = norm3(axis);
  if (s < kMinVal) { axis[0] = 1; axis[1] = axis[2] = 0; } else { axis[0] /= s; axis[1] /= s; axis[2] /= s; }
  float speed = 2 * atan2f(s, qd[0]);
  if (speed > 3.14159265358979323846f) speed -= 2 * 3.14159265358979323846f;
  for (int k = 0; k < 3; k++) res[k] = axis[k] * speed;
}

struct FeedbackArgs {
  const float* u_nom;   // [B][H][nu]
  const float* x_nom;   // [B][H][dim_state]
  const float* t_nom;   // [B][H] relative to the problem's rollout start
  const float* gains;   // [B][H][nu][n]
  const float* du;      // [B][H][nu] or nullptr
  int mode;             // 0/1/2 time-indexed, 3 step-indexed
  int H;
  int nper;             // candidates per problem: candidate `cand` follows problem cand / nper's policy
};

// ctrl <- clamp(u + scale * K * (x (-) x_nom)) with the policy of candidate `cand`'s problem; global-memory reads are
// lane-strided (coalesced).  The problem's slices are resolved here, from the candidate index the caller keeps live
// anyway, so the step loop of the rollout kernels holds no extra register for them.
template <class SP>
__device__ __noinline__ void k_policy_feedback(Ctx& c, const FeedbackArgs& fa, float step, int index, int cand) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nq = M.nq, nv = M.nv, nu = M.nu, ds = nq + nv, n = 2 * nv, H = fa.H;
  const size_t pH = (size_t)(cand / fa.nper) * H;
  const float* u_nom = fa.u_nom + pH * nu;
  const float* x_nom = fa.x_nom + pH * ds;
  const float* t_nom = fa.t_nom + pH;
  const float* gains = fa.gains + pH * nu * n;
  const float* du = fa.du ? fa.du + pH * nu : nullptr;
  float *xn = DF(xnom), *dx = DF(dx), *ctrl = DF(ctrl);
  int rep = 0;
  float scale = 1.f;
  if (fa.mode == 3) {
    for (int i = lane; i < ds; i += 32) xn[i] = x_nom[index * ds + i];
    for (int i = lane; i < nu; i += 32) ctrl[i] = u_nom[index * nu + i] + (du ? step * du[index * nu + i] : 0.f);
  } else {
    int b[2];
    find_interval(b, t_nom, c.time, H);
    rep = (b[0] == b[1]) ? 0 : fa.mode;
    for (int i = lane; i < ds; i += 32) xn[i] = interp1(c.time, t_nom, x_nom, ds, H, rep, i);
    for (int i = lane; i < nu; i += 32) ctrl[i] = interp1(c.time, t_nom, u_nom, nu, H - 1, rep, i);
    scale = step;
  }
  __syncwarp();
  // state difference in the tangent space (StateDiff, mjpc/utilities.cc:543-553)
  const int *jtype = MI(jnt_type), *jqadr = MI(jnt_qposadr), *jdadr = MI(jnt_dofadr);
  const float *qpos = DF(qpos), *qvel = DF(qvel);
  for (int j = lane; j < M.njnt; j += 32) {
    const int qa = jqadr[j], da = jdadr[j];
    const int t = jtype[j];
    if (t == JNT_FREE) {
      for (int k = 0; k < 3; k++) dx[da + k] = qpos[qa + k] - xn[qa + k];
      float qn[4] = {xn[qa + 3], xn[qa + 4], xn[qa + 5], xn[qa + 6]};
      if (rep != 0) quat_normalize(qn);
      sub_quat(dx + da + 3, qpos + qa + 3, qn);
    } else if (t == JNT_BALL) {
      float qn[4] = {xn[qa], xn[qa + 1], xn[qa + 2], xn[qa + 3]};
      if (rep != 0) quat_normalize(qn);
      sub_quat(dx + da, qpos + qa, qn);
    } else {
      dx[da] = qpos[qa] - xn[qa];
    }
  }
  for (int i = lane; i < nv; i += 32) dx[nv + i] = qvel[i] - xn[nq + i];
  __syncwarp();
  const float* range = MF(actuator_ctrlrange);
  for (int i = lane; i < nu; i += 32) {
    float a = 0;
    if (fa.mode == 3) {
      const float* K = gains + ((size_t)index * nu + i) * n;
      for (int j = 0; j < n; j++) a += K[j] * dx[j];
    } else {
      for (int j = 0; j < n; j++) a += interp1(c.time, t_nom, gains, nu * n, H - 1, rep, i * n + j) * dx[j];
    }
    const float u = ctrl[i] + scale * a;
    ctrl[i] = fmaxf(range[2 * i], fminf(range[2 * i + 1], u));
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------ ray casting
__device__ __forceinline__ float ray_geom(const float* gpos, const float* gmat, const float* size, int type,
                                          const float* pnt, const float* vec) {
  float dp[3] = {pnt[0] - gpos[0], pnt[1] - gpos[1], pnt[2] - gpos[2]};
  float lp[3], lv[3];
  rot_vec_T(lp, gmat, dp);
  rot_vec_T(lv, gmat, vec);
  if (type == GEOM_PLANE) {
    if (lv[2] > -kMinVal) return -1;
    const float x = -lp[2] / lv[2];
    if (x < 0) return -1;
    const float p0 = lp[0] + x * lv[0], p1 = lp[1] + x * lv[1];
    if ((size[0] <= 0 || fabsf(p0) <= size[0]) && (size[1] <= 0 || fabsf(p1) <= size[1])) return x;
    return -1;
  }
  if (type == GEOM_SPHERE) {
    const float a = dot3(lv, lv), b = dot3(lv, lp), cc = dot3(lp, lp) - size[0] * size[0];
    const float det = b * b - a * cc;
    if (det < 0 || a < kMinVal) return -1;
    const float sq = sqrtf(det);
    const float x0 = (-b - sq) / a, x1 = (-b + sq) / a;
    if (x0 >= 0) return x0;
    if (x1 >= 0) return x1;
    return -1;
  }
  if (type == GEOM_BOX) {
    float best = -1;
    for (int i = 0; i < 3; i++) {
      if (fabsf(lv[i]) <= kMinVal) continue;
      for (int s = -1; s <= 1; s += 2) {
        const float x = ((float)s * size[i] - lp[i]) / lv[i];
        if (x < 0) continue;
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
        const float q1 = lp[i1] + x * lv[i1], q2 = lp[i2] + x * lv[i2];
        if (fabsf(q1) <= size[i1] && fabsf(q2) <= size[i2] && (best < 0 || x < best)) best = x;
      }
    }
    return best;
  }
  return -1;
}
template <class SP>
__device__ __forceinline__ float ground_height(Ctx& c, const float* pos, bool* ok) {
  auto&& M = SP::model(c);
  const float down[3] = {0, 0, -1};
  const float query[3] = {pos[0], pos[1], pos[2] + 0.5f};
  const int *rg = MI(ray_geoms), *gtype = MI(geom_type);
  const float *gxpos = DF(geom_xpos), *gxmat = DF(geom_xmat), *gsize = MF(geom_size);
  float best = -1;
  for (int k = 0; k < M.nray; k++) {
    const int g = rg[k];
    const float x = ray_geom(gxpos + 3 * g, gxmat + 9 * g, gsize + 3 * g, gtype[g], query, down);
    if (x >= 0 && (best < 0 || x < best)) best = x;
  }
  if (best < 0) { *ok = false; return 0; }
  return pos[2] + 0.5f - best;
}

// ------------------------------------------------------------------------------------------ residuals
struct QuadrupedFn {
  const float* S;
  const int* I;
  const float* prm;
  __device__ float param(int qi) const { return prm[I[qi]]; }
  __device__ int mode() const { return (int)S[QS_MODE]; }
  __device__ float GetPhase(float time) const { return S[QS_PHASE_START] + (time - S[QS_PHASE_START_TIME]) * S[QS_PHASE_VELOCITY]; }
  __device__ int GetGait() const { return mode() == kModeBiped ? 2 : (int)S[QS_GAIT]; }
  __device__ float StepHeight(float time, float footphase, float duty_ratio) const {
    const float pi = 3.14159265358979323846f;
    float angle = fmodf(time + pi - footphase, 2 * pi) - pi;
    float value = 0;
    if (duty_ratio < 1) {
      angle *= 0.5f / (1 - duty_ratio);
      value = cosf(fmaxf(-pi / 2, fminf(pi / 2, angle)));
    }
    return fabsf(value) < 1e-6f ? 0.f : value;
  }
  __device__ float FootStepOne(float time, int gait, int f) const {
    const float kGaitPhase[5][4] = {{0, 0, 0, 0}, {0, 0.75f, 0.5f, 0.25f}, {0, 0.5f, 0.5f, 0},
                                    {0, 0.33f, 0.33f, 0.66f}, {0, 0.4f, 0.05f, 0.35f}};
    return param(QI_PARAM_AMPLITUDE) * StepHeight(time, 2 * 3.14159265358979323846f * kGaitPhase[gait][f], param(QI_PARAM_DUTY));
  }
  __device__ void Walk(float* pos, float time) const {
    const float* heading = S + QS_HEADING;
    const float* position = S + QS_POSITION;
    if (fabsf(S[QS_ANGVEL]) < 0.01f) {
      float fw[2] = {heading[0], heading[1]};
      const float n = sqrtf(fw[0] * fw[0] + fw[1] * fw[1]);
      if (n < kMinVal) { fw[0] = 1; fw[1] = 0; } else { fw[0] /= n; fw[1] /= n; }
      pos[0] = position[0] + heading[0] + time * S[QS_SPEED] * fw[0];
      pos[1] = position[1] + heading[1] + time * S[QS_SPEED] * fw[1];
    } else {
      const float angle = time * S[QS_ANGVEL];
      const float co = cosf(angle), s = sinf(angle);
      pos[0] = co * heading[0] - s * heading[1] + position[0];
      pos[1] = s * heading[0] + co * heading[1] + position[1];
    }
  }
  __device__ float FlipHeight(float time) const {
    const float kHeightQuadruped = 0.25f, kLeapHeight = 0.5f;
    const float jump = S[QS_JUMP_TIME], flight = S[QS_FLIGHT_TIME], land = S[QS_LAND_TIME];
    if (time >= jump + flight + land) return kHeightQuadruped + S[QS_GROUND];
    float h = 0;
    if (time < jump) {
      h = kHeightQuadruped + time * S[QS_CROUCH_VEL] + 0.5f * time * time * S[QS_JUMP_ACC];
    } else if (time >= jump && time < jump + flight) {
      time -= jump;
      h = kLeapHeight + S[QS_JUMP_VEL] * time - 0.5f * 9.81f * time * time;
    } else if (time >= jump + flight) {
      time -= jump + flight;
      h = kLeapHeight - S[QS_JUMP_VEL] * time + 0.5f * S[QS_LAND_ACC] * time * time;
    }
    return h + S[QS_GROUND];
  }
  __device__ void FlipQuat(float* quat, float time) const {
    const float pi = 3.14159265358979323846f;
    const float jump = S[QS_JUMP_TIME], flight = S[QS_FLIGHT_TIME], land = S[QS_LAND_TIME], crouch = S[QS_CROUCH_TIME];
    float angle = 0;
    if (time >= jump + flight + land) {
      angle = 2 * pi;
    } else if (time >= crouch && time < jump) {
      time -= crouch;
      angle = 0.5f * S[QS_JUMP_ROT_ACC] * time * time + S[QS_JUMP_ROT_VEL] * time;
    } else if (time >= jump && time < jump + flight) {
      time -= jump;
      angle = pi / 2 + S[QS_FLIGHT_ROT_VEL] * time;
    } else if (time >= jump + flight) {
      time -= jump + flight;
      angle = 1.75f * pi + S[QS_FLIGHT_ROT_VEL] * time - 0.5f * S[QS_LAND_ROT_ACC] * time * time;
    }
    const int flip_dir = (int)param(QI_PARAM_FLIP_DIR);
    float axis[3] = {0, flip_dir ? 1.f : -1.f, 0};
    float q[4];
    axis_angle_quat(q, axis, angle);
    quat_mul(quat, S + QS_ORIENTATION, q);
  }
};

template <class SP>
__device__ __noinline__ void k_residual_quadruped(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  QuadrupedFn fn{MF(task_state), MI(task_ids), MF(task_parameters)};
  const int* I = fn.I;
  const float* S = fn.S;
  float* residual = DF(residual);
  const float kHeightQuadruped = 0.25f, kHeightBiped = 0.6f, kFootRadius = 0.02f;
  const int cur = fn.mode();
  const float* gx = DF(geom_xpos);
  const float* foot_pos[4];
  for (int f = 0; f < 4; f++) foot_pos[f] = gx + 3 * I[QI_FOOT_GEOM + f];
  const int handstand_i = (int)fn.param(QI_PARAM_BIPED_TYPE);
  float avg[3];
  if (cur == kModeBiped) {
    const int a = handstand_i ? kFootFL : kFootHL, b = handstand_i ? kFootFR : kFootHR;
    for (int k = 0; k < 3; k++) avg[k] = 0.5f * (foot_pos[a][k] + foot_pos[b][k]);
  } else {
    for (int k = 0; k < 3; k++)
      avg[k] = 0.25f * (((foot_pos[kFootHL][k] + foot_pos[kFootHR][k]) + foot_pos[kFootFL][k]) + foot_pos[kFootFR][k]);
  }
  const int torso = I[QI_TORSO_BODY];
  const float* torso_xmat = DF(xmat) + 9 * torso;
  const float* goal_pos = DF(mocap_pos) + 3 * I[QI_GOAL_MOCAP];
  const float* compos = DF(subtree_com) + 3 * torso;
  const float* torso_pos = DF(xipos) + 3 * torso;
  const float* comvel = DF(subtree_linvel) + 3 * torso;
  const bool is_biped = cur == kModeBiped;
  const float height_goal = is_biped ? kHeightBiped : kHeightQuadruped;
  const float mode_time = c.time - S[QS_MODE_START_TIME];
  const int nu = M.nu;
  if (lane == 0) {
    int counter = 0;
    // Upright
    if (cur != kModeFlip) {
      if (cur == kModeBiped) residual[counter++] = torso_xmat[6] - (handstand_i ? -1 : 1);
      else residual[counter++] = torso_xmat[8] - 1;
      residual[counter++] = 0;
      residual[counter++] = 0;
    } else {
      float quat[4];
      fn.FlipQuat(quat, mode_time);
      sub_quat(residual + counter, DF(xquat) + 4 * torso, quat);
      counter += 3;
    }
    // Height
    if (cur == kModeScramble) residual[counter++] = 0;
    else if (cur == kModeFlip) residual[counter++] = torso_pos[2] - fn.FlipHeight(mode_time);
    else residual[counter++] = (torso_pos[2] - avg[2]) - height_goal;
    // Position
    const float* head = DF(site_xpos) + 3 * I[QI_HEAD_SITE];
    float target[3] = {goal_pos[0], goal_pos[1], goal_pos[2]};
    if (cur == kModeWalk) fn.Walk(target, mode_time);
    residual[counter++] = head[0] - target[0];
    residual[counter++] = head[1] - target[1];
    residual[counter++] = cur == kModeScramble ? 2 * (head[2] - target[2]) : 0.f;
    // Balance (after the 4 gait entries)
    const float fall_time = sqrtf(2 * height_goal / 9.81f);
    residual[11] = compos[0] + comvel[0] * fall_time - avg[0];
    residual[12] = compos[1] + comvel[1] * fall_time - avg[1];
    // Yaw + angular momentum (after effort and posture)
    float th[2] = {torso_xmat[0], torso_xmat[3]};
    if (cur == kModeBiped) {
      const int hs = handstand_i ? 1 : -1;
      th[0] = hs * torso_xmat[2];
      th[1] = hs * torso_xmat[5];
    }
    const float n = sqrtf(th[0] * th[0] + th[1] * th[1]);
    if (n < kMinVal) { th[0] = 1; th[1] = 0; } else { th[0] /= n; th[1] /= n; }
    const float heading_goal = fn.param(QI_PARAM_HEADING);
    const int yb = 13 + 2 * nu;
    residual[yb] = th[0] - cosf(heading_goal);
    residual[yb + 1] = th[1] - sinf(heading_goal);
    for (int k = 0; k < 3; k++) residual[yb + 2 + k] = comvel[k];
  }
  // Gait: one foot per lane (4 down-rays in parallel)
  bool ok = true;
  if (lane < 4) {
    const int f = lane;
    const int gait = fn.GetGait();
    const float step = fn.FootStepOne(fn.GetPhase(c.time), gait, f);
    bool skip = false;
    if (is_biped) {
      const bool front_hand = !handstand_i && (f == kFootFL || f == kFootFR);
      const bool back_hand = handstand_i && (f == kFootHL || f == kFootHR);
      skip = front_hand || back_hand;
    }
    float out = 0;
    if (!skip) {
      float query[3] = {foot_pos[f][0], foot_pos[f][1], foot_pos[f][2]};
      if (cur == kModeScramble) {
        float tg[3];
        for (int k = 0; k < 3; k++) tg[k] = goal_pos[k] - foot_pos[f][k];
        tg[2] = 0;
        normalize3(tg);
        for (int k = 0; k < 3; k++) query[k] += 0.15f * tg[k];
      }
      const float gh = ground_height<SP>(c, query, &ok);
      const float height_target = gh + kFootRadius + step;
      float hd = foot_pos[f][2] - height_target;
      if (cur == kModeScramble) hd = fminf(0.f, hd);
      out = step ? hd : 0.f;
    }
    residual[7 + f] = out;
  }
  if (__any_sync(kFull, !ok)) c.warn = 1;
  // Effort and Posture: one actuator per lane
  if (lane < nu) {
    const int i = lane;
    residual[13 + i] = 2e-2f * DF(actuator_force)[i];
    const float* home = MF(key_qpos) + M.nq * I[QI_KEY_HOME];
    float v = DF(qpos)[7 + i] - home[7 + i];
    if (cur == kModeFlip) {
      if (mode_time < S[QS_CROUCH_TIME]) {
        const float* crouch = MF(key_qpos) + M.nq * I[QI_KEY_CROUCH];
        v = DF(qpos)[7 + i] - crouch[7 + i];
      } else if (mode_time >= S[QS_CROUCH_TIME] && mode_time < S[QS_JUMP_TIME] + S[QS_FLIGHT_TIME]) {
        v = 0;
      }
    }
    const float gain = (i % 3 == 0) ? 2.f : 1.f;  // kJointPostureGain {2,1,1}
    v *= gain;
    if (cur == kModeBiped) {
      const float arm = fn.param(QI_PARAM_ARM_POSTURE);
      const int base = handstand_i ? 6 : 0;
      if (i >= base && i < base + 6) v *= arm;
    }
    residual[13 + nu + i] = v;
  }
  __syncwarp();
}

template <class SP>
__device__ __noinline__ void k_residual(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  float* r = DF(residual);
  switch (M.residual_id) {
    case RESIDUAL_PARTICLE:
      for (int i = lane; i < M.nq; i += 32) r[i] = DF(qpos)[i] - (i < 2 ? DF(mocap_pos)[i] : 0.f);
      for (int i = lane; i < M.nv; i += 32) r[2 + i] = DF(qvel)[i];
      __syncwarp();
      break;
    case RESIDUAL_PARTICLE_COPY:
      for (int i = lane; i < M.nq; i += 32) r[i] = DF(qpos)[i];
      for (int i = lane; i < M.nv; i += 32) r[M.nq + i] = DF(qvel)[i];
      __syncwarp();
      break;
    case RESIDUAL_CARTPOLE:
      if (lane == 0) {
        r[0] = cosf(DF(qpos)[1]) - 1;
        r[1] = DF(qpos)[0] - MF(task_parameters)[0];
        r[2] = DF(qvel)[1];
        r[3] = DF(ctrl)[0];
      }
      __syncwarp();
      break;
    case RESIDUAL_QUADRUPED_FLAT: k_residual_quadruped<SP>(c); break;
    case RESIDUAL_HUMANOID_STAND: {
      // mjpc/tasks/humanoid/stand/stand.cc:30-97; task_ids = {torso body, head body, sites sp0..sp3}
      const int* I = MI(task_ids);
      const float *sx = DF(site_xpos), *head = DF(xipos) + 3 * I[1], *com = DF(subtree_com) + 3 * I[0],
                  *vel = DF(subtree_linvel) + 3 * I[0];
      if (lane == 0) {
        float favg[3] = {0, 0, 0};
        for (int k = 0; k < 4; k++)
          for (int q = 0; q < 3; q++) favg[q] += 0.25f * sx[3 * I[2 + k] + q];
        r[0] = head[2] - favg[2] - MF(task_parameters)[0];
        const float dx = favg[0] - (com[0] + vel[0] * 0.2f), dy = favg[1] - (com[1] + vel[1] * 0.2f);
        r[1] = sqrtf(dx * dx + dy * dy);
        r[2] = vel[0]; r[3] = vel[1];
      }
      for (int i = lane; i < M.nv - 6; i += 32) r[4 + i] = DF(qvel)[6 + i];
      for (int i = lane; i < M.nu; i += 32) r[4 + M.nv - 6 + i] = DF(ctrl)[i];
      __syncwarp();
      break;
    }
    case RESIDUAL_SHADOW_REORIENT: {
      // mjpc/tasks/shadow_reorient/hand.cc:37-84 (81 residuals); task_ids = {grasp site, cube body, goal body, grasp key}.
      // qpos + 7 / qvel + 6 for 26 values are the reference's literal offsets (they start inside the cube's joint).
      const int* I = MI(task_ids);
      const int cube = I[1], goal = I[2];
      if (lane == 0) {
        const float *palm = DF(site_xpos) + 3 * I[0], *pos = DF(xpos) + 3 * cube;
        for (int q = 0; q < 3; q++) r[q] = pos[q] - palm[q];
        float gq[4];
        for (int q = 0; q < 4; q++) gq[q] = DF(xquat)[4 * goal + q];
        quat_normalize(gq);
        sub_quat(r + 3, gq, DF(xquat) + 4 * cube);
        const float* cv = DF(cvel) + 6 * cube;
        float off[3], wx[3];
        for (int q = 0; q < 3; q++) off[q] = pos[q] - DF(subtree_com)[3 * MI(body_rootid)[cube] + q];
        cross3(wx, cv, off);
        for (int q = 0; q < 3; q++) r[6 + q] = cv[3 + q] + wx[q];
      }
      for (int i = lane; i < M.nu; i += 32) r[9 + i] = DF(actuator_force)[i];
      {
        const float* key = MF(key_qpos) + M.nq * I[3];
        for (int i = lane; i < 26; i += 32) { r[9 + M.nu + i] = DF(qpos)[7 + i] - key[7 + i]; r[9 + M.nu + 26 + i] = DF(qvel)[6 + i]; }
      }
      __syncwarp();
      break;
    }
    case RESIDUAL_HUMANOID_TRACK: {
      // mjpc/tasks/humanoid/tracking/tracking.cc:94-216; task_ids = 16 tracking sites then 16 mocap ids,
      // task_state = [mode, reference_time (rebased)], keyframes in HBM (c.gkey).  One tracked body per lane.
      const int lengths[10] = {121, 154, 115, 78, 145, 188, 260, 279, 39, 510};
      const int* I = MI(task_ids);
      const float* S = MF(task_state);
      const int mode = (int)S[0];
      int start = 0;
      for (int i = 0; i < mode; i++) start += lengths[i];
      const int last = start + lengths[mode] - 1;
      const float idx = fminf((float)last, fmaxf(0.f, (c.time - S[1]) * 30.0f + (float)start));
      const int k0 = (int)floorf(idx), k1 = min(k0 + 1, last);
      const float w1 = idx - (float)k0, w0 = 1.f - w1;
      const int nm3 = 3 * M.nmocap, nj = M.nv - 6, nu = M.nu;
      for (int i = lane; i < nj; i += 32) r[i] = DF(qvel)[6 + i];
      for (int i = lane; i < nu; i += 32) r[nj + i] = DF(ctrl)[i];
      float mp[3] = {0, 0, 0}, sp[3] = {0, 0, 0}, vel[3] = {0, 0, 0};
      if (lane < 16) {
        const float *p0 = c.gkey + (size_t)nm3 * k0 + 3 * I[16 + lane], *p1 = c.gkey + (size_t)nm3 * k1 + 3 * I[16 + lane];
        const int site = I[lane], body = MI(site_bodyid)[site];
        const float *sx = DF(site_xpos) + 3 * site, *cv = DF(cvel) + 6 * body,
                    *com = DF(subtree_com) + 3 * MI(body_rootid)[body];
        float off[3], wx[3];
        for (int q = 0; q < 3; q++) {
          const float a = __ldg(p0 + q), b = __ldg(p1 + q);
          mp[q] = a * w0 + b * w1; sp[q] = sx[q]; off[q] = sx[q] - com[q];
          vel[q] = (b - a) * 30.0f;
        }
        cross3(wx, cv, off);
        for (int q = 0; q < 3; q++) vel[q] -= cv[3 + q] + wx[q];
      }
      float am[3], as[3];
      for (int q = 0; q < 3; q++) { am[q] = warp_sum(mp[q]) * (1.f / 16.f); as[q] = warp_sum(sp[q]) * (1.f / 16.f); }
      const int o = nj + nu;
      if (lane < 3) r[o + lane] = am[lane] - as[lane];
      if (lane < 16)
        for (int q = 0; q < 3; q++) {
          r[o + 3 + 3 * lane + q] = (mp[q] - am[q]) - (sp[q] - as[q]);
          r[o + 51 + 3 * lane + q] = vel[q];
        }
      __syncwarp();
      break;
    }
    default: break;
  }
}

}  // namespace mjpc_dev
