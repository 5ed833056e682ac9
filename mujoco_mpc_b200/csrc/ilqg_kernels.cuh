// ilqg_kernels.cuh - iLQG sweeps on the device.
//
//   fd_center_kernel / fd_column_kernel   ModelDerivatives::Compute (mjpc/planners/model_derivatives.cc:45-165):
//       one warp per (timestep, perturbed column); every warp runs the same forward-dynamics device code as the
//       rollout kernel ([EXT] mjd_transitionFD restated: one-sided differences, clamped control nudges,
//       tangent-space state differences).  H*(2nv+nu) independent warps fill the machine.
//   cost_derivatives_kernel               CostDerivatives::Compute (mjpc/planners/cost_derivatives.cc:77-230):
//       one CTA per timestep, Gauss-Newton products accumulated in shared memory.
//   backward_pass_kernel                  RiccatiStep recursion (mjpc/planners/ilqg/backward_pass.cc:65-250,
//       mjpc/planners/ilqg/planner.cc:429-520): ONE CTA, strictly sequential in t (value function dependence),
//       matrices resident in shared memory, box-QP ([EXT] mju_boxQP restated: projected Newton) on one warp.
//       The n=36, m=12 products are fp32 CUDA-core FMAs: a Hopper wgmma tile is at least 64x8x8 per warpgroup with
//       operands in swizzled shared-memory tiles and TF32 inputs, which for 36x36x36 products costs more in
//       staging than the ~0.3 MFLOP per step it would accelerate, and TF32's 10-bit mantissa breaks the
//       Riccati recursion's accuracy (DESIGN.md "tensor cores").
#pragma once
#include <cuda_runtime.h>

#include <type_traits>
#include <utility>
#include <vector>

#include <mutex>

#include "device_memory.h"
#include "rollout_kernels.cuh"

namespace mjpc_dev {

// ------------------------------------------------------------------------------------------ norms with derivatives
// a^b for the exponents of the derivative formulas that can be exactly zero (L22 q/2 - 1, PowerLoss p - 1 and p - 2,
// SmoothAbs2 q - 2).  Under -use_fast_math powf is ex2(b * lg2(a)), so 0^0 = ex2(0 * -inf) = NaN where IEEE and the fp64
// reference give 1; every other input takes the unchanged powf path.
__device__ __forceinline__ float pow_zero_exp(float a, float b) { return b == 0.f ? 1.f : powf(a, b); }

// value; g[n]; H[n*n] (mjpc/norm.cc:50-210). Executed by ONE thread (n <= 16 per term in practice).
__device__ inline float norm_full(float* g, float* Hn, const float* x, const float* params, int n, int type) {
  float y = 0;
  const float p = params[0], q = params[1];
  for (int i = 0; i < n * n; i++) Hn[i] = 0;
  switch (type) {
    case kNull: y = x[0]; g[0] = 1; break;
    case kQuadratic:
      for (int i = 0; i < n; i++) { y += x[i] * x[i]; g[i] = x[i]; Hn[i * n + i] = 1; }
      y *= 0.5f;
      break;
    case kL22: {
      float cc = 0;
      for (int i = 0; i < n; i++) cc += x[i] * x[i];
      const float a = powf(cc, q / 2) + powf(p, q);
      const float s = powf(a, 1 / q);
      y = s - p;
      const float dd = pow_zero_exp(cc, q / 2 - 1);
      const float b = s / a * dd;
      for (int i = 0; i < n; i++) g[i] = b * x[i];
      const float c2 = (1 - q) * dd / a + (q - 2) / fmaxf(cc, 1e-15f);
      for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) Hn[i + j * n] = b * ((i == j ? 1.f : 0.f) + x[i] * x[j] * c2);
      break;
    }
    case kL2: {
      float s = 0;
      for (int i = 0; i < n; i++) s += x[i] * x[i];
      s = sqrtf(s + p * p);
      y = s - p;
      for (int i = 0; i < n; i++) g[i] = s ? x[i] / s : 0.f;
      if (s)
        for (int i = 0; i < n; i++)
          for (int j = 0; j < n; j++) Hn[i + j * n] = ((i == j ? 1.f : 0.f) - g[i] * g[j]) / s;
      break;
    }
    case kCosh:
      for (int i = 0; i < n; i++) {
        y += p * p * (coshf(x[i] / p) - 1);
        g[i] = p * sinhf(x[i] / p);
        Hn[i * n + i] = coshf(x[i] / p);
      }
      break;
    case kPowerLoss:
      for (int i = 0; i < n; i++) {
        const float s = fabsf(x[i]);
        y += powf(s, p);
        g[i] = (x[i] > 0 ? 1.f : (x[i] < 0 ? -1.f : 0.f)) * p * pow_zero_exp(s, p - 1);
        Hn[i * n + i] = (p - 1) * p * pow_zero_exp(s, p - 2);
      }
      break;
    case kSmoothAbsLoss:
      for (int i = 0; i < n; i++) {
        const float s = sqrtf(x[i] * x[i] + p * p);
        y += s - p;
        g[i] = s ? x[i] / s : 0.f;
        Hn[n * i + i] = s ? (1 - g[i] * g[i]) / s : 0.f;
      }
      break;
    case kSmoothAbs2Loss:
      for (int i = 0; i < n; i++) {
        const float a = fabsf(x[i]);
        const float dd = powf(a, q);
        const float e = dd + powf(p, q);
        const float s = powf(e, 1 / q);
        y += s - p;
        const float c2 = s * pow_zero_exp(a, q - 2) / e;
        g[i] = c2 * x[i];
        Hn[i * n + i] = c2 * (q - 1) * (1 - dd / e);
      }
      break;
    case kRectifyLoss:
      for (int i = 0; i < n; i++) {
        if (p > 0) {
          // overflow-safe softplus / sigmoid (softplus_stable, dev_task.cuh): e = e^-|z| lies in (0, 1]
          const float z = x[i] / p, e = expf(-fabsf(z));
          y += p * softplus_stable(z);
          g[i] = z >= 0 ? 1 / (1 + e) : e / (1 + e);
          Hn[i * n + i] = e / (p * (1 + e) * (1 + e));
        } else {
          y += x[i] > 0 ? x[i] : 0.f;
          g[i] = x[i] > 0 ? 1.f : 0.f;
        }
      }
      break;
  }
  return y;
}

// ------------------------------------------------------------------------------------------ model derivatives
// A sweep holds gridDim.y independent problems with common H, skip and mode (so common evaluate / interpolate lists);
// problem b = blockIdx.y reads and writes the b-th [H]-row slice of every per-problem array below.
struct FdArgs {
  DevModel M;
  DevLayout L;
  const float* pack;
  int pack_stride;          // model variants: problem b stages its variant block (problem_pack); 0: the one pack
  const int* pack_index;    // [B]
  const float* x;  // [B][H][ds]
  const float* u;  // [B][H][nu]
  const float* t;  // [B][H] times relative to the problem's t[0]
  const float* mocap;       // [B][7 nmocap]
  const float* task_state;  // [B][task_state_size] (rebased to the problem's t[0]) or nullptr
  const float* weight;      // [B][num_term] or nullptr (the packed Task::weight)
  const float* parameters;  // [B][num_parameters] or nullptr (the packed Task::parameters)
  int H;
  float eps;
  const int* eval_t;  // [neval] evaluated time steps (derivative_skip, model_derivatives.cc:56-72)
  int neval, mode;    // mode 0 one-sided, 1 centred
  float* yp;          // [B][neval*ncol][ds]  centred mode: next state of the +eps evaluation
  float* rp;          // [B][neval*ncol][nr]  ... and its residual
  float* y0;  // [B][H][ds]   centre next state
  float* r0;  // [B][H][nr]   centre residual
  float* q0;  // [B][H][nv]   centre qacc (warm start of the perturbed solves)
  float *A, *B, *C, *D;     // [B][H][..]
};

// one problem's slices of the FdArgs arrays
struct FdProb {
  const float *x, *u, *t, *mocap, *task_state, *weight, *parameters;
  float *yp, *rp, *y0, *r0, *q0, *A, *B, *C, *D;
};
template <class SP>
__device__ __forceinline__ FdProb fd_problem(const Ctx& c, const FdArgs& A, int prob) {
  auto&& M = SP::model(c);
  const size_t b = prob, H = A.H, nq = M.nq, nv = M.nv, nu = M.nu, ds = nq + nv, n = 2 * nv, nr = M.num_residual;
  const size_t ncol = nu + 2 * nv, nevc = (size_t)A.neval * ncol;
  FdProb P;
  P.x = A.x + b * H * ds; P.u = A.u + b * H * nu; P.t = A.t + b * H; P.mocap = A.mocap + b * 7 * M.nmocap;
  P.task_state = A.task_state ? A.task_state + b * M.task_state_size : nullptr;
  P.weight = A.weight ? A.weight + b * M.num_term : nullptr;
  P.parameters = A.parameters ? A.parameters + b * M.num_parameters : nullptr;
  P.yp = A.yp + b * nevc * ds; P.rp = A.rp + b * nevc * nr;
  P.y0 = A.y0 + b * H * ds; P.r0 = A.r0 + b * H * nr; P.q0 = A.q0 + b * H * nv;
  P.A = A.A + b * H * n * n; P.B = A.B + b * H * n * nu; P.C = A.C + b * H * nr * n; P.D = A.D + b * H * nr * nu;
  return P;
}

// the problem's task snapshot, as in the rollout prologue; then the state, control and mocap of step t and the warm
// start (NULL: zeros)
template <class SP>
__device__ __forceinline__ void fd_load_state(Ctx& c, const FdProb& P, int t, const float* warmstart) {
  auto&& M = SP::model(c);
  const size_t x = (size_t)t * (M.nq + M.nv);
  load_task<SP>(c, 0, P.task_state, P.weight, P.parameters);
  load_state<SP>(c, P.x + x, P.x + x + M.nq, P.u + (size_t)t * M.nu, warmstart, P.mocap);
  c.time = P.t[t];
  __syncwarp();
}

template <class SP>
__device__ __forceinline__ void fd_center_body(const FdArgs& A) {
  float* smem = g_smem;
  const float* pack = problem_pack(A.pack, A.pack_stride, A.pack_index, (int)blockIdx.y);
  stage_model_pack(smem, pack, (unsigned)((A.M.nf + A.M.ni) * 4));
  Ctx c;
  init_ctx(c, &A.M, &A.L, smem, threadIdx.x, pack, A.pack_stride);
  auto&& M = SP::model(c);
  const int lane = c.lane, t = A.eval_t[blockIdx.x], nq = M.nq, nv = M.nv, ds = nq + nv, nr = M.num_residual;
  const FdProb P = fd_problem<SP>(c, A, blockIdx.y);
  fd_load_state<SP>(c, P, t, nullptr);
  k_forward<SP>(c);
  k_residual<SP>(c);
  for (int i = lane; i < nr; i += 32) P.r0[(size_t)t * nr + i] = DF(residual)[i];
  for (int i = lane; i < nv; i += 32) P.q0[(size_t)t * nv + i] = DF(qacc)[i];
  k_euler<SP>(c);
  for (int i = lane; i < nq; i += 32) P.y0[(size_t)t * ds + i] = DF(qpos)[i];
  for (int i = lane; i < nv; i += 32) P.y0[(size_t)t * ds + nq + i] = DF(qvel)[i];
}

// one warp per (evaluated t, column). columns: [0, nu) controls, [nu, nu+nv) velocities, [nu+nv, nu+2nv) positions.
// Centred mode runs the +eps evaluation, parks its next state / residual in HBM scratch, reloads the state, runs the
// -eps evaluation and differences the two ([EXT] mjd_transitionFD flg_centered); a control that can only be nudged one
// way inside ctrlrange falls back to the one-sided difference.
template <class SP>
__device__ __forceinline__ void fd_perturb(Ctx& c, int col, int nu, int nv, float h) {
  const int lane = c.lane;
  if (col < nu) {
    if (lane == 0) DF(ctrl)[col] += h;
  } else if (col < nu + nv) {
    if (lane == 0) DF(qvel)[col - nu] += h;
  } else {
    // tangent-space position perturbation ([EXT] mj_integratePos with a unit vector)
    const int dof = col - nu - nv;
    if (lane == 0) {
      const int j = MI(dof_jntid)[dof];
      const int qa = MI(jnt_qposadr)[j], da = MI(jnt_dofadr)[j], k = dof - da, ty = MI(jnt_type)[j];
      float* qpos = DF(qpos);
      if (ty == JNT_FREE) {
        if (k < 3) qpos[qa + k] += h;
        else { float w[3] = {0, 0, 0}; w[k - 3] = 1; quat_integrate(qpos + qa + 3, w, h); }
      } else if (ty == JNT_BALL) {
        float w[3] = {0, 0, 0}; w[k] = 1; quat_integrate(qpos + qa, w, h);
      } else {
        qpos[qa] += h;
      }
    }
  }
  __syncwarp();
}

template <class SP>
__device__ __forceinline__ void fd_column_body(const FdArgs& A) {
  float* smem = g_smem;
  const float* pack = problem_pack(A.pack, A.pack_stride, A.pack_index, (int)blockIdx.y);
  stage_model_pack(smem, pack, (unsigned)((A.M.nf + A.M.ni) * 4));
  Ctx c;
  init_ctx(c, &A.M, &A.L, smem, threadIdx.x, pack, A.pack_stride);
  auto&& M = SP::model(c);
  const int lane = c.lane, nq = M.nq, nv = M.nv, nu = M.nu, ds = nq + nv, n = 2 * nv, nr = M.num_residual;
  const int ncol = nu + 2 * nv;
  const int te = blockIdx.x / ncol, col = blockIdx.x - te * ncol;
  const int t = A.eval_t[te];
  const bool last = t == A.H - 1;
  if (last && col < nu) return;  // only C is computed at the final time step (model_derivatives.cc:89-93)
  const FdProb P = fd_problem<SP>(c, A, blockIdx.y);
  fd_load_state<SP>(c, P, t, P.q0 + (size_t)t * nv);
  float h = A.eps;  // signed step of a one-sided difference
  bool centred = A.mode == 1;
  if (col < nu) {
    const int i = col;
    const bool limited = MI(actuator_ctrllimited)[i] != 0;
    const float lo = MF(actuator_ctrlrange)[2 * i], hi = MF(actuator_ctrlrange)[2 * i + 1];
    const float u0 = DF(ctrl)[i];
    const bool inside = u0 >= lo && u0 <= hi;
    const bool fwd = !limited || (inside && u0 + A.eps >= lo && u0 + A.eps <= hi);
    const bool back = !limited || (inside && u0 - A.eps >= lo && u0 - A.eps <= hi);
    if (!fwd && !back) {
      for (int k = lane; k < n; k += 32) P.B[((size_t)t * n + k) * nu + i] = 0;
      for (int k = lane; k < nr; k += 32) P.D[((size_t)t * nr + k) * nu + i] = 0;
      return;
    }
    centred = centred && fwd && back;
    if (!centred) h = fwd ? A.eps : -A.eps;
    __syncwarp();   // every lane has read u0 before lane 0 overwrites it
  }
  float* yp = P.yp + (size_t)blockIdx.x * ds;
  float* rp = P.rp + (size_t)blockIdx.x * nr;
  fd_perturb<SP>(c, col, nu, nv, centred ? A.eps : h);
  k_forward<SP>(c);
  k_residual<SP>(c);
  if (centred) {
    for (int k = lane; k < nr; k += 32) rp[k] = DF(residual)[k];
    if (!last) {
      k_euler<SP>(c);
      for (int i = lane; i < nq; i += 32) yp[i] = DF(qpos)[i];
      for (int i = lane; i < nv; i += 32) yp[nq + i] = DF(qvel)[i];
    }
    __syncwarp();
    fd_load_state<SP>(c, P, t, P.q0 + (size_t)t * nv);
    fd_perturb<SP>(c, col, nu, nv, -A.eps);
    k_forward<SP>(c);
    k_residual<SP>(c);
  }
  // centred: (plus - minus) / 2 eps with the current evaluation as "minus"; one-sided: (this - centre) / h
  const float ih = centred ? -0.5f / A.eps : 1.0f / h;
  const float* rref = centred ? rp : P.r0 + (size_t)t * nr;
  // residual columns
  float* Cout = col < nu ? P.D : P.C;
  const int cw = col < nu ? nu : n;
  const int cc = col < nu ? col : (col < nu + nv ? nv + (col - nu) : col - nu - nv);
  for (int k = lane; k < nr; k += 32)
    Cout[((size_t)t * nr + k) * cw + cc] = (DF(residual)[k] - rref[k]) * ih;
  if (last) return;
  k_euler<SP>(c);
  // next-state difference in the tangent space (StateDiff / mj_differentiatePos)
  float* Sout = col < nu ? P.B : P.A;
  const float* y0 = centred ? yp : P.y0 + (size_t)t * ds;
  const int *jtype = MI(jnt_type), *jqadr = MI(jnt_qposadr), *jdadr = MI(jnt_dofadr);
  const float *qpos = DF(qpos), *qvel = DF(qvel);
  for (int j = lane; j < M.njnt; j += 32) {
    const int qa = jqadr[j], da = jdadr[j], ty = jtype[j];
    if (ty == JNT_FREE) {
      for (int k = 0; k < 3; k++) Sout[((size_t)t * n + da + k) * cw + cc] = (qpos[qa + k] - y0[qa + k]) * ih;
      float dq[3];
      sub_quat(dq, qpos + qa + 3, y0 + qa + 3);
      for (int k = 0; k < 3; k++) Sout[((size_t)t * n + da + 3 + k) * cw + cc] = dq[k] * ih;
    } else if (ty == JNT_BALL) {
      float dq[3];
      sub_quat(dq, qpos + qa, y0 + qa);
      for (int k = 0; k < 3; k++) Sout[((size_t)t * n + da + k) * cw + cc] = dq[k] * ih;
    } else {
      Sout[((size_t)t * n + da) * cw + cc] = (qpos[qa] - y0[qa]) * ih;
    }
  }
  for (int i = lane; i < nv; i += 32) Sout[((size_t)t * n + nv + i) * cw + cc] = (qvel[i] - y0[nq + i]) * ih;
}

// linear interpolation of the skipped time steps (model_derivatives.cc:109-164): one CTA per (interpolated t, problem)
struct FdInterpArgs {
  const int *t, *e0, *e1;   // [ninterp]
  const float* w;           // [ninterp] weight of e1
  float *A, *B, *C, *D;     // [B][H][..]
  int nA, nB, nC, nD, H;
};
extern "C" __global__ void __launch_bounds__(256) fd_interp_kernel(const __grid_constant__ FdInterpArgs P) {
  const int k = blockIdx.x, t = P.t[k], e0 = P.e0[k], e1 = P.e1[k];
  const size_t prob = blockIdx.y;
  const float w = P.w[k];
  auto lerp = [&](float* X0, int sz) {
    float* X = X0 + prob * P.H * sz;
    for (int i = threadIdx.x; i < sz; i += blockDim.x)
      X[(size_t)t * sz + i] = (1.f - w) * X[(size_t)e0 * sz + i] + w * X[(size_t)e1 * sz + i];
  };
  lerp(P.A, P.nA); lerp(P.B, P.nB); lerp(P.C, P.nC); lerp(P.D, P.nD);
}

extern "C" __global__ void __launch_bounds__(32) fd_center_kernel(const __grid_constant__ FdArgs A) { fd_center_body<DynSpec>(A); }
extern "C" __global__ void __launch_bounds__(32) fd_column_kernel(const __grid_constant__ FdArgs A) { fd_column_body<DynSpec>(A); }
// statically specialised instances (spec_quadruped.h), selected by the host when the live model matches
extern "C" __global__ void __launch_bounds__(32) fd_center_kernel_quadruped(const __grid_constant__ FdArgs A) {
  fd_center_body<StaticSpec<SpecQuadruped>>(A);
}
extern "C" __global__ void __launch_bounds__(32) fd_column_kernel_quadruped(const __grid_constant__ FdArgs A) {
  fd_column_body<StaticSpec<SpecQuadruped>>(A);
}

// ------------------------------------------------------------------------------------------ cost derivatives
// gridDim.y independent problems: problem b reads and writes the b-th [H]-row slice of every array
struct CostArgs {
  DevModel M;
  const float* pack;
  const float* residual;  // [B][H][nr]
  const float* C;         // [B][H][nr][n]
  const float* D;         // [B][H][nr][m]
  const float* weight;    // [B][num_term] or nullptr (the packed Task::weight)
  int H, n, m;
  float *cx, *cu, *cxx, *cuu, *cxu;   // [B][H][..]
};

// one CTA per (time step, problem); dynamic smem: g[nr] Hn[kmax^2] Sx[kmax*n] Su[kmax*m] acc[n + m + n*n + m*m + n*m] cval[1]
extern "C" __global__ void __launch_bounds__(256) cost_derivatives_kernel(const __grid_constant__ CostArgs A) {
  extern __shared__ __align__(16) float sm[];
  const DevModel& M = A.M;
  const int t = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, n = A.n, m = A.m, nr = M.num_residual;
  const float* mf = A.pack;
  const int* mi = reinterpret_cast<const int*>(A.pack + M.nf);
  const int *dimr = mi + M.io[I_task_dim_norm_residual], *ntype = mi + M.io[I_task_norm], *npar = mi + M.io[I_task_num_norm_parameter];
  const size_t pb = blockIdx.y, H = A.H;
  const float* wgt = A.weight ? A.weight + pb * M.num_term : mf + M.fo[F_task_weight];
  const float* prm = mf + M.fo[F_task_norm_parameter];
  const float *res = A.residual + pb * H * nr, *Cm = A.C + pb * H * nr * n, *Dm = A.D + pb * H * nr * m;
  int kmax = 1;
  for (int i = 0; i < M.num_term; i++) kmax = max(kmax, dimr[i]);
  float* g = sm;
  float* Hn = g + nr;
  float* Sx = Hn + kmax * kmax;
  float* Su = Sx + kmax * n;
  float* acc = Su + kmax * m;
  float *aCx = acc, *aCu = aCx + n, *aCxx = aCu + m, *aCuu = aCxx + n * n, *aCxu = aCuu + m * m;
  float* cval = aCxu + n * m;
  const int nacc = n + m + n * n + m * m + n * m;
  for (int i = tid; i < nacc; i += nt) acc[i] = 0;
  if (tid == 0) *cval = 0;
  __syncthreads();
  int f = 0, p = 0;
  for (int i = 0; i < M.num_term; i++) {
    const int k = dimr[i];
    const float w = wgt[i] / (float)A.H;
    const float* r = res + (size_t)t * nr + f;
    const float* rx = Cm + ((size_t)t * nr + f) * n;
    const float* ru = Dm + ((size_t)t * nr + f) * m;
    if (tid == 0) {
      float pr[2] = {npar[i] > 0 ? prm[p] : 0.f, npar[i] > 1 ? prm[p + 1] : 0.f};
      *cval += w * norm_full(g, Hn, r, pr, k, ntype[i]);
    }
    __syncthreads();
    for (int e = tid; e < k * n; e += nt) { const int a = e / n, b = e - a * n; float s = 0; for (int q = 0; q < k; q++) s += Hn[a * k + q] * rx[q * n + b]; Sx[e] = s; }
    for (int e = tid; e < k * m; e += nt) { const int a = e / m, b = e - a * m; float s = 0; for (int q = 0; q < k; q++) s += Hn[a * k + q] * ru[q * m + b]; Su[e] = s; }
    for (int a = tid; a < n; a += nt) { float s = 0; for (int b = 0; b < k; b++) s += rx[b * n + a] * g[b]; aCx[a] += w * s; }
    for (int a = tid; a < m; a += nt) { float s = 0; for (int b = 0; b < k; b++) s += ru[b * m + a] * g[b]; aCu[a] += w * s; }
    __syncthreads();
    for (int e = tid; e < n * n; e += nt) { const int a = e / n, b = e - a * n; float s = 0; for (int q = 0; q < k; q++) s += Sx[q * n + a] * rx[q * n + b]; aCxx[e] += w * s; }
    for (int e = tid; e < n * m; e += nt) { const int a = e / m, b = e - a * m; float s = 0; for (int q = 0; q < k; q++) s += Sx[q * n + a] * ru[q * m + b]; aCxu[e] += w * s; }
    for (int e = tid; e < m * m; e += nt) { const int a = e / m, b = e - a * m; float s = 0; for (int q = 0; q < k; q++) s += Su[q * m + a] * ru[q * m + b]; aCuu[e] += w * s; }
    __syncthreads();
    f += k;
    p += npar[i];
  }
  // risk transformation (cost_derivatives.cc:160-224): scale, then outer products of the SCALED gradients
  if (fabsf(M.risk) >= 1e-6f) {
    const float s = expf(M.risk * (*cval));
    for (int a = tid; a < n; a += nt) aCx[a] *= s;
    for (int a = tid; a < m; a += nt) aCu[a] *= s;
    __syncthreads();
    for (int e = tid; e < n * n; e += nt) { const int a = e / n, b = e - a * n; aCxx[e] = aCxx[e] * s + M.risk * s * aCx[a] * aCx[b]; }
    for (int e = tid; e < n * m; e += nt) { const int a = e / m, b = e - a * m; aCxu[e] = aCxu[e] * s + M.risk * s * aCx[a] * aCu[b]; }
    for (int e = tid; e < m * m; e += nt) { const int a = e / m, b = e - a * m; aCuu[e] = aCuu[e] * s + M.risk * s * aCu[a] * aCu[b]; }
    __syncthreads();
  }
  const size_t row = pb * H + t;
  for (int a = tid; a < n; a += nt) A.cx[row * n + a] = aCx[a];
  for (int a = tid; a < m; a += nt) A.cu[row * m + a] = aCu[a];
  for (int e = tid; e < n * n; e += nt) A.cxx[row * n * n + e] = aCxx[e];
  for (int e = tid; e < m * m; e += nt) A.cuu[row * m * m + e] = aCuu[e];
  for (int e = tid; e < n * m; e += nt) A.cxu[row * n * m + e] = aCxu[e];
}

// ------------------------------------------------------------------------------------------ backward pass
// one CTA per problem: problem b reads and writes the b-th [H]-row slice of every array, mu[b], dV[b][2], status[b]
struct BackwardArgs {
  const float *A, *B, *cx, *cu, *cxx, *cxu, *cuu, *actions, *ctrlrange;
  int n, m, H, reg_type, limits;
  const float* mu;        // [B]
  float *K, *du, *dV, *Vx, *Vxx;
  int* status;            // [B]
};

// dense Cholesky / solve for the tiny box-QP blocks, single thread
__device__ inline float chol_serial(float* A, int n) {
  float minp = 3.4e38f;
  for (int j = 0; j < n; j++) {
    float s = A[j * n + j];
    for (int k = 0; k < j; k++) s -= A[j * n + k] * A[j * n + k];
    minp = fminf(minp, s);
    if (s < 1e-15f) s = 1e-15f;
    const float l = sqrtf(s);
    A[j * n + j] = l;
    for (int i = j + 1; i < n; i++) {
      float tt = A[i * n + j];
      for (int k = 0; k < j; k++) tt -= A[i * n + k] * A[j * n + k];
      A[i * n + j] = tt / l;
    }
  }
  return minp;
}
__device__ inline void chol_solve_serial(float* x, const float* L, const float* b, int n) {
  for (int i = 0; i < n; i++) { float s = b[i]; for (int k = 0; k < i; k++) s -= L[i * n + k] * x[k]; x[i] = s / L[i * n + i]; }
  for (int i = n - 1; i >= 0; i--) { float s = x[i]; for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k]; x[i] = s / L[i * n + i]; }
}
// projected-Newton box QP (same algorithm and constants as oracle/ilqg.h box_qp). scratch >= 6n floats + n ints
__device__ inline int box_qp_serial(float* res, float* R, int* index, const float* Hm, const float* g, int n,
                                    const float* lower, const float* upper, float* scratch) {
  // fp32 floors on the reference's fp64 constants (mingrad 1e-16, minstep 1e-22): below ~1e-7 relative neither the
  // free-gradient norm nor a backtracked step is resolvable in fp32, and looping on them only burns serial time
  const int maxiter = 100;
  const float mingrad = 1e-6f, backtrack = 0.5f, minstep = 1e-7f, armijo = 0.01f;
  float *grad = scratch, *search = grad + n, *cand = search + n, *tmp = cand + n, *rhs = tmp + n, *sol = rhs + n;
  int* clamped = reinterpret_cast<int*>(sol + n);
  for (int i = 0; i < n; i++) { res[i] = fmaxf(lower[i], fminf(upper[i], res[i])); clamped[i] = 0; }
  auto value_of = [&](const float* x) {
    float v = 0;
    for (int i = 0; i < n; i++) { float a = 0; for (int j = 0; j < n; j++) a += Hm[i * n + j] * x[j]; v += x[i] * (0.5f * a + g[i]); }
    return v;
  };
  float value = value_of(res);
  int nfree = 0;
  for (int iter = 0; iter < maxiter; iter++) {
    for (int i = 0; i < n; i++) { float a = g[i]; for (int j = 0; j < n; j++) a += Hm[i * n + j] * res[j]; grad[i] = a; }
    bool changed = iter == 0;
    nfree = 0;
    for (int i = 0; i < n; i++) {
      const int cl = (res[i] == lower[i] && grad[i] > 0) || (res[i] == upper[i] && grad[i] < 0);
      if (cl != clamped[i]) changed = true;
      clamped[i] = cl;
      if (!cl) index[nfree++] = i;
    }
    if (nfree == 0) break;
    if (changed) {
      for (int a = 0; a < nfree; a++)
        for (int b = 0; b < nfree; b++) R[a * nfree + b] = Hm[index[a] * n + index[b]];
      if (!(chol_serial(R, nfree) > 1e-15f)) return -1;
    }
    float norm2 = 0;
    for (int a = 0; a < nfree; a++) norm2 += grad[index[a]] * grad[index[a]];
    float gscale = 0;
    for (int i = 0; i < n; i++) gscale += g[i] * g[i];
    if (norm2 < mingrad * mingrad * (1.f + gscale)) break;
    for (int i = 0; i < n; i++) tmp[i] = clamped[i] ? res[i] : 0.f;
    for (int a = 0; a < nfree; a++) {
      const int i = index[a];
      float s = g[i];
      for (int j = 0; j < n; j++) s += Hm[i * n + j] * tmp[j];
      rhs[a] = s;
    }
    chol_solve_serial(sol, R, rhs, nfree);
    for (int i = 0; i < n; i++) search[i] = 0;
    for (int a = 0; a < nfree; a++) search[index[a]] = -sol[a] - res[index[a]];
    float sdotg = 0;
    for (int i = 0; i < n; i++) sdotg += search[i] * grad[i];
    if (sdotg >= 0) break;
    float step = 1, vc = value;
    bool accepted = false;
    while (step > minstep) {
      for (int i = 0; i < n; i++) cand[i] = fmaxf(lower[i], fminf(upper[i], res[i] + step * search[i]));
      vc = value_of(cand);
      if ((vc - value) / (step * sdotg) >= armijo) { accepted = true; break; }
      step *= backtrack;
    }
    if (!accepted) break;
    for (int i = 0; i < n; i++) res[i] = cand[i];
    value = vc;
  }
  return nfree;
}

// ---- warp-parallel versions (warp 0 of the CTA; n <= 32; lane i owns element / row i).  Same algorithm and
// constants as the serial code above; the left-looking Cholesky and the forward substitution subtract in the
// same order as the serial loops, reductions are butterfly sums (identical in every lane, so control flow stays
// warp-uniform).  The serial box-QP dominated the backward pass before.
__device__ inline float chol_warp(float* A, int n, int lane) {
  float minp = 3.4e38f;
  for (int j = 0; j < n; j++) {
    float s = 0.f;
    if (lane >= j && lane < n) {
      s = A[lane * n + j];
      for (int k = 0; k < j; k++) s -= A[lane * n + k] * A[j * n + k];
    }
    float piv = __shfl_sync(kFull, s, j);
    minp = fminf(minp, piv);
    if (piv < 1e-15f) piv = 1e-15f;
    const float l = sqrtf(piv);
    if (lane == j) A[j * n + j] = l;
    else if (lane > j && lane < n) A[lane * n + j] = s / l;
    __syncwarp();
  }
  return minp;
}
// x = (L L^T)^-1 b for lane < n (value returned per lane; b passed per lane)
__device__ inline float chol_solve_warp(const float* L, float b, int n, int lane) {
  float y = b;
  for (int i = 0; i < n; i++) {
    const float xi = __shfl_sync(kFull, y, i) / L[i * n + i];
    if (lane == i) y = xi;
    else if (lane > i && lane < n) y -= L[lane * n + i] * xi;
  }
  for (int i = n - 1; i >= 0; i--) {
    const float xi = __shfl_sync(kFull, y, i) / L[i * n + i];
    if (lane == i) y = xi;
    else if (lane < i) y -= L[i * n + lane] * xi;
  }
  return y;
}
// scratch >= 2n floats.  res/R/index as in box_qp_serial; returns nfree or -1 (not positive definite)
__device__ inline int box_qp_warp(float* res, float* R, int* index, const float* Hm, const float* g, int n,
                                  const float* lower, const float* upper, float* scratch, int lane) {
  const int maxiter = 100;
  const float mingrad = 1e-6f, backtrack = 0.5f, minstep = 1e-7f, armijo = 0.01f;
  float *xs = scratch, *ts = scratch + n;        // shared copies of the current iterate / a temporary vector
  const bool act = lane < n;
  const float lo = act ? lower[lane] : 0.f, hi = act ? upper[lane] : 0.f, gi = act ? g[lane] : 0.f;
  float x = act ? fmaxf(lo, fminf(hi, res[lane])) : 0.f;
  auto hrow = [&](const float* v) { float a = 0.f; if (act) for (int j = 0; j < n; j++) a += Hm[lane * n + j] * v[j]; return a; };
  auto value_of = [&](float xv) {   // xv: this lane's element; the vector is published through ts
    if (act) ts[lane] = xv;
    __syncwarp();
    const float a = hrow(ts);
    const float v = warp_sum(act ? xv * (0.5f * a + gi) : 0.f);
    __syncwarp();
    return v;
  };
  float value = value_of(x);
  const float gscale = warp_sum(gi * gi);
  int nfree = 0, clamped = 0;
  for (int iter = 0; iter < maxiter; iter++) {
    if (act) xs[lane] = x;
    __syncwarp();
    const float grad = gi + hrow(xs);
    const int cl = act && ((x == lo && grad > 0) || (x == hi && grad < 0));
    bool changed = iter == 0 || __any_sync(kFull, cl != clamped);
    clamped = cl;
    const unsigned fmask = __ballot_sync(kFull, act && !cl);
    nfree = __popc(fmask);
    const int pos = __popc(fmask & ((1u << lane) - 1u));
    if (act && !cl) index[pos] = lane;
    __syncwarp();
    if (nfree == 0) break;
    if (changed) {
      for (int e = lane; e < nfree * nfree; e += 32) { const int a = e / nfree, b = e - a * nfree; R[e] = Hm[index[a] * n + index[b]]; }
      __syncwarp();
      if (!(chol_warp(R, nfree, lane) > 1e-15f)) return -1;
    }
    const float norm2 = warp_sum((act && !cl) ? grad * grad : 0.f);
    if (norm2 < mingrad * mingrad * (1.f + gscale)) break;
    if (act) ts[lane] = cl ? x : 0.f;
    __syncwarp();
    float rhs = 0.f;
    if (lane < nfree) { const int i = index[lane]; rhs = g[i]; for (int j = 0; j < n; j++) rhs += Hm[i * n + j] * ts[j]; }
    __syncwarp();
    const float sol = chol_solve_warp(R, rhs, nfree, lane);
    if (lane < nfree) ts[index[lane]] = sol;     // scatter the free solution back to full indexing
    __syncwarp();
    const float search = (act && !cl) ? -ts[lane] - x : 0.f;
    __syncwarp();
    const float sdotg = warp_sum(search * grad);
    if (sdotg >= 0) break;
    float step = 1, vc = value, cand = x;
    bool accepted = false;
    while (step > minstep) {
      cand = act ? fmaxf(lo, fminf(hi, x + step * search)) : 0.f;
      vc = value_of(cand);
      if ((vc - value) / (step * sdotg) >= armijo) { accepted = true; break; }
      step *= backtrack;
    }
    if (!accepted) break;
    x = cand;
    value = vc;
  }
  if (act) res[lane] = x;
  __syncwarp();
  return nfree;
}

// dynamic smem layout (floats): At[n*n] Bt[n*m] W[n*n] T1[n*n] Qxx[n*n] Qxu[n*m] Quu[m*m] QxuR[n*m] QuuR[m*m]
//   K[m*n] Wx[n] Qx[n] Qu[m] du[m] Qd[m] qp_res[m] qp_R[m*m] qp_lo[m] qp_hi[m] scratch[8m] + index[m] ints
// One CTA walks the 63 dependent Riccati steps; within a step the 36x36x36 products are spread over all threads.  The
// thread count is a latency knob, not a throughput one: with 8 warps (2 per scheduler) the shared-memory load -> FMA
// chains of the products were exposed; 512 threads measured faster than 256 and 1024 - the rest is the serial box-QP
// and gain solves between the barriers.
constexpr int kBackwardThreads = 512;
extern "C" __global__ void __launch_bounds__(kBackwardThreads) backward_pass_kernel(const __grid_constant__ BackwardArgs P0) {
  extern __shared__ __align__(16) float sm[];
  const int n = P0.n, m = P0.m, H = P0.H, tid = threadIdx.x, nt = blockDim.x;
  // this CTA's problem: its slices, its regularisation
  const size_t pb = blockIdx.x, Hs = H;
  BackwardArgs P = P0;
  P.A += pb * Hs * n * n; P.B += pb * Hs * n * m; P.cx += pb * Hs * n; P.cu += pb * Hs * m; P.cxx += pb * Hs * n * n;
  P.cxu += pb * Hs * n * m; P.cuu += pb * Hs * m * m; P.actions += pb * Hs * m;
  P.K += pb * Hs * m * n; P.du += pb * Hs * m; P.dV += 2 * pb; P.Vx += pb * Hs * n; P.Vxx += pb * Hs * n * n;
  P.status += pb;
  const float mu = P0.mu[pb];
  float* At = sm; float* Bt = At + n * n; float* W = Bt + n * m; float* T1 = W + n * n; float* Qxx = T1 + n * n;
  float* Qxu = Qxx + n * n; float* Quu = Qxu + n * m; float* QxuR = Quu + m * m; float* QuuR = QxuR + n * m;
  float* K = QuuR + m * m; float* Wx = K + m * n; float* Qx = Wx + n; float* Qu = Qx + n; float* du = Qu + m;
  float* Qd = du + m; float* qp_res = Qd + m; float* qp_R = qp_res + m; float* qp_lo = qp_R + m * m; float* qp_hi = qp_lo + m;
  float* scratch = qp_hi + m;
  int* qp_index = reinterpret_cast<int*>(scratch + 8 * m);
  __shared__ int s_mf, s_ok;
  __shared__ float s_dV[2];
  if (tid == 0) { s_dV[0] = s_dV[1] = 0; s_ok = 1; }
  for (int i = tid; i < m; i += nt) qp_res[i] = 0;
  // terminal value function
  for (int i = tid; i < n; i += nt) { const float v = P.cx[(size_t)(H - 1) * n + i]; Wx[i] = v; if (P.Vx) P.Vx[(size_t)(H - 1) * n + i] = v; }
  for (int i = tid; i < n * n; i += nt) { const float v = P.cxx[(size_t)(H - 1) * n * n + i]; W[i] = v; if (P.Vxx) P.Vxx[(size_t)(H - 1) * n * n + i] = v; }
  __syncthreads();
  for (int t = H - 2; t >= 0; t--) {
    for (int i = tid; i < n * n; i += nt) At[i] = P.A[(size_t)t * n * n + i];
    for (int i = tid; i < n * m; i += nt) Bt[i] = P.B[(size_t)t * n * m + i];
    __syncthreads();
    // T1 = At' W ; Qx, Qu
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; float s = 0; for (int k = 0; k < n; k++) s += At[k * n + i] * W[k * n + j]; T1[e] = s; }
    for (int i = tid; i < n; i += nt) { float s = P.cx[(size_t)t * n + i]; for (int k = 0; k < n; k++) s += At[k * n + i] * Wx[k]; Qx[i] = s; }
    for (int i = tid; i < m; i += nt) { float s = P.cu[(size_t)t * m + i]; for (int k = 0; k < n; k++) s += Bt[k * m + i] * Wx[k]; Qu[i] = s; }
    __syncthreads();
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; float s = P.cxx[(size_t)t * n * n + e]; for (int k = 0; k < n; k++) s += T1[i * n + k] * At[k * n + j]; Qxx[e] = s; }
    for (int e = tid; e < n * m; e += nt) { const int i = e / m, j = e - i * m; float s = P.cxu[(size_t)t * n * m + e]; for (int k = 0; k < n; k++) s += T1[i * n + k] * Bt[k * m + j]; Qxu[e] = s; }
    __syncthreads();
    // Quu = cuu + Bt' W Bt : T1[0:m*n] = Bt' W
    for (int e = tid; e < m * n; e += nt) { const int i = e / n, j = e - i * n; float s = 0; for (int k = 0; k < n; k++) s += Bt[k * m + i] * W[k * n + j]; T1[e] = s; }
    __syncthreads();
    for (int e = tid; e < m * m; e += nt) { const int i = e / m, j = e - i * m; float s = P.cuu[(size_t)t * m * m + e]; for (int k = 0; k < n; k++) s += T1[i * n + k] * Bt[k * m + j]; Quu[e] = s; }
    __syncthreads();
    // regularisation (backward_pass.cc:115-153)
    if (P.reg_type == 2) {
      // value regularisation: Vreg = W + mu I ; QxuR = cxu + At' Vreg Bt ; QuuR = cuu + Bt' Vreg Bt
      for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; float s = 0; for (int k = 0; k < n; k++) s += At[k * n + i] * (W[k * n + j] + (k == j ? mu : 0.f)); T1[e] = s; }
      __syncthreads();
      for (int e = tid; e < n * m; e += nt) { const int i = e / m, j = e - i * m; float s = P.cxu[(size_t)t * n * m + e]; for (int k = 0; k < n; k++) s += T1[i * n + k] * Bt[k * m + j]; QxuR[e] = s; }
      __syncthreads();
      for (int e = tid; e < m * n; e += nt) { const int i = e / n, j = e - i * n; float s = 0; for (int k = 0; k < n; k++) s += Bt[k * m + i] * (W[k * n + j] + (k == j ? mu : 0.f)); T1[e] = s; }
      __syncthreads();
      for (int e = tid; e < m * m; e += nt) { const int i = e / m, j = e - i * m; float s = P.cuu[(size_t)t * m * m + e]; for (int k = 0; k < n; k++) s += T1[i * n + k] * Bt[k * m + j]; QuuR[e] = s; }
    } else {
      for (int e = tid; e < n * m; e += nt) QxuR[e] = Qxu[e];
      for (int e = tid; e < m * m; e += nt) QuuR[e] = Quu[e];
    }
    __syncthreads();
    if (mu != 0.f) {
      if (P.reg_type == 0) {
        for (int i = tid; i < m; i += nt) QuuR[i * m + i] += mu;
      } else if (P.reg_type == 1) {
        for (int e = tid; e < n * m; e += nt) { const int i = e / m, j = e - i * m; float s = 0; for (int k = 0; k < n; k++) s += At[k * n + i] * Bt[k * m + j]; QxuR[e] += mu * s; }
        for (int e = tid; e < m * m; e += nt) { const int i = e / m, j = e - i * m; float s = 0; for (int k = 0; k < n; k++) s += Bt[k * m + i] * Bt[k * m + j]; QuuR[e] += mu * s; }
      }
    }
    for (int e = tid; e < m * n; e += nt) K[e] = 0;
    __syncthreads();
    // control step: box QP (or plain solve) on warp 0, gains on all threads
    if (tid < 32) {
      int mf;
      if (P.limits == 1) {
        if (tid < m) {
          qp_lo[tid] = P.ctrlrange[2 * tid] - P.actions[(size_t)t * m + tid];
          qp_hi[tid] = P.ctrlrange[2 * tid + 1] - P.actions[(size_t)t * m + tid];
        }
        __syncwarp();
        mf = box_qp_warp(qp_res, qp_R, qp_index, QuuR, Qu, m, qp_lo, qp_hi, scratch, tid);
        if (mf >= 0 && tid < m) du[tid] = qp_res[tid];
      } else {
        for (int i = tid; i < m * m; i += 32) qp_R[i] = QuuR[i];
        __syncwarp();
        mf = (chol_warp(qp_R, m, tid) > 1e-15f) ? m : -1;
        if (mf >= 0) {
          if (tid < m) qp_index[tid] = tid;
          const float sol = chol_solve_warp(qp_R, tid < m ? Qu[tid] : 0.f, m, tid);
          if (tid < m) du[tid] = -sol;
        }
      }
      if (tid == 0) { s_mf = mf; if (mf < 0) s_ok = 0; }
    }
    __syncthreads();
    if (!s_ok) break;
    const int mf = s_mf;
    // K on the free dims: column j of -H_free^-1 Qxu_free' (unregularised Qxu, backward_pass.cc:176-192)
    for (int j = tid; j < n; j += nt) {
      float rhs[32], sol[32];
      for (int i = 0; i < mf; i++) rhs[i] = Qxu[j * m + qp_index[i]];
      chol_solve_serial(sol, qp_R, rhs, mf);
      for (int i = 0; i < mf; i++) K[qp_index[i] * n + j] = -sol[i];
    }
    for (int i = tid; i < m; i += nt) { float s = 0; for (int j = 0; j < m; j++) s += Quu[i * m + j] * du[j]; Qd[i] = s; }
    __syncthreads();
    if (tid == 0) {
      float d0 = 0, d1 = 0;
      for (int i = 0; i < m; i++) { d0 += du[i] * Qu[i]; d1 += 0.5f * du[i] * Qd[i]; }
      s_dV[0] += d0; s_dV[1] += d1;
    }
    // T1[0:m*n] = Quu K
    for (int e = tid; e < m * n; e += nt) { const int i = e / n, j = e - i * n; float s = 0; for (int k = 0; k < m; k++) s += Quu[i * m + k] * K[k * n + j]; T1[e] = s; }
    __syncthreads();
    // new value function: Vx -> Wx, Vxx -> At (scratch) then symmetrised into W
    for (int i = tid; i < n; i += nt) {
      float s = Qx[i];
      for (int k = 0; k < m; k++) s += K[k * n + i] * (Qd[k] + Qu[k]) + Qxu[i * m + k] * du[k];
      Qx[i] = s;
    }
    for (int e = tid; e < n * n; e += nt) {
      const int i = e / n, j = e - i * n;
      float s = Qxx[e];
      for (int k = 0; k < m; k++) s += K[k * n + i] * T1[k * n + j] + Qxu[i * m + k] * K[k * n + j] + K[k * n + i] * Qxu[j * m + k];
      At[e] = s;
    }
    __syncthreads();
    for (int i = tid; i < n; i += nt) { Wx[i] = Qx[i]; if (P.Vx) P.Vx[(size_t)t * n + i] = Qx[i]; }
    for (int e = tid; e < n * n; e += nt) {
      const int i = e / n, j = e - i * n;
      const float v = 0.5f * (At[i * n + j] + At[j * n + i]);
      W[e] = v;
      if (P.Vxx) P.Vxx[(size_t)t * n * n + e] = v;
    }
    for (int e = tid; e < m * n; e += nt) P.K[(size_t)t * m * n + e] = K[e];
    for (int i = tid; i < m; i += nt) P.du[(size_t)t * m + i] = du[i];
    __syncthreads();
  }
  if (s_ok) {
    for (int e = tid; e < m * n; e += nt) P.K[(size_t)(H - 1) * m * n + e] = P.K[(size_t)(H - 2) * m * n + e];
    for (int i = tid; i < m; i += nt) P.du[(size_t)(H - 1) * m + i] = P.du[(size_t)(H - 2) * m + i];
  }
  if (tid == 0) { P.dV[0] = s_dV[0]; P.dV[1] = s_dV[1]; *P.status = s_ok; }
}

// ------------------------------------------------------------------------------------------ gradient sweep
// Gradient::Compute (mjpc/planners/gradient/gradient.cc:76-107), the loop of the host GradientSweep
// (csrc/host/gradient_planner.cc) in fp64, one CTA per problem:
//   Vx = cx[T-1];  for t = T-1 .. 1:  Qx = cx[t-1] + A[t-1]' Vx,  Qu = cu[t-1] + B[t-1]' Vx,  k[t-1] = -Qu,
//   dV0 += -Qu . Qu,  Vx = Qx;  k[T-1] = k[T-2].
// Thread j < n sums Qx[j], thread n + j sums Qu[j], each serially over i in the host's order from (double)cx / cu, so
// that reads of A[t-1] / B[t-1] rows are coalesced over j.  Thread 0 accumulates dV0 in the host's (t descending,
// j ascending) order.  Every product and sum is rounded on its own (__dmul_rn / __dadd_rn: -use_fast_math would contract
// them into DFMA), which makes k and dV0 bitwise the host's (baseline x86-64: no FMA).
struct GradientArgs {
  const float *A, *B, *cx, *cu;   // [nprob][H][..] as the derivative sweeps leave them
  double *k, *dV0;                // [nprob][H][m], [nprob]
  int n, m, H;
};

extern "C" __global__ void __launch_bounds__(128) gradient_sweep_kernel(const __grid_constant__ GradientArgs P) {
  extern __shared__ __align__(16) double gsm[];
  const int n = P.n, m = P.m, H = P.H, tid = threadIdx.x, nt = blockDim.x, b = blockIdx.x;
  // smem: Vx [2][n] and Qu [2][m], ping-pong by step parity (cur)
  const float* A = P.A + (size_t)b * H * n * n;
  const float* Bm = P.B + (size_t)b * H * n * m;
  const float* cx = P.cx + (size_t)b * H * n;
  const float* cu = P.cu + (size_t)b * H * m;
  double* k = P.k + (size_t)b * H * m;
  for (int j = tid; j < n; j += nt) gsm[j] = (double)cx[(size_t)(H - 1) * n + j];
  __syncthreads();
  double dV0 = 0.0;
  int cur = 0;
  for (int t = H - 1; t > 0; t--) {
    const double* Vx = gsm + cur * n;
    double* Vn = gsm + (cur ^ 1) * n;
    double* Qu = gsm + 2 * n + cur * m;
    for (int j = tid; j < n + m; j += nt) {
      if (j < n) {
        const float* At = A + (size_t)(t - 1) * n * n;
        double a = (double)cx[(size_t)(t - 1) * n + j];
        for (int i = 0; i < n; i++) a = __dadd_rn(a, __dmul_rn((double)At[(size_t)i * n + j], Vx[i]));
        Vn[j] = a;
      } else {
        const int ju = j - n;
        const float* Bt = Bm + (size_t)(t - 1) * n * m;
        double a = (double)cu[(size_t)(t - 1) * m + ju];
        for (int i = 0; i < n; i++) a = __dadd_rn(a, __dmul_rn((double)Bt[(size_t)i * m + ju], Vx[i]));
        Qu[ju] = a;
        k[(size_t)(t - 1) * m + ju] = -a;
        if (t == H - 1) k[(size_t)(H - 1) * m + ju] = -a;   // row H-1 repeats row H-2
      }
    }
    __syncthreads();
    // this step's Qu is rewritten two steps later, after the next barrier, which thread 0 reaches only once it has read it
    if (tid == 0)
      for (int j = 0; j < m; j++) dV0 = __dadd_rn(dV0, __dmul_rn(-Qu[j], Qu[j]));
    cur ^= 1;
  }
  if (tid == 0) P.dV0[b] = dV0;
}

// ------------------------------------------------------------------------------------------ host launchers
// (the dynamic shared-memory opt-in is a per-kernel, process-wide attribute: only ever raised; handles may be created
// from several threads, hence the lock)
inline cudaError_t raise_smem_limit(const void* fn, size_t bytes) {
  static std::vector<std::pair<const void*, size_t>> seen;
  static std::mutex mtx;
  const std::lock_guard<std::mutex> lock(mtx);
  // a refused request (more than the device allows) is not recorded, and its error is cleared so that it does not
  // surface in a later call's error check
  auto set = [&]() {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) cudaGetLastError();
    return e;
  };
  for (auto& e : seen)
    if (e.first == fn) {
      if (e.second >= bytes) return cudaSuccess;
      const cudaError_t r = set();
      if (r == cudaSuccess) e.second = bytes;
      return r;
    }
  const cudaError_t r = set();
  if (r == cudaSuccess) seen.emplace_back(fn, bytes);
  return r;
}

// fn(A) on grid x block threads, as fn<<<grid, block, smem, st>>>(A) would launch it (a launch error surfaces at the
// caller's cudaGetLastError)
template <class Args>
inline void launch_kernel(const void* fn, dim3 grid, int block, size_t smem, cudaStream_t st, const Args& A) {
  void* args[] = {const_cast<Args*>(&A)};
  cudaLaunchKernel(fn, grid, dim3(block), args, smem, st);
}

// Device buffers of the iLQG sweeps for up to `nprob` problems of max_horizon rows each (per-problem arrays are
// [nprob][H][..]); sized for one problem at create, grown by ilqg_reserve when a batched sweep needs more.  The arrays
// are carved from one owned allocation, every piece 256-byte aligned as an allocation of its own would be.
struct IlqgBuffers {
  int H = 0, ds = 0, n = 0, nu = 0, nr = 0, nv = 0, nprob = 0;
  float *x = nullptr, *u = nullptr, *t = nullptr, *mocap = nullptr, *ts = nullptr, *w = nullptr, *prm = nullptr,
        *y0 = nullptr, *r0 = nullptr, *q0 = nullptr, *A = nullptr, *B = nullptr, *C = nullptr, *D = nullptr,
        *res = nullptr, *cx = nullptr, *cu = nullptr, *cxx = nullptr, *cuu = nullptr, *cxu = nullptr, *act = nullptr,
        *K = nullptr, *du = nullptr, *dV = nullptr, *Vx = nullptr, *Vxx = nullptr, *mu = nullptr, *yp = nullptr,
        *rp = nullptr, *iw = nullptr;
  double *gk = nullptr, *gdV = nullptr;   // gradient sweep: k [nprob][H][nu], dV0 [nprob]
  int* status = nullptr;
  int* idx = nullptr;   // [4 H]: evaluate list, then interpolate t / e0 / e1 (common to all problems)
  mjpc_mem::DeviceArray<unsigned char> mem;
};

// allocates everything for nprob problems into an empty b; on failure -4
inline int ilqg_init(IlqgBuffers& b, const DevModel& M, int H, int nprob = 1) {
  b.H = H; b.nv = M.nv; b.ds = M.nq + M.nv; b.n = 2 * M.nv; b.nu = M.nu; b.nr = M.num_residual; b.nprob = nprob;
  const size_t Hs = H, n = b.n, m = b.nu, nr = b.nr, ds = b.ds, P = nprob;
  // two passes over the fields: the first sizes the allocation (base null), the second points each field into it
  unsigned char* base = nullptr;
  size_t bytes = 0;
  auto take = [&](auto*& p, size_t count) {
    using T = std::remove_reference_t<decltype(*p)>;
    p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (std::max<size_t>(count, 1) * sizeof(T) + 255) & ~(size_t)255;
  };
  auto carve = [&] {
    take(b.x, P * Hs * ds); take(b.u, P * Hs * m); take(b.t, P * Hs); take(b.mocap, P * 7 * (size_t)M.nmocap + 1);
    take(b.ts, P * M.task_state_size + 1); take(b.w, P * M.num_term + 1); take(b.prm, P * M.num_parameters + 1);
    take(b.y0, P * Hs * ds); take(b.r0, P * Hs * nr); take(b.q0, P * Hs * M.nv); take(b.A, P * Hs * n * n);
    take(b.B, P * Hs * n * m); take(b.C, P * Hs * nr * n); take(b.D, P * Hs * nr * m); take(b.res, P * Hs * nr);
    take(b.cx, P * Hs * n); take(b.cu, P * Hs * m); take(b.cxx, P * Hs * n * n); take(b.cuu, P * Hs * m * m);
    take(b.cxu, P * Hs * n * m); take(b.act, P * Hs * m); take(b.K, P * Hs * m * n); take(b.du, P * Hs * m);
    take(b.dV, 2 * P); take(b.Vx, P * Hs * n); take(b.Vxx, P * Hs * n * n); take(b.mu, P);
    take(b.yp, P * (Hs + 2) * (m + n) * ds); take(b.rp, P * (Hs + 2) * (m + n) * nr + 1); take(b.iw, Hs + 1);
    take(b.gk, P * Hs * m); take(b.gdV, P); take(b.status, P); take(b.idx, 4 * Hs + 8);
  };
  carve();
  if (b.mem.alloc(bytes)) return -4;
  base = b.mem; bytes = 0;
  carve();
  return 0;
}

// grow b to hold nprob problems (never shrinks).  On an allocation failure b keeps its old buffers and stays usable.
inline int ilqg_reserve(IlqgBuffers& b, const DevModel& M, int nprob, cudaStream_t st) {
  if (nprob <= b.nprob) return 0;
  IlqgBuffers nb;
  if (int rc = ilqg_init(nb, M, b.H, nprob)) return rc;
  if (cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return -4; }
  b = std::move(nb);
  return 0;
}

#define ILQG_TRY(e) do { if ((e) != cudaSuccess) { cudaGetLastError(); return -4; } } while (0)

// nprob problems with common H / skip / mode, on the fd_center / fd_column instances given.  Host inputs are [nprob][..]:
// x, u, trel (relative to each problem's t[0]), mocap, ts (rebased likewise); w / prm (float weights / parameters) may
// be nullptr for the packed values.  A NULL host output A / B / C / D is not copied back: it stays in b only.  With
// pack_stride != 0, problem p runs on model variant pack_index[p] (FdArgs).
inline int ilqg_model_derivatives(IlqgBuffers& b, const DevModel& M, const float* d_pack, int pack_stride,
                                  const int* pack_index, cudaStream_t st,
                                  const void* fd_center, const void* fd_column, int nprob,
                                  const float* x, const float* u, const float* trel, const float* mocap, const float* ts,
                                  const float* w, const float* prm, int H, float eps, float* A, float* B, float* C,
                                  float* D, size_t smem, int* launches, cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr,
                                  int skip = 0, int mode = 0) {
  const size_t n = b.n, m = b.nu, nr = b.nr, ds = b.ds, P = nprob;
  ILQG_TRY(cudaMemcpyAsync(b.x, x, P * H * ds * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.u, u, P * H * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.t, trel, P * H * 4, cudaMemcpyHostToDevice, st));
  if (M.nmocap) ILQG_TRY(cudaMemcpyAsync(b.mocap, mocap, P * 7 * M.nmocap * 4, cudaMemcpyHostToDevice, st));
  if (M.task_state_size) ILQG_TRY(cudaMemcpyAsync(b.ts, ts, P * M.task_state_size * 4, cudaMemcpyHostToDevice, st));
  if (w && M.num_term) ILQG_TRY(cudaMemcpyAsync(b.w, w, P * M.num_term * 4, cudaMemcpyHostToDevice, st));
  if (prm && M.num_parameters) ILQG_TRY(cudaMemcpyAsync(b.prm, prm, P * M.num_parameters * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemsetAsync(b.A, 0, P * H * n * n * 4, st)); ILQG_TRY(cudaMemsetAsync(b.B, 0, P * H * n * m * 4, st));
  ILQG_TRY(cudaMemsetAsync(b.C, 0, P * H * nr * n * 4, st)); ILQG_TRY(cudaMemsetAsync(b.D, 0, P * H * nr * m * 4, st));
  // evaluate / interpolate lists exactly as ModelDerivatives::Compute builds them (model_derivatives.cc:56-72)
  std::vector<int> ev, it_t, it_e0, it_e1;
  std::vector<float> it_w;
  if (H >= 2) {
    const int s2 = skip + 1;
    ev.push_back(0);
    for (int t = s2; t < H - s2; t += s2) ev.push_back(t);
    ev.push_back(H - 2); ev.push_back(H - 1);
    for (int t = 0, e = 0; t < H; t++) {
      if (e == (int)ev.size() || ev[e] > t) {
        int upper = 0;                                  // FindInterval (utilities.h:125-144)
        while (upper < (int)ev.size() && !(t < ev[upper])) upper++;
        const int lower = upper - 1;
        int b0, b1;
        if (lower < 0) b0 = b1 = 0;
        else if (lower > (int)ev.size() - 1) b0 = b1 = (int)ev.size() - 1;
        else { b0 = std::max(lower, 0); b1 = std::min(upper, (int)ev.size() - 1); }
        it_t.push_back(t); it_e0.push_back(ev[b0]); it_e1.push_back(ev[b1]);
        it_w.push_back(b0 == b1 ? 0.f : (float)(double(t - ev[b0]) / double(ev[b1] - ev[b0])));
      } else e++;
    }
    // drop duplicate evaluations (T-2 appears twice when skip = 0): same result, half the work
    std::vector<int> uniq;
    for (int t : ev) if (std::find(uniq.begin(), uniq.end(), t) == uniq.end()) uniq.push_back(t);
    ev = uniq;
  } else ev.push_back(0);
  const int neval = (int)ev.size(), ninterp = (int)it_t.size();
  ILQG_TRY(cudaMemcpyAsync(b.idx, ev.data(), neval * 4, cudaMemcpyHostToDevice, st));
  if (ninterp) {
    ILQG_TRY(cudaMemcpyAsync(b.idx + H + 2, it_t.data(), ninterp * 4, cudaMemcpyHostToDevice, st));
    ILQG_TRY(cudaMemcpyAsync(b.idx + 2 * H + 4, it_e0.data(), ninterp * 4, cudaMemcpyHostToDevice, st));
    ILQG_TRY(cudaMemcpyAsync(b.idx + 3 * H + 6, it_e1.data(), ninterp * 4, cudaMemcpyHostToDevice, st));
    ILQG_TRY(cudaMemcpyAsync(b.iw, it_w.data(), ninterp * 4, cudaMemcpyHostToDevice, st));
  }
  ILQG_TRY(cudaStreamSynchronize(st));   // the index vectors are pageable host memory
  FdArgs a;
  std::memset(&a, 0, sizeof(a));
  a.eval_t = b.idx; a.neval = neval; a.mode = mode; a.yp = b.yp; a.rp = b.rp;
  a.M = M; a.L = make_layout(M, 1); a.pack = d_pack; a.pack_stride = pack_stride; a.pack_index = pack_index; a.x = b.x; a.u = b.u; a.t = b.t; a.mocap = b.mocap;
  a.task_state = M.task_state_size ? b.ts : nullptr; a.H = H; a.eps = eps; a.y0 = b.y0; a.r0 = b.r0; a.q0 = b.q0;
  a.weight = (w && M.num_term) ? b.w : nullptr; a.parameters = (prm && M.num_parameters) ? b.prm : nullptr;
  a.A = b.A; a.B = b.B; a.C = b.C; a.D = b.D;
  if (e0) ILQG_TRY(cudaEventRecord(e0, st));   // kernel-only span (copies and memsets stay outside)
  launch_kernel(fd_center, dim3(neval, nprob), 32, smem, st, a);
  launch_kernel(fd_column, dim3(neval * (M.nu + 2 * M.nv), nprob), 32, smem, st, a);
  *launches += 2;
  if (ninterp) {
    FdInterpArgs ia;
    ia.t = b.idx + H + 2; ia.e0 = b.idx + 2 * H + 4; ia.e1 = b.idx + 3 * H + 6; ia.w = b.iw;
    ia.A = b.A; ia.B = b.B; ia.C = b.C; ia.D = b.D;
    ia.nA = (int)(n * n); ia.nB = (int)(n * m); ia.nC = (int)(nr * n); ia.nD = (int)(nr * m); ia.H = H;
    fd_interp_kernel<<<dim3(ninterp, nprob), 256, 0, st>>>(ia);
    *launches += 1;
  }
  if (e1) ILQG_TRY(cudaEventRecord(e1, st));
  ILQG_TRY(cudaGetLastError());
  if (A) ILQG_TRY(cudaMemcpyAsync(A, b.A, P * H * n * n * 4, cudaMemcpyDeviceToHost, st));
  if (B) ILQG_TRY(cudaMemcpyAsync(B, b.B, P * H * n * m * 4, cudaMemcpyDeviceToHost, st));
  if (C) ILQG_TRY(cudaMemcpyAsync(C, b.C, P * H * nr * n * 4, cudaMemcpyDeviceToHost, st));
  if (D) ILQG_TRY(cudaMemcpyAsync(D, b.D, P * H * nr * m * 4, cudaMemcpyDeviceToHost, st));
  if (A || B || C || D) ILQG_TRY(cudaStreamSynchronize(st));
  return 0;
}

// dynamic shared memory of cost_derivatives_kernel for a model whose widest cost term has kmax residuals
inline size_t cost_derivatives_smem(const DevModel& M, int kmax) {
  const size_t n = 2 * (size_t)M.nv, m = M.nu, nr = M.num_residual, k = kmax;
  return (nr + k * k + k * n + k * m + n + m + n * n + m * m + n * m + 8) * 4;
}

// nprob problems; w [nprob][num_term] (float) or nullptr for the packed Task::weight; kmax = the widest cost term
// (the kernel lays its scratch out with it: the caller checks cost_derivatives_smem against the device limit).
// cd_resident: C and D are already in b (the model-derivative sweep just left them there) and are not uploaded.  A NULL
// host output is not copied back.
inline int ilqg_cost_derivatives(IlqgBuffers& b, const DevModel& M, const float* d_pack, cudaStream_t st, int nprob,
                                 const float* w, const float* residual, const float* C, const float* D, int H, float* cx,
                                 float* cu, float* cxx, float* cuu, float* cxu, int kmax, int* launches,
                                 cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr, bool cd_resident = false) {
  const size_t n = b.n, m = b.nu, nr = b.nr, P = nprob;
  ILQG_TRY(cudaMemcpyAsync(b.res, residual, P * H * nr * 4, cudaMemcpyHostToDevice, st));
  if (!cd_resident) {
    ILQG_TRY(cudaMemcpyAsync(b.C, C, P * H * nr * n * 4, cudaMemcpyHostToDevice, st));
    ILQG_TRY(cudaMemcpyAsync(b.D, D, P * H * nr * m * 4, cudaMemcpyHostToDevice, st));
  }
  if (w && M.num_term) ILQG_TRY(cudaMemcpyAsync(b.w, w, P * M.num_term * 4, cudaMemcpyHostToDevice, st));
  CostArgs a;
  std::memset(&a, 0, sizeof(a));
  a.M = M; a.pack = d_pack; a.residual = b.res; a.C = b.C; a.D = b.D; a.H = H; a.n = (int)n; a.m = (int)m;
  a.weight = (w && M.num_term) ? b.w : nullptr;
  a.cx = b.cx; a.cu = b.cu; a.cxx = b.cxx; a.cuu = b.cuu; a.cxu = b.cxu;
  const size_t smem = cost_derivatives_smem(M, kmax);
  ILQG_TRY(raise_smem_limit((const void*)cost_derivatives_kernel, smem));
  if (e0) ILQG_TRY(cudaEventRecord(e0, st));
  cost_derivatives_kernel<<<dim3(H, nprob), 256, smem, st>>>(a);
  if (e1) ILQG_TRY(cudaEventRecord(e1, st));
  *launches += 1;
  ILQG_TRY(cudaGetLastError());
  if (cx) ILQG_TRY(cudaMemcpyAsync(cx, b.cx, P * H * n * 4, cudaMemcpyDeviceToHost, st));
  if (cu) ILQG_TRY(cudaMemcpyAsync(cu, b.cu, P * H * m * 4, cudaMemcpyDeviceToHost, st));
  if (cxx) ILQG_TRY(cudaMemcpyAsync(cxx, b.cxx, P * H * n * n * 4, cudaMemcpyDeviceToHost, st));
  if (cuu) ILQG_TRY(cudaMemcpyAsync(cuu, b.cuu, P * H * m * m * 4, cudaMemcpyDeviceToHost, st));
  if (cxu) ILQG_TRY(cudaMemcpyAsync(cxu, b.cxu, P * H * n * m * 4, cudaMemcpyDeviceToHost, st));
  if (cx || cu || cxx || cuu || cxu) ILQG_TRY(cudaStreamSynchronize(st));
  return 0;
}

// the gradient sweep of nprob problems on the A, B, cx and cu the derivative sweeps left in b; k [nprob][H][nu] and
// dV0 [nprob] (double) copied to the host
inline int ilqg_gradient_sweep(IlqgBuffers& b, cudaStream_t st, int nprob, int H, double* k, double* dV0, int* launches,
                               cudaEvent_t e1 = nullptr) {
  const size_t m = b.nu, P = nprob;
  GradientArgs a;
  a.A = b.A; a.B = b.B; a.cx = b.cx; a.cu = b.cu; a.k = b.gk; a.dV0 = b.gdV; a.n = b.n; a.m = b.nu; a.H = H;
  gradient_sweep_kernel<<<nprob, 128, (2 * b.n + 2 * b.nu) * sizeof(double), st>>>(a);
  if (e1) ILQG_TRY(cudaEventRecord(e1, st));
  *launches += 1;
  ILQG_TRY(cudaGetLastError());
  ILQG_TRY(cudaMemcpyAsync(k, b.gk, P * H * m * sizeof(double), cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaMemcpyAsync(dV0, b.gdV, P * sizeof(double), cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaStreamSynchronize(st));
  return 0;
}

// nprob problems, one CTA each; mu [nprob], dV [nprob][2], status_out [nprob]
inline int ilqg_backward_pass(IlqgBuffers& b, const DevModel& M, const float* d_pack, cudaStream_t st, int nprob,
                              const float* A, const float* B, const float* cx, const float* cu, const float* cxx,
                              const float* cxu, const float* cuu, const float* actions, int H, const float* mu,
                              int reg_type, int limits, float* K, float* du, float* dV, float* Vx, float* Vxx,
                              int* status_out, int* launches, cudaEvent_t e0 = nullptr, cudaEvent_t e1 = nullptr) {
  const size_t n = b.n, m = b.nu, P = nprob;
  if (m > 32) return -5;
  ILQG_TRY(cudaMemcpyAsync(b.A, A, P * H * n * n * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.B, B, P * H * n * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.cx, cx, P * H * n * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.cu, cu, P * H * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.cxx, cxx, P * H * n * n * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.cxu, cxu, P * H * n * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.cuu, cuu, P * H * m * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.act, actions, P * H * m * 4, cudaMemcpyHostToDevice, st));
  ILQG_TRY(cudaMemcpyAsync(b.mu, mu, P * 4, cudaMemcpyHostToDevice, st));
  BackwardArgs a;
  std::memset(&a, 0, sizeof(a));
  a.A = b.A; a.B = b.B; a.cx = b.cx; a.cu = b.cu; a.cxx = b.cxx; a.cxu = b.cxu; a.cuu = b.cuu; a.actions = b.act;
  a.ctrlrange = d_pack + M.fo[F_actuator_ctrlrange];
  a.n = (int)n; a.m = (int)m; a.H = H; a.reg_type = reg_type; a.limits = limits; a.mu = b.mu;
  a.K = b.K; a.du = b.du; a.dV = b.dV; a.Vx = b.Vx; a.Vxx = b.Vxx; a.status = b.status;
  const size_t smem = (4 * n * n + 3 * n * m + 3 * m * m + m * n + 2 * n + 12 * m + 9 * m + 16) * 4;
  ILQG_TRY(raise_smem_limit((const void*)backward_pass_kernel, smem));
  if (e0) ILQG_TRY(cudaEventRecord(e0, st));
  backward_pass_kernel<<<nprob, kBackwardThreads, smem, st>>>(a);
  if (e1) ILQG_TRY(cudaEventRecord(e1, st));
  *launches += 1;
  ILQG_TRY(cudaGetLastError());
  ILQG_TRY(cudaMemcpyAsync(K, b.K, P * H * m * n * 4, cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaMemcpyAsync(du, b.du, P * H * m * 4, cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaMemcpyAsync(dV, b.dV, P * 2 * 4, cudaMemcpyDeviceToHost, st));
  if (Vx) ILQG_TRY(cudaMemcpyAsync(Vx, b.Vx, P * H * n * 4, cudaMemcpyDeviceToHost, st));
  if (Vxx) ILQG_TRY(cudaMemcpyAsync(Vxx, b.Vxx, P * H * n * n * 4, cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaMemcpyAsync(status_out, b.status, P * 4, cudaMemcpyDeviceToHost, st));
  ILQG_TRY(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace mjpc_dev
