// estimator_kernels.cuh - the Kalman and Unscented filters (csrc/host/estimator.h) on the device: B filters of one
// kind, one CTA per filter, in fp64.  The kernels restate the reference's filters (mjpc/estimators/unscented.cc,
// kalman.cc) as the Python mirror mujoco_mpc_b200/estimator.py (Unscented, Kalman) writes them, with each output summed
// in a fixed serial order and every product that feeds a sum rounded on its own (__dmul_rn / __dadd_rn: the build's
// -use_fast_math contracts plain a * b + c into an FMA), so results do not depend on the compiler's contractions.
// Rows of the step launch: filter b owns rows [b rows, (b + 1) rows), laid out as the mirror's backend call
// (Unscented: the 2 ndstate sigma points, nominal last; Kalman: the centre, then the perturbations).
//
//   estimator_rows_kernel      the step inputs of every row: state, ctrl, warm start and mocap of its filter
//                              (Unscented: the Cholesky factor of P first; a factor that is not full rank fails the
//                              filter: a pivot below 1e-15 or not finite)
//   step_batch_kernel*         one launch of all B rows (engine.cu), the measurement sensors of each pre-step state
//   unscented_update_kernel    means, QuaternionMeans, differences, covariances, gain update, state and time
//   kalman_measurement_kernel  C, S = C P C' + R, gain update, correction
//   kalman_prediction_kernel   A, P = A P A' + Q, the centre's next state, time
//
// A failed factorisation sets status[b] to the factor's mjpc_b200_bank::Status, and an update whose new state or
// covariance is not finite sets NONFINITE_RESULT; either leaves filter b's state, covariance, time, warm start and
// warnings untouched, and the other filters do not depend on it.  Every update is formed in scratch (the new state,
// o_Pn the new covariance) and committed only once all of it is finite.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>

#include "filter_bank.h"

namespace mjpc_dev {

constexpr int kFilterThreads = 128;
constexpr int kFilterKalman = 1, kFilterUnscented = 2;   // the reference's `estimator` numeric (estimators/include.cc)

struct FilterBankArgs {
  int nq, nv, nu, nmocap, njnt;
  const int* jnt;   // [3][njnt]: type, qposadr, dofadr
  int kind, B, rows, ny, phase;
  double timestep, sigma_step, weight_mean0, weight_covariance0, weight_sigma, epsilon;
  int centered;
  // per filter, persistent: state [nq+nv], covariance [ndstate^2], time, noise, warm start [nv] and warnings
  double *state, *P, *time, *noise_process, *noise_sensor;
  float* warm;
  int* warnings;
  // per filter, per update: ctrl [nu], measured sensors [ny], mocap [7 nmocap]; status
  const float* ctrl; const double* sensor; const float* mocap;
  int* status;
  // the step launch's rows: inputs written by estimator_rows_kernel, outputs read by the update kernels
  float *qpos, *qvel, *rctrl, *rwarm, *rmocap;
  const float *qacc, *next_qpos, *next_qvel, *sensordata;
  const int* counts;
  // per filter scratch [scratch_words] and its offsets
  double* scratch;
  size_t scratch_words;
  int o_F, o_mean, o_ymean, o_ds, o_dy, o_S, o_X, o_P0, o_T, o_C, o_e, o_corr, o_rows, o_Pn;
};

// the per-filter scratch offsets (doubles) for ndstate ns, nx = nq + nv, ny sensor values and R rows; returns the total
inline size_t filter_scratch_layout(FilterBankArgs& a) {
  const int ns = 2 * a.nv, nx = a.nq + a.nv, ny = a.ny, R = a.rows;
  size_t w = 0;
  auto take = [&](size_t n) { const int at = (int)w; w += (n + 1) & ~(size_t)1; return at; };
  a.o_F = take((size_t)ns * ns); a.o_mean = take(nx); a.o_ymean = take(ny); a.o_ds = take((size_t)R * ns);
  a.o_dy = take((size_t)R * ny); a.o_S = take((size_t)ny * ny); a.o_X = take((size_t)ns * ny);
  a.o_P0 = take((size_t)ns * ns); a.o_T = take((size_t)ns * ny); a.o_C = take((size_t)ny * ns); a.o_e = take(ny);
  a.o_corr = take(ns); a.o_rows = take((size_t)R * nx); a.o_Pn = take((size_t)ns * ns);
  a.scratch_words = w;
  return w;
}

// ------------------------------------------------------------------------- fp64, every product rounded on its own
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

// o = a * b (quaternions), each component summed left to right as mju_mulQuat writes it
__device__ inline void fb_quat_mul(double* o, const double* a, const double* b) {
  o[0] = dsub(dsub(dsub(dmul(a[0], b[0]), dmul(a[1], b[1])), dmul(a[2], b[2])), dmul(a[3], b[3]));
  o[1] = dsub(dadd(dadd(dmul(a[0], b[1]), dmul(a[1], b[0])), dmul(a[2], b[3])), dmul(a[3], b[2]));
  o[2] = dadd(dadd(dsub(dmul(a[0], b[2]), dmul(a[1], b[3])), dmul(a[2], b[0])), dmul(a[3], b[1]));
  o[3] = dadd(dsub(dadd(dmul(a[0], b[3]), dmul(a[1], b[2])), dmul(a[2], b[1])), dmul(a[3], b[0]));
}

// mju_subQuat: qb * quat(res) = qa (planner.cc SubQuat)
__device__ inline void fb_sub_quat(double* res, const double* qa, const double* qb) {
  const double n[4] = {qb[0], -qb[1], -qb[2], -qb[3]};
  double d[4];
  fb_quat_mul(d, n, qa);
  double axis[3] = {d[1], d[2], d[3]};
  const double s = sqrt(dadd(dadd(dmul(axis[0], axis[0]), dmul(axis[1], axis[1])), dmul(axis[2], axis[2])));
  if (s < 1e-15) { axis[0] = 1; axis[1] = axis[2] = 0; } else { for (int c = 0; c < 3; c++) axis[c] = axis[c] / s; }
  double speed = dmul(2.0, atan2(s, d[0]));
  if (speed > M_PI) speed = dsub(speed, dmul(2.0, M_PI));
  for (int c = 0; c < 3; c++) res[c] = dmul(axis[c], speed);
}

// mju_quatIntegrate: q * exp(scale v / 2), normalised (estimator.py quat_integrate)
__device__ inline void fb_quat_integrate(double* q, const double* v, double scale) {
  const double w[3] = {dmul(v[0], scale), dmul(v[1], scale), dmul(v[2], scale)};
  const double a = sqrt(dadd(dadd(dmul(w[0], w[0]), dmul(w[1], w[1])), dmul(w[2], w[2])));
  double r[4] = {1, 0, 0, 0};
  if (a >= 1e-15) {
    const double s = sin(a / 2) / a;
    r[0] = cos(a / 2); r[1] = dmul(s, w[0]); r[2] = dmul(s, w[1]); r[3] = dmul(s, w[2]);
  }
  double o[4];
  fb_quat_mul(o, q, r);
  const double n = sqrt(dadd(dadd(dadd(dmul(o[0], o[0]), dmul(o[1], o[1])), dmul(o[2], o[2])), dmul(o[3], o[3])));
  for (int k = 0; k < 4; k++) q[k] = o[k] / n;
}

// mj_integratePos: qpos (+) scale dq, dq(k) the tangent vector's entry k (estimator.py integrate_pos)
template <class DQ>
__device__ inline void fb_integrate_pos(const FilterBankArgs& A, double* qpos, DQ dq, double scale) {
  for (int j = 0; j < A.njnt; j++) {
    const int type = A.jnt[j], a = A.jnt[A.njnt + j], d = A.jnt[2 * A.njnt + j];
    if (type == 0 || type == 1) {
      const int p = a + (type == 0 ? 3 : 0), v = d + (type == 0 ? 3 : 0);
      if (type == 0)
        for (int c = 0; c < 3; c++) qpos[a + c] = dadd(qpos[a + c], dmul(scale, dq(d + c)));
      const double w[3] = {dq(v), dq(v + 1), dq(v + 2)};
      fb_quat_integrate(qpos + p, w, scale);
    } else {
      qpos[a] = dadd(qpos[a], dmul(scale, dq(d)));
    }
  }
}

// x (+) scale dx, positions through fb_integrate_pos, velocities added (estimator.py _Filter._state_add)
template <class DQ>
__device__ inline void fb_state_add(const FilterBankArgs& A, double* x, DQ dx, double scale) {
  fb_integrate_pos(A, x, dx, scale);
  for (int k = 0; k < A.nv; k++) x[A.nq + k] = dadd(x[A.nq + k], dmul(scale, dx(A.nv + k)));
}

// StateDiff: dx [2 nv] = x_to (-) x_from (planner.cc)
__device__ inline void fb_state_diff(const FilterBankArgs& A, double* dx, const double* x_to, const double* x_from) {
  for (int j = 0; j < A.njnt; j++) {
    const int type = A.jnt[j], qa = A.jnt[A.njnt + j], da = A.jnt[2 * A.njnt + j];
    if (type == 0) {
      for (int c = 0; c < 3; c++) dx[da + c] = dsub(x_to[qa + c], x_from[qa + c]);
      fb_sub_quat(&dx[da + 3], x_to + qa + 3, x_from + qa + 3);
    } else if (type == 1) {
      fb_sub_quat(&dx[da], x_to + qa, x_from + qa);
    } else {
      dx[da] = dsub(x_to[qa], x_from[qa]);
    }
  }
  for (int i = 0; i < A.nv; i++) dx[A.nv + i] = dsub(x_to[A.nq + i], x_from[A.nq + i]);
}

// ------------------------------------------------------------------------------------------ block-wide linear algebra
// CholFactor (mju_cholFactor) of the row-major n x n M in place, pivots below mindiag raised to it; every thread gets
// the rank, which counts the pivots >= mindiag that are finite (a NaN or infinite pivot is raised to mindiag and not
// counted).  Column j: thread 0 forms the pivot, then the rows below it in parallel, each summed serially.
__device__ inline int fb_chol_factor(double* M, int n, double mindiag) {
  __shared__ int rank;
  if (threadIdx.x == 0) rank = 0;
  for (int j = 0; j < n; j++) {
    if (threadIdx.x == 0) {
      double d = M[(size_t)j * n + j];
      for (int k = 0; k < j; k++) d = dsub(d, dmul(M[(size_t)j * n + k], M[(size_t)j * n + k]));
      if (d >= mindiag && d <= DBL_MAX) rank++; else d = mindiag;
      M[(size_t)j * n + j] = sqrt(d);
    }
    __syncthreads();
    const double djj = M[(size_t)j * n + j];
    for (int i = j + 1 + threadIdx.x; i < n; i += blockDim.x) {
      double a = M[(size_t)i * n + j];
      for (int k = 0; k < j; k++) a = dsub(a, dmul(M[(size_t)i * n + k], M[(size_t)j * n + k]));
      M[(size_t)i * n + j] = a / djj;
    }
    __syncthreads();
  }
  const int r = rank;
  __syncthreads();
  return r;
}

// CholSolve (mju_cholSolve) by one thread: x = (L L')^-1 x
__device__ inline void fb_chol_solve(const double* L, int n, double* x) {
  for (int i = 0; i < n; i++) {
    double a = x[i];
    for (int k = 0; k < i; k++) a = dsub(a, dmul(L[(size_t)i * n + k], x[k]));
    x[i] = a / L[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    double a = x[i];
    for (int k = i + 1; k < n; k++) a = dsub(a, dmul(L[(size_t)k * n + i], x[k]));
    x[i] = a / L[(size_t)i * n + i];
  }
}

// true on every thread when the n values v are all finite
__device__ inline bool fb_all_finite(const double* v, int n) {
  int bad = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) bad |= !(fabs(v[i]) <= DBL_MAX);
  return !__syncthreads_or(bad);
}

// P [n]^2 = (P + P') / 2, each pair by one thread
__device__ inline void fb_symmetrize(double* P, int n) {
  for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
    const int r = i / n, c = i - r * n;
    if (c <= r) continue;
    const double s = dmul(0.5, dadd(P[(size_t)r * n + c], P[(size_t)c * n + r]));
    P[(size_t)r * n + c] = P[(size_t)c * n + r] = s;
  }
  __syncthreads();
}

// The gain update (estimator.py _Filter._gain): corr = X S^-1 e, P = P0 - X S^-1 X' symmetrised (P may alias P0), with X [ns][ny] and S
// [ny]^2 (overwritten by its factor), e (overwritten by S^-1 e) and T [ns][ny] scratch.  false, with corr and P
// untouched, when S is not full rank.
__device__ inline bool fb_gain_update(const double* X, double* S, double* e, const double* P0, double* corr, double* P,
                                      double* T, int ns, int ny) {
  if (fb_chol_factor(S, ny, 1e-15) < ny) return false;
  for (int r = threadIdx.x; r <= ns; r += blockDim.x) {   // rows of T = S^-1 X[r], and r = ns: e
    double* x = r < ns ? T + (size_t)r * ny : e;
    if (r < ns) for (int c = 0; c < ny; c++) x[c] = X[(size_t)r * ny + c];
    fb_chol_solve(S, ny, x);
  }
  __syncthreads();
  for (int r = threadIdx.x; r < ns; r += blockDim.x) {
    double a = 0.0;
    for (int c = 0; c < ny; c++) a = dadd(a, dmul(X[(size_t)r * ny + c], e[c]));
    corr[r] = a;
  }
  for (int i = threadIdx.x; i < ns * ns; i += blockDim.x) {
    const int r = i / ns, c = i - r * ns;
    double a = 0.0;
    for (int k = 0; k < ny; k++) a = dadd(a, dmul(X[(size_t)r * ny + k], T[(size_t)c * ny + k]));
    P[i] = dsub(P0[i], a);
  }
  __syncthreads();
  fb_symmetrize(P, ns);
  return true;
}

// Principal eigenvector of a symmetric 4 x 4 matrix by cyclic Jacobi rotations, signed to agree with ref (estimator.py
// principal_eigenvector4), by one thread
__device__ inline void fb_principal_eigenvector4(double* out, const double* K, const double* ref) {
  double Am[16], V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int k = 0; k < 16; k++) Am[k] = K[k];
  for (int sweep = 0; sweep < 50; sweep++) {
    double off = 0;
    for (int p = 0; p < 4; p++) for (int q = p + 1; q < 4; q++) off = dadd(off, dmul(Am[4 * p + q], Am[4 * p + q]));
    if (off < 1e-300) break;
    for (int p = 0; p < 4; p++)
      for (int q = p + 1; q < 4; q++) {
        if (Am[4 * p + q] == 0) continue;
        const double th = dsub(Am[4 * q + q], Am[4 * p + p]) / dmul(2.0, Am[4 * p + q]);
        const double t = fabs(th) > 1e150 ? 0.5 / th
                                          : (th >= 0 ? 1.0 : -1.0) / dadd(fabs(th), sqrt(dadd(dmul(th, th), 1.0)));
        const double c = 1 / sqrt(dadd(dmul(t, t), 1.0)), s = dmul(t, c);
        for (int k = 0; k < 4; k++) {
          const double akp = Am[4 * k + p], akq = Am[4 * k + q];
          Am[4 * k + p] = dsub(dmul(c, akp), dmul(s, akq)); Am[4 * k + q] = dadd(dmul(s, akp), dmul(c, akq));
        }
        for (int k = 0; k < 4; k++) {
          const double apk = Am[4 * p + k], aqk = Am[4 * q + k];
          Am[4 * p + k] = dsub(dmul(c, apk), dmul(s, aqk)); Am[4 * q + k] = dadd(dmul(s, apk), dmul(c, aqk));
        }
        for (int k = 0; k < 4; k++) {
          const double vkp = V[4 * k + p], vkq = V[4 * k + q];
          V[4 * k + p] = dsub(dmul(c, vkp), dmul(s, vkq)); V[4 * k + q] = dadd(dmul(s, vkp), dmul(c, vkq));
        }
      }
  }
  int best = 0;
  for (int k = 1; k < 4; k++) if (Am[5 * k] > Am[5 * best]) best = k;
  double dot = 0;
  for (int k = 0; k < 4; k++) dot = dadd(dot, dmul(V[4 * k + best], ref[k]));
  const double sg = dot >= 0 ? 1.0 : -1.0;
  double n = 0;
  for (int k = 0; k < 4; k++) n = dadd(n, dmul(V[4 * k + best], V[4 * k + best]));
  n = sqrt(n);
  for (int k = 0; k < 4; k++) out[k] = dmul(sg, V[4 * k + best]) / n;
}

// ------------------------------------------------------------------------------------------------- shared pieces
// the step outputs of filter b's rows as doubles: rows [R][nx] (next states)
__device__ inline void fb_load_next(const FilterBankArgs& A, int b, double* rows) {
  const int nq = A.nq, nv = A.nv, nx = nq + nv, R = A.rows;
  for (int i = threadIdx.x; i < R * nx; i += blockDim.x) {
    const int r = i / nx, k = i - r * nx;
    const size_t row = (size_t)b * R + r;
    rows[i] = k < nq ? (double)A.next_qpos[row * nq + k] : (double)A.next_qvel[row * nv + k - nq];
  }
  __syncthreads();
}

// After a successful update (estimator.py _Filter._commit): the new state x [nq+nv] and covariance Pn [ndstate^2] from
// scratch when both are finite (else status NONFINITE_RESULT and nothing is written), then time += timestep when
// `advance`, the warm start from row `centre` and the rows' warnings.  true when committed.
__device__ inline bool fb_commit(const FilterBankArgs& A, int b, const double* x, const double* Pn, bool advance,
                                 int centre) {
  const int nx = A.nq + A.nv, ns = 2 * A.nv;
  if (!fb_all_finite(x, nx) || !fb_all_finite(Pn, ns * ns)) {
    if (threadIdx.x == 0) A.status[b] = mjpc_b200_bank::NONFINITE_RESULT;
    return false;
  }
  for (int k = threadIdx.x; k < nx; k += blockDim.x) A.state[(size_t)b * nx + k] = x[k];
  for (int k = threadIdx.x; k < ns * ns; k += blockDim.x) A.P[(size_t)b * ns * ns + k] = Pn[k];
  if (advance && threadIdx.x == 0) A.time[b] = dadd(A.time[b], A.timestep);
  const size_t row0 = (size_t)b * A.rows;
  for (int k = threadIdx.x; k < A.nv; k += blockDim.x) A.warm[(size_t)b * A.nv + k] = A.qacc[(row0 + centre) * A.nv + k];
  if (threadIdx.x == 0) {
    int w = 0;
    for (int i = 0; i < A.rows; i++) w += A.counts[4 * (row0 + i) + 3] != 0;
    A.warnings[b] += w;
  }
  return true;
}

// -------------------------------------------------------------------------------------------------------- kernels
// The step rows of every filter.  phase 0: Unscented sigma points from the Cholesky factor of P (a factor that is not
// full rank fails the filter; its rows then repeat its state).  phase 1: Kalman measurement rows, phase 2: Kalman
// prediction rows, both the centre state and its +-epsilon tangent-space perturbations (estimator.py Kalman.perturbed).
extern "C" __global__ void __launch_bounds__(kFilterThreads) estimator_rows_kernel(const __grid_constant__ FilterBankArgs A) {
  const int b = blockIdx.x, nq = A.nq, nv = A.nv, nx = nq + nv, ns = 2 * nv, R = A.rows;
  double* W = A.scratch + (size_t)b * A.scratch_words;
  double* rows = W + A.o_rows;
  const double* x = A.state + (size_t)b * nx;
  bool ok = true;
  if (A.phase == 0) {
    double* F = W + A.o_F;
    for (int i = threadIdx.x; i < ns * ns; i += blockDim.x) F[i] = A.P[(size_t)b * ns * ns + i];
    __syncthreads();
    ok = fb_chol_factor(F, ns, 1e-15) == ns;
  }
  if (A.phase < 2 && threadIdx.x == 0)
    A.status[b] = ok ? mjpc_b200_bank::UPDATED : mjpc_b200_bank::COVARIANCE_FACTOR_FAILED;
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    double* xr = rows + (size_t)r * nx;
    for (int k = 0; k < nx; k++) xr[k] = x[k];
    if (A.phase == 0) {
      if (!ok || r == R - 1) continue;   // nominal point last
      const int i = r % ns;
      const double* F = W + A.o_F;
      const double step = A.sigma_step;
      fb_state_add(A, xr, [&](int j) { return j >= i ? dmul(step, F[(size_t)j * ns + i]) : 0.0; }, r < ns ? 1.0 : -1.0);
    } else if (r > 0) {
      const int i = (r - 1) % ns;
      const double e = r - 1 < ns ? A.epsilon : -A.epsilon;
      if (i < nv) fb_integrate_pos(A, xr, [&](int j) { return j == i ? 1.0 : 0.0; }, e);
      else xr[nq + i - nv] = dadd(xr[nq + i - nv], e);
    }
  }
  __syncthreads();
  const size_t row0 = (size_t)b * R;
  for (int i = threadIdx.x; i < R * nx; i += blockDim.x) {
    const int r = i / nx, k = i - r * nx;
    if (k < nq) A.qpos[(row0 + r) * nq + k] = (float)rows[i];
    else A.qvel[(row0 + r) * nv + k - nq] = (float)rows[i];
  }
  const int nm = 7 * A.nmocap;
  for (int i = threadIdx.x; i < R * nv; i += blockDim.x) A.rwarm[row0 * nv + i] = A.warm[(size_t)b * nv + i % nv];
  for (int i = threadIdx.x; i < R * A.nu; i += blockDim.x) A.rctrl[row0 * A.nu + i] = A.ctrl[(size_t)b * A.nu + i % A.nu];
  for (int i = threadIdx.x; i < R * nm; i += blockDim.x) A.rmocap[row0 * nm + i] = A.mocap[(size_t)b * nm + i % nm];
}

// Unscented.update after the sigma-point launch (unscented.cc EvaluateSigmaPoints .. Update)
extern "C" __global__ void __launch_bounds__(kFilterThreads) unscented_update_kernel(const __grid_constant__ FilterBankArgs A) {
  const int b = blockIdx.x, nq = A.nq, nv = A.nv, nx = nq + nv, ns = 2 * nv, ny = A.ny, R = A.rows;
  if (A.status[b] != 0) return;
  double* W = A.scratch + (size_t)b * A.scratch_words;
  double *rows = W + A.o_rows, *mean = W + A.o_mean, *ymean = W + A.o_ymean, *ds = W + A.o_ds, *dy = W + A.o_dy,
         *cyy = W + A.o_S, *csy = W + A.o_X, *css = W + A.o_P0, *e = W + A.o_e, *corr = W + A.o_corr;
  const float* ys = A.sensordata + (size_t)b * R * ny;
  fb_load_next(A, b, rows);
  // means: the nominal (last) point weighs weight_mean0, the others weight_sigma
  for (int k = threadIdx.x; k < nx + ny; k += blockDim.x) {
    double a = 0.0;
    for (int i = 0; i < R; i++) {
      const double w = i == R - 1 ? A.weight_mean0 : A.weight_sigma;
      a = dadd(a, dmul(w, k < nx ? rows[(size_t)i * nx + k] : (double)ys[(size_t)i * ny + k - nx]));
    }
    if (k < nx) mean[k] = a; else ymean[k - nx] = a;
  }
  __syncthreads();
  // QuaternionMeans: one thread per free / ball joint, with the covariance weights
  for (int j = threadIdx.x; j < A.njnt; j += blockDim.x) {
    const int type = A.jnt[j];
    if (type != 0 && type != 1) continue;
    const int a = A.jnt[A.njnt + j] + (type == 0 ? 3 : 0);
    double K[16] = {0};
    for (int i = 0; i < R; i++) {
      const double* q = rows + (size_t)i * nx + a;
      const double w = dmul(4.0, i == R - 1 ? A.weight_covariance0 : A.weight_sigma);
      for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) K[4 * r + c] = dadd(K[4 * r + c], dmul(dmul(w, q[r]), q[c]));
    }
    const double total = dadd(A.weight_covariance0, dmul((double)(R - 1), A.weight_sigma));
    for (int r = 0; r < 4; r++) K[5 * r] = dsub(K[5 * r], total);
    fb_principal_eigenvector4(mean + a, K, rows + (size_t)(R - 1) * nx + a);
  }
  __syncthreads();
  // differences
  for (int i = threadIdx.x; i < R; i += blockDim.x) fb_state_diff(A, ds + (size_t)i * ns, rows + (size_t)i * nx, mean);
  for (int i = threadIdx.x; i < R * ny; i += blockDim.x) dy[i] = dsub((double)ys[i], ymean[i % ny]);
  __syncthreads();
  // covariances: cov_yy = R + sum w dy dy', cov_sy = sum w ds dy', cov_ss = Q + sum w ds ds'
  const double* np = A.noise_process + (size_t)b * ns;
  const double* nsens = A.noise_sensor + (size_t)b * ny;
  for (int i = threadIdx.x; i < ny * ny + ns * ny + ns * ns; i += blockDim.x) {
    const double *u, *v;
    int r, c, su, sv;
    double a = 0.0, *out;
    if (i < ny * ny) {
      r = i / ny; c = i - r * ny; u = dy; v = dy; su = sv = ny; out = cyy + i; if (r == c) a = nsens[r];
    } else if (i < ny * ny + ns * ny) {
      const int k = i - ny * ny; r = k / ny; c = k - r * ny; u = ds; v = dy; su = ns; sv = ny; out = csy + k;
    } else {
      const int k = i - ny * ny - ns * ny; r = k / ns; c = k - r * ns; u = ds; v = ds; su = sv = ns; out = css + k;
      if (r == c) a = np[r];
    }
    for (int p = 0; p < R; p++) {
      const double w = p == R - 1 ? A.weight_covariance0 : A.weight_sigma;
      a = dadd(a, dmul(dmul(w, u[(size_t)p * su + r]), v[(size_t)p * sv + c]));
    }
    *out = a;
  }
  for (int k = threadIdx.x; k < ny; k += blockDim.x) e[k] = dsub(A.sensor[(size_t)b * ny + k], ymean[k]);
  __syncthreads();
  double* Pn = W + A.o_Pn;
  if (!fb_gain_update(csy, cyy, e, css, corr, Pn, W + A.o_T, ns, ny)) {
    if (threadIdx.x == 0) A.status[b] = mjpc_b200_bank::SENSOR_FACTOR_FAILED;
    return;
  }
  if (threadIdx.x == 0) fb_state_add(A, mean, [&](int j) { return corr[j]; }, 1.0);   // mean becomes the new state
  __syncthreads();
  fb_commit(A, b, mean, Pn, true, R - 1);
}

// Kalman.update_measurement (kalman.cc UpdateMeasurement) after the measurement launch
extern "C" __global__ void __launch_bounds__(kFilterThreads) kalman_measurement_kernel(const __grid_constant__ FilterBankArgs A) {
  const int b = blockIdx.x, nv = A.nv, nx = A.nq + nv, ns = 2 * nv, ny = A.ny;
  double* W = A.scratch + (size_t)b * A.scratch_words;
  double *Cm = W + A.o_C, *PCt = W + A.o_X, *S = W + A.o_S, *e = W + A.o_e, *corr = W + A.o_corr, *x = W + A.o_mean,
         *Pn = W + A.o_Pn;
  double* P = A.P + (size_t)b * ns * ns;
  const float* y = A.sensordata + (size_t)b * A.rows * ny;
  const double h = A.centered ? 2 * A.epsilon : A.epsilon;
  // C [ny][ns] from the sensor differences; y_hat = the centre's sensors
  for (int k = threadIdx.x; k < ny * ns; k += blockDim.x) {
    const int r = k / ns, i = k - r * ns;
    const float* yp = y + (size_t)(1 + i) * ny;
    const float* ym = A.centered ? y + (size_t)(1 + ns + i) * ny : y;
    Cm[k] = dsub((double)yp[r], (double)ym[r]) / h;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ns * ny; k += blockDim.x) {   // P C' [ns][ny]
    const int r = k / ny, c = k - r * ny;
    double a = 0;
    for (int j = 0; j < ns; j++) a = dadd(a, dmul(P[(size_t)r * ns + j], Cm[(size_t)c * ns + j]));
    PCt[k] = a;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ny * ny; k += blockDim.x) {   // S = C P C' + R
    const int r = k / ny, c = k - r * ny;
    double a = 0;
    for (int j = 0; j < ns; j++) a = dadd(a, dmul(Cm[(size_t)r * ns + j], PCt[(size_t)j * ny + c]));
    S[k] = dadd(a, r == c ? A.noise_sensor[(size_t)b * ny + r] : 0.0);
  }
  for (int k = threadIdx.x; k < ny; k += blockDim.x) e[k] = dsub(A.sensor[(size_t)b * ny + k], (double)y[k]);
  for (int k = threadIdx.x; k < nx; k += blockDim.x) x[k] = A.state[(size_t)b * nx + k];
  __syncthreads();
  if (!fb_gain_update(PCt, S, e, P, corr, Pn, W + A.o_T, ns, ny)) {
    if (threadIdx.x == 0) A.status[b] = mjpc_b200_bank::SENSOR_FACTOR_FAILED;
    return;
  }
  if (threadIdx.x == 0) fb_state_add(A, x, [&](int j) { return corr[j]; }, 1.0);
  __syncthreads();
  fb_commit(A, b, x, Pn, false, 0);
}

// Kalman.update_prediction (kalman.cc UpdatePrediction) after the prediction launch
extern "C" __global__ void __launch_bounds__(kFilterThreads) kalman_prediction_kernel(const __grid_constant__ FilterBankArgs A) {
  const int b = blockIdx.x, nv = A.nv, nx = A.nq + nv, ns = 2 * nv;
  if (A.status[b] != 0) return;
  double* W = A.scratch + (size_t)b * A.scratch_words;
  double *rows = W + A.o_rows, *Am = W + A.o_F, *cols = W + A.o_ds, *PAt = W + A.o_P0, *Pn = W + A.o_Pn;
  const double* P = A.P + (size_t)b * ns * ns;
  const double h = A.centered ? 2 * A.epsilon : A.epsilon;
  fb_load_next(A, b, rows);
  // column i of A: (next(x (+) eps e_i) (-) next(x [(+) -eps e_i])) / h
  for (int i = threadIdx.x; i < ns; i += blockDim.x)
    fb_state_diff(A, cols + (size_t)i * ns, rows + (size_t)(1 + i) * nx, A.centered ? rows + (size_t)(1 + ns + i) * nx : rows);
  __syncthreads();
  for (int k = threadIdx.x; k < ns * ns; k += blockDim.x) {
    const int r = k / ns, i = k - r * ns;
    Am[k] = cols[(size_t)i * ns + r] / h;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ns * ns; k += blockDim.x) {   // P A'
    const int r = k / ns, c = k - r * ns;
    double s = 0;
    for (int j = 0; j < ns; j++) s = dadd(s, dmul(P[(size_t)r * ns + j], Am[(size_t)c * ns + j]));
    PAt[k] = s;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ns * ns; k += blockDim.x) {   // A P A' + Q
    const int r = k / ns, c = k - r * ns;
    double s = 0;
    for (int j = 0; j < ns; j++) s = dadd(s, dmul(Am[(size_t)r * ns + j], PAt[(size_t)j * ns + c]));
    Pn[k] = dadd(s, r == c ? A.noise_process[(size_t)b * ns + r] : 0.0);
  }
  __syncthreads();
  fb_symmetrize(Pn, ns);
  fb_commit(A, b, rows, Pn, true, 0);   // the new state: the centre's next state, row 0
}

}  // namespace mjpc_dev
