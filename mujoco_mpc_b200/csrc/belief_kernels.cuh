// belief_kernels.cuh - initial-state ensembles (mjpc_b200_rollout_spline_belief_batched): the member states of every
// problem of a launch, drawn on the device from the problem's state covariance, and the same arithmetic on the host
// (mjpc_b200_host_state_member).
//
//   state_sample_kernel   one CTA per problem: the Cholesky factor L of (P + P')/2 in fp64 (shared memory; pivots
//                         within belief_tolerance of zero give zero columns), then for
//                         each member k >= 1 the tangent vector dx = L z and the state mean (+) dx written as float
//                         into launch row b K + k.  Row b K (member 0) keeps the mean as staged.
//
// The functions marked __host__ __device__ are the one definition of the draw, the factor and the state update; the
// host twin runs them serially, the kernel splits their loops over threads without changing any sum's order, so device
// and host differ only by the device's fused multiply-adds in fp64, far below the float rounding of the member states.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace mjpc_dev {

constexpr int kBeliefThreads = 128;
constexpr unsigned kBeliefKey = 3u;               // Philox key word 1 of the state-ensemble draws (rollout_kernels.cuh)
constexpr unsigned kBeliefTag = 0x42454C46u;      // 'BELF'

// Philox4x32-10 (Salmon et al. 2011) on counter c with key (k0, k1): the integer words, identical on host and device
__host__ __device__ inline void belief_philox(unsigned c[4], unsigned k0, unsigned k1) {
  for (int r = 0; r < 10; r++) {
    const unsigned long long p0 = 0xD2511F53ull * c[0], p1 = 0xCD9E8D57ull * c[2];
    const unsigned hi0 = (unsigned)(p0 >> 32), lo0 = (unsigned)p0, hi1 = (unsigned)(p1 >> 32), lo1 = (unsigned)p1;
    const unsigned n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

// z of element e of member k of problem b: Philox key (seed + b, 3), counter (iteration, k, e, 'BELF'), Box-Muller in
// fp64 on the first two words.  Key word 1 = 3 is used by no other stream (knots 0, rollout force noise 1, plants 2).
__host__ __device__ inline double belief_normal(unsigned seed, unsigned iteration, int b, int k, int e) {
  unsigned c[4] = {iteration, (unsigned)k, (unsigned)e, kBeliefTag};
  belief_philox(c, seed + (unsigned)b, kBeliefKey);
  const double u1 = ((double)c[0] + 0.5) * 2.3283064365386963e-10, u2 = ((double)c[1] + 0.5) * 2.3283064365386963e-10;
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}

// The pivot tolerances of the factorisation of the symmetric n x n matrix A (row-major, lower triangle read), one per
// row: tau[i] = n 2^-40 max(A_ii, 0).  The pivot of row j is A_jj minus the squares of row j of L, which sum to A_jj
// in exact arithmetic, so without pivoting its rounding is about n eps A_jj times the growth that the leading block's
// conditioning adds; tau allows a growth of 2^12.  A positive definite A has every pivot at or above its smallest
// eigenvalue and tau[j] <= n 2^-40 times its largest, so with cond(A) below 2^40 / n it is factored exactly as
// without the tolerance; so is any diagonal A.
__host__ __device__ inline void belief_tolerance(const double* A, int n, int i, double* tau) {
  tau[i] = A[i * n + i] > 0.0 ? n * 0x1p-40 * A[i * n + i] : 0.0;
}
// Step j of the right-looking factorisation of the symmetric lower triangle A (row-major n x n): the pivot d.
// d > tau[j] gives L[j][j] = sqrt(d).  |d| <= tau[j] is a rounded zero: the column becomes zero (a state direction
// with no uncertainty) when every entry below it is a rounded coupling of a positive semi-definite trailing block too,
// A_ij^2 <= 4 tau[j] (max(A_ii, 0) + tau[i]) (exactly, A_ij^2 <= d A_ii, with d and A_ii each off by up to their
// tolerance).  Anything else (d < -tau[j], a real coupling below a zero pivot, a non-finite pivot) fails: false.
__host__ __device__ inline bool belief_pivot(double* A, int n, int j, const double* tau) {
  const double d = A[j * n + j];
  if (d > tau[j] && d <= 1.7976931348623157e308) { A[j * n + j] = sqrt(d); return true; }
  if (!(fabs(d) <= tau[j])) return false;
  for (int i = j + 1; i < n; i++) {
    const double a = A[i * n + j], aii = A[i * n + i] > 0.0 ? A[i * n + i] : 0.0;
    if (!(a * a <= 4.0 * tau[j] * (aii + tau[i]))) return false;
  }
  A[j * n + j] = 0.0;
  return true;
}
// below the pivot of column j: L[i][j] = A[i][j] / L[j][j] (0 for a zero column)
__host__ __device__ inline void belief_column(double* A, int n, int j, int i) {
  const double p = A[j * n + j];
  A[i * n + j] = p > 0.0 ? A[i * n + j] / p : 0.0;
}
// the trailing update of entry (i, c), j < c <= i
__host__ __device__ inline void belief_update(double* A, int n, int j, int i, int c) {
  A[i * n + c] -= A[i * n + j] * A[c * n + j];
}
// dx[i] = sum_{j <= i} L[i][j] z[j], summed from j = 0
__host__ __device__ inline double belief_row(const double* L, const double* z, int n, int i) {
  double s = 0.0;
  for (int j = 0; j <= i; j++) s += L[i * n + j] * z[j];
  return s;
}

// q (+) w for a unit quaternion q: q * exp(w / 2), normalised (mju_quatIntegrate with scale 1, as mj_integratePos
// applies it).  A rotation of exactly zero leaves q as it is, bit for bit (not renormalised).
__host__ __device__ inline void belief_quat(double* q, const double* w) {
  if (w[0] == 0.0 && w[1] == 0.0 && w[2] == 0.0) return;
  const double a = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double r[4] = {1, 0, 0, 0};
  if (a >= 1e-15) {
    const double s = sin(a / 2) / a;
    r[0] = cos(a / 2); r[1] = s * w[0]; r[2] = s * w[1]; r[3] = s * w[2];
  }
  const double o[4] = {q[0] * r[0] - q[1] * r[1] - q[2] * r[2] - q[3] * r[3],
                       q[0] * r[1] + q[1] * r[0] + q[2] * r[3] - q[3] * r[2],
                       q[0] * r[2] - q[1] * r[3] + q[2] * r[0] + q[3] * r[1],
                       q[0] * r[3] + q[1] * r[2] - q[2] * r[1] + q[3] * r[0]};
  const double nrm = sqrt(o[0] * o[0] + o[1] * o[1] + o[2] * o[2] + o[3] * o[3]);
  for (int c = 0; c < 4; c++) q[c] = o[c] / nrm;
}
// a scalar coordinate x (+) d: x itself when d is 0 (so a zero perturbation keeps every bit, the sign of zero too)
__host__ __device__ inline double belief_add(double x, double d) { return d != 0.0 ? x + d : x; }

// One joint's part of the position half of mean (+) dx (mj_integratePos): q its qpos entries in double, updated in
// place; d its entries of dx
__host__ __device__ inline void belief_joint(double* q, const double* d, int type) {
  if (type == 0) {          // free: position added, orientation through the quaternion
    for (int c = 0; c < 3; c++) q[c] = belief_add(q[c], d[c]);
    belief_quat(q + 3, d + 3);
  } else if (type == 1) {   // ball
    belief_quat(q, d);
  } else {                  // slide, hinge
    q[0] = belief_add(q[0], d[0]);
  }
}
// the number of qpos entries of a joint of this type
__host__ __device__ inline int belief_width(int type) { return type == 0 ? 7 : type == 1 ? 4 : 1; }

struct BeliefArgs {
  int B, K, n;                 // problems, members per problem, tangent dimension n = 2 nv
  int nq, nv, njnt;
  const int* jnt;              // [3][njnt]: type, qposadr, dofadr
  const double* cov;           // [B][n][n]
  unsigned seed, iteration;
  float* rows;                 // the launch's state rows [B K][nq + nv]; row b K holds problem b's mean
  const int* variant_index;    // the selected variant of each problem (nullptr: no variants)
  int* row_index;              // out: the variant of each launch row [B K] (when variant_index is set)
  int* status;                 // out [B]: 0, or 1 when the factorisation failed (no row of the problem is written)
};

// dynamic shared memory of state_sample_kernel for tangent dimension n: L [n][n], z [n], dx [n], the pivot tolerances
// [n], the mean [nq + nv]
inline size_t belief_smem(int n, int nq, int nv) { return ((size_t)n * n + 3 * (size_t)n + nq + nv) * sizeof(double); }

extern "C" __global__ void __launch_bounds__(kBeliefThreads) state_sample_kernel(const BeliefArgs A) {
  extern __shared__ double s_belief[];
  const int b = blockIdx.x, tid = threadIdx.x, n = A.n, nx = A.nq + A.nv;
  double* L = s_belief;
  double* z = L + (size_t)n * n;
  double* dx = z + n;
  double* tau = dx + n;
  double* mean = tau + n;
  const int R = b * A.K;
  if (A.variant_index && tid < A.K) A.row_index[R + tid] = A.variant_index[b];
  // (P + P') / 2, lower triangle
  const double* P = A.cov + (size_t)b * n * n;
  for (int w = tid; w < n * n; w += blockDim.x) {
    const int i = w / n, c = w - i * n;
    if (c <= i) L[w] = 0.5 * (P[i * n + c] + P[c * n + i]);
  }
  for (int i = tid; i < nx; i += blockDim.x) mean[i] = (double)A.rows[(size_t)R * nx + i];
  __shared__ int ok;
  if (tid == 0) ok = 1;
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) belief_tolerance(L, n, i, tau);
  __syncthreads();
  for (int j = 0; j < n; j++) {
    if (tid == 0 && !belief_pivot(L, n, j, tau)) ok = 0;
    __syncthreads();
    if (!ok) break;
    for (int i = j + 1 + tid; i < n; i += blockDim.x) belief_column(L, n, j, i);
    __syncthreads();
    // the trailing lower triangle j < c <= i < n, one entry per thread
    const int m = n - j - 1;
    for (int w = tid; w < m * m; w += blockDim.x) {
      const int i = j + 1 + w / m, c = j + 1 + w % m;
      if (c <= i) belief_update(L, n, j, i, c);
    }
    __syncthreads();
  }
  if (tid == 0) A.status[b] = ok ? 0 : 1;
  if (!ok) return;
  for (int k = 1; k < A.K; k++) {
    for (int e = tid; e < n; e += blockDim.x) z[e] = belief_normal(A.seed, A.iteration, b, k, e);
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) dx[i] = belief_row(L, z, n, i);
    __syncthreads();
    float* row = A.rows + (size_t)(R + k) * nx;
    for (int j = tid; j < A.njnt; j += blockDim.x) {
      const int type = A.jnt[j], qa = A.jnt[A.njnt + j], da = A.jnt[2 * A.njnt + j];
      double q[7];
      const int w = belief_width(type);
      for (int c = 0; c < w; c++) q[c] = mean[qa + c];
      belief_joint(q, dx + da, type);
      for (int c = 0; c < w; c++) row[qa + c] = (float)q[c];
    }
    for (int i = tid; i < A.nv; i += blockDim.x) row[A.nq + i] = (float)belief_add(mean[A.nq + i], dx[A.nv + i]);
    __syncthreads();
  }
}

}  // namespace mjpc_dev
