// dev_data.cuh - per-trajectory simulation state ("mjData") as it lives in shared memory, one block of
// floats per trajectory, plus the small device math kit.  One (main) warp owns one trajectory - the static rollout
// instances add helper warps that work on the same block between barriers ("helper warps" below): every array below is
// private to that warp, phases are separated by __syncwarp(), and lanes split work by body / dof /
// constraint row / matrix entry.
#pragma once
#include <cuda_runtime.h>

#include <utility>

#include "dev_model.h"

// Code-footprint control: with one warp per scheduler every instruction-cache
// miss is exposed, and fully unrolled straight-line code in the Newton loop would stream from L2 on every
// iteration.  MJPC_ROLL marks loops whose unrolling buys no ILP worth its code size.
#define MJPC_ROLL _Pragma("unroll 1")

namespace mjpc_dev {

constexpr int kMaxSplinePoints = 64;  // knot_times has a fixed capacity so that only the LAST array depends on P
// name, element count (expression over M = DevModel, P = spline points)
#define MJPC_D_ARRAYS(X)                                                                                          \
  X(qpos, M.nq) X(qvel, M.nv) X(ctrl, M.nu) X(qacc, M.nv) X(qacc_warmstart, M.nv) X(mocap_pos, 3 * M.nmocap)      \
  X(mocap_quat, 4 * M.nmocap) X(xpos, 3 * M.nbody) X(xquat, 4 * M.nbody) X(xmat, 9 * M.nbody)                     \
  X(xipos, 3 * M.nbody) X(ximat, 9 * M.nbody) X(xanchor, 3 * M.njnt) X(xaxis, 3 * M.njnt)                         \
  X(geom_xpos, 3 * M.ngeom) X(geom_xmat, 9 * M.ngeom) X(site_xpos, 3 * M.nsite) X(subtree_com, 3 * M.nbody)       \
  X(cinert, 10 * M.nbody) X(crb, 10 * M.nbody) X(cdof, 6 * M.nv) X(cdof_dot, 6 * M.nv) X(cvel, 6 * M.nbody)       \
  X(cacc, 6 * M.nbody) X(cfrc, 6 * M.nbody) X(cfrc_sub, 6 * M.nbody) X(subtree_linvel, 3 * M.nbody)               \
  X(body_linvel, 3 * M.nbody) X(qM, M.nv * M.nv) X(qLD, M.nv * M.nv) X(qH, M.nv * M.nv) X(dofbuf, 6 * M.nv)       \
  X(ldinv, M.nv) X(hinv, M.nv) X(qfrc_bias, M.nv) X(qfrc_passive, M.nv) X(qfrc_actuator, M.nv)                    \
  X(qfrc_smooth, M.nv) X(qacc_smooth, M.nv) X(qfrc_constraint, M.nv) X(actuator_force, M.nu) X(Ma, M.nv)          \
  X(grad, M.nv) X(search, M.nv) X(Mv, M.nv) X(vtmp, M.nv) X(con_dist, M.maxcon) X(con_pos, 3 * M.maxcon)          \
  X(con_frame, 9 * M.maxcon) X(con_friction, 5 * M.maxcon) X(con_solref, 2 * M.maxcon)                            \
  X(con_solimp, 5 * M.maxcon) X(con_mu, M.maxcon) X(con_margin, M.maxcon) X(con_dim, M.maxcon)                    \
  X(con_g1, M.maxcon) X(con_g2, M.maxcon) X(con_adr, M.maxcon) X(efc_J, M.maxefc * 16)                            \
  X(efc_W, 2 * M.maxcon * 16) X(con_nd, M.maxcon) X(con_dof, M.maxcon * 16) X(con_loc, M.maxcon * M.nv)           \
  X(con_boff, M.maxcon + 1) X(con_xf, M.maxcon * 16) X(efc_blk, 1024) X(efc_dof, M.maxefc) X(efc_sgn, M.maxefc)     \
  X(efc_Jd, (M.maxefc + 8) * ((M.nv + 3) / 4 * 4)) X(efc_Xd, 2 * M.maxcon * ((M.nv + 3) / 4 * 4)) X(efc_pos, M.maxefc) X(efc_margin, M.maxefc) X(efc_diag, M.maxefc)                    \
  X(efc_R, M.maxefc) X(efc_D, M.maxefc) X(efc_K, M.maxefc) X(efc_B, M.maxefc) X(efc_imp, M.maxefc)                \
  X(efc_aref, M.maxefc) X(efc_hw, M.maxefc) X(efc_force, M.maxefc) X(efc_jar, M.maxefc) X(efc_Jv, M.maxefc) X(efc_floss, M.maxefc)    \
  X(efc_type, M.maxefc) X(efc_id, M.maxefc) X(efc_state, M.maxefc) X(efc_item, M.maxefc) X(efc_hc, 36 * M.maxcon) X(con_mlo, M.maxcon) X(con_mhi, M.maxcon) \
  X(efc_w, 6 * M.maxefc) X(con_side, M.maxcon) X(con_mbody, M.maxcon) X(efc_drow, M.maxefc) \
  X(residual, M.num_residual) X(xnom, M.nq + M.nv) X(dx, 2 * M.nv) X(xfrc, 6 * M.nbody) X(knot_times, kMaxSplinePoints) X(knots, P * M.nu)

enum DataArrayId {
#define X(n, sz) D_##n,
  MJPC_D_ARRAYS(X)
#undef X
      D_COUNT
};

struct DevLayout {
  int off[D_COUNT];
  int total;  // floats per warp (multiple of 4)
};

inline DevLayout make_layout(const DevModel& M, int P) {
  DevLayout L;
  int o = 0;
#define X(n, sz) L.off[D_##n] = o; o += (((sz) + 3) / 4) * 4;
  MJPC_D_ARRAYS(X)
#undef X
  L.total = o;
  return L;
}

#ifdef __CUDACC__
constexpr unsigned kFull = 0xffffffffu;
constexpr float kMinVal = 1e-15f;
constexpr float kCapsuleParallel = 16 * 1.1920929e-7f;   // 16 fp32 eps: collide_capsule_capsule's parallel test
constexpr float kMaxVal = 1e10f;
constexpr float kTolFloor = 1e-6f;
constexpr float kGradFloor = 16.f;   // the fp32 gradient cannot be driven below kGradFloor * eps * |its terms| (k_solve)  // fp32 floor on opt.tolerance (same rule as the oracle's fp32 instantiation)
constexpr float kMinImp = 0.0001f, kMaxImp = 0.9999f, kMinMu = 1e-5f;
enum { CNSTR_FRICTION_DOF = 0, CNSTR_LIMIT_JOINT, CNSTR_CONTACT_FRICTIONLESS, CNSTR_CONTACT_ELLIPTIC };
enum { STATE_SATISFIED = 0, STATE_QUADRATIC, STATE_LINEARNEG, STATE_LINEARPOS, STATE_CONE };

// Everything a trajectory touches lives in the CTA's dynamic shared memory:
//   [model floats nf][model ints ni][DevModel header][DevLayout][the trajectory's state]
// All accessors derive their pointers from the g_smem symbol with 32-bit float indices, so the compiler emits
// LDS/STS with shared-window addressing (pointers kept in a struct degrade to generic LD + 64-bit address
// arithmetic: that was ~45 % of the executed instructions in the first profile).
extern __shared__ __align__(16) float g_smem[];

struct Ctx {
  int hdr;    // float index of the DevModel header copy
  int lay;    // float index of the DevLayout copy
  int ibase;  // float index where the model's int arrays start
  int dbase;  // float index of this warp's state block
  int lane;
  int ncon, nefc, nitem, niter, nlim;
  int ndrow;   // constraint rows whose Hessian contribution is assembled row by row (efc_drow): contacts between two moving bodies, tendon limits
  const float* gkey;  // HBM: keyframe mocap positions [nkey][3*nmocap] (too large for the shared-memory pack)
  int xfrc_on;  // NoisyRollout: DF(xfrc) holds Cartesian force/torque per body, added to the smooth forces
  int npseudo;  // tendon-limit pseudo-contacts at the tail of the contact list (included in ncon)
  int warn;
  float time;
  // co-resident pair synchronisation (pair_sync_* below); sync == nullptr: off.  Only lane 0 of the main warp uses these.
  unsigned* sync;        // HBM: this SM's record (32 words)
  int sync_slot;         // 0 / 1: which of the SM's two candidates this one is; -1: not paired
  int wide_pending;      // helper-warp kernels: a posted phase has not been met yet (wide_settle)
#ifdef MJPC_PHASE_TIMING
  long long tph[9], tlast;   // profiling build only: SM cycles per pipeline phase (slots 0-7 are reported, 8 is "elsewhere")
#endif
};
// Profiling build (-DMJPC_PHASE_TIMING): PHASE_AT(c, map, i) adds the SM cycles since the previous timer call to slot i
// when the build records timer mapping `map` (-DMJPC_PHASE_MAP=<map>, profiles/phase_times.py --map):
//   0  pipeline phases: kinematics + com (+ CRB), collision, constraint rows, velocities + smooth forces + reference,
//      solve (rest), Hessian assembly, Cholesky factor + solve, policy + residual + cost + Euler + output
//   1  the Newton solve: J^T f + gradient + termination, M/J products, line search, step + constraint update, warm-start
//      evaluations, Hessian (one warp: the assembly; helper warps: the post and the wait at the join), Cholesky factor +
//      solve; slot 7 counts line-search evaluations (everything outside the solve is total - slots 0..6)
//   2  the first fork of a task-warp CTA: kinematics + com, collision, constraint rows, the main warp's wait at join 1,
//      reference + solve, the task warp's fork interval (CRB, velocities, smooth forces), -, the rest of the step
#ifndef MJPC_PHASE_MAP
#define MJPC_PHASE_MAP 0
#endif
#ifdef MJPC_PHASE_TIMING
#define PHASE_AT(c, m, i) do { if (MJPC_PHASE_MAP == (m)) { const long long t_ = clock64(); (c).tph[i] += t_ - (c).tlast; (c).tlast = t_; } } while (0)
#else
#define PHASE_AT(c, m, i) do { } while (0)
#endif
#define PHASE(c, i) PHASE_AT(c, 0, i)
// ---- model / state accessors.  Every device function is a template over a "spec" SP:
//   DynSpec          sizes and offsets are read from the header copy in shared memory (any model)
//   StaticSpec<K>    sizes and offsets are compile-time constants taken from a generated table K (spec_*.h):
//                    every shared-memory address becomes an immediate, size-dependent loops unroll, option
//                    branches fold.  The state block sits at a fixed address: a CTA holds one trajectory.
// Float options (timestep, tolerance, risk ...) always come from the live header: CM(c).timestep.
template <int V> struct IntC { static constexpr int v = V; };
constexpr int kHdrWords = (int)((sizeof(DevModel) + 15) / 16) * 4;
constexpr int kLayWords = (int)((sizeof(DevLayout) + 15) / 16) * 4;

struct DynSpec {
  static constexpr bool kStatic = false, kTreeFactor = false;
  static constexpr int kNV = 0, kNHPair = 0;
  static constexpr int kWide = 1, kTask = 0;
  static __device__ __forceinline__ const DevModel& hdr(const Ctx& c) { return *reinterpret_cast<const DevModel*>(g_smem + c.hdr); }
  static __device__ __forceinline__ const DevModel& model(const Ctx& c) { return hdr(c); }
  template <int ID> static __device__ __forceinline__ float* mf(const Ctx& c) { return g_smem + hdr(c).fo[ID]; }
  template <int ID> static __device__ __forceinline__ int* mi(const Ctx& c) {
    return reinterpret_cast<int*>(g_smem + c.ibase) + hdr(c).io[ID];
  }
  template <int ID> static __device__ __forceinline__ float* df(const Ctx& c) {
    return g_smem + c.dbase + reinterpret_cast<const DevLayout*>(g_smem + c.lay)->off[ID];
  }
};

// The dof tree of a static spec (K::kDofParent, parent before child) as warp_tree_factor_solve reads it: the ancestors
// of each dof, and the elimination order - by height above the leaves (a dof after all its descendants), within one
// height by descending index.
template <class K, int N>
struct DofTree {
  static constexpr int kN = N;
  static __host__ __device__ constexpr unsigned anc(int j) {
    unsigned m = 0;
    for (int a = K::kDofParent[j]; a >= 0; a = K::kDofParent[a]) m |= 1u << a;
    return m;
  }
  static __host__ __device__ constexpr int col(int t) {
    int h[64] = {}, hmax = 0;
    for (int k = N - 1; k >= 0; k--) {
      const int p = K::kDofParent[k];
      if (p >= 0 && h[k] + 1 > h[p]) h[p] = h[k] + 1;
      if (h[k] > hmax) hmax = h[k];
    }
    for (int l = 0; l <= hmax; l++)
      for (int j = N - 1; j >= 0; j--)
        if (h[j] == l && t-- == 0) return j;
    return -1;
  }
};

// W > 1: the CTA holds W warps for ONE trajectory - warp 0 runs the pipeline, warps 1..W-1 are helpers that join it for
// the phases with more independent work items than one warp has lanes (wide_* below)
// T = 1: one more warp (index W) runs the phases that do not depend on the constraint pipeline concurrently with it
// D = true: the SPD solves keep the dense factor (warp_chol_factor_solve) instead of the dof tree's (step_batch_body)
template <class K, int W = 1, int T = 0, bool D = false>
struct StaticSpec {
  static constexpr bool kStatic = true, kTreeFactor = !D;
  static constexpr int kWide = W, kTask = T;
  static __host__ __device__ constexpr int w(size_t byte_off, int i = 0) { return K::kModelWords[byte_off / 4 + i]; }
  struct View {
#define X(n) static constexpr int n = w(offsetof(DevModel, n));
    MJPC_M_INTS(X)
#undef X
  };
  static constexpr int kNV = View::nv, kNHPair = View::nhpair;
  using Tree = DofTree<K, kNV>;
  static constexpr int kHdr = View::nf + View::ni;
  static constexpr int kData0 = kHdr + kHdrWords + kLayWords;
  static __device__ __forceinline__ const DevModel& hdr(const Ctx&) { return *reinterpret_cast<const DevModel*>(g_smem + kHdr); }
  static __device__ __forceinline__ View model(const Ctx&) { return View{}; }
  template <int ID> static __device__ __forceinline__ float* mf(const Ctx&) {
    return g_smem + IntC<w(offsetof(DevModel, fo), ID)>::v;
  }
  template <int ID> static __device__ __forceinline__ int* mi(const Ctx&) {
    return reinterpret_cast<int*>(g_smem) + IntC<View::nf + w(offsetof(DevModel, io), ID)>::v;
  }
  template <int ID> static __device__ __forceinline__ float* df(const Ctx&) {
    return g_smem + IntC<kData0 + K::kLayoutOff[ID]>::v;
  }
};

#define CM(c) (SP::hdr(c))
#define MF(n) (SP::template mf<F_##n>(c))
#define MI(n) (SP::template mi<I_##n>(c))
#define DF(n) (SP::template df<D_##n>(c))
#define DI(n) (reinterpret_cast<int*>(SP::template df<D_##n>(c)))

// ---------------------------------------------------------------------------------------- helper warps
// One trajectory is a chain of dependent phases; at 256 candidates every warp has an issue port to itself and the
// kernel's duration is that chain's latency.  Phases whose work items outnumber the 32 lanes (Hessian entries, ...)
// are therefore spread over W warps of the same CTA: the main warp posts a command and its scalar context to a
// mailbox, all W warps meet on a named barrier, run the phase with a stride of 32*W items, and meet again.  The
// per-item arithmetic is unchanged, so results are bitwise those of the one-warp kernel.
// The Newton Hessian assembly (WIDE_HESSIAN) runs on the helper warps alone while the main warp forms J^T f, the
// gradient and the termination test (k_solve): the main warp posts without waiting (wide_post_async) and meets the
// helpers again before the Cholesky factor (wide_join).
//   named barriers: 1 = post (main arrives / helpers wait, 32*W), 3 = join (helpers arrive / main waits, 32*W),
//   4 = between the helpers' own passes (32*(W-1)).  Post and join are separate barriers: a helper that has arrived at
//   the join and goes on to wait for the next post must not be counted twice in one barrier generation.
enum { WIDE_EXIT = 0, WIDE_HESSIAN = 1 };
struct WideBox {
  int cmd, ncon, nlim, ndrow, nefc; int task_exit, task_warn; float task_cost;
#ifdef MJPC_PHASE_TIMING
  long long task_fork_cycles;   // timer mapping 2: the task warp's fork intervals, summed over the steps
#endif
};
__device__ __forceinline__ WideBox& wide_box() { __shared__ WideBox box; return box; }
template <class SP>
__device__ __forceinline__ void wide_bar() {
  if constexpr (SP::kWide > 1) asm volatile("bar.sync 1, %0;" ::"n"(32 * SP::kWide) : "memory");
  else __syncwarp();
}
// main warp <-> task warp (fork / join points of the step, rollout_kernels.cuh)
__device__ __forceinline__ void task_bar() { asm volatile("bar.sync 2, 64;" ::: "memory"); }
// lane index / lane count of the trajectory's thread group
template <class SP> __device__ __forceinline__ int wide_lane(const Ctx& c) { return SP::kWide > 1 ? (int)threadIdx.x : c.lane; }
// The thread group a wide phase runs on: all W warps of the trajectory (kHelpers = false; W = 1: the warp itself), or
// the W-1 helper warps alone (warps 1..W-1 of the CTA)
template <class SP, bool kHelpers>
struct WideGroup {
  static constexpr int kWarps = kHelpers ? SP::kWide - 1 : SP::kWide;
  static __device__ __forceinline__ int lane(const Ctx& c) { return kHelpers ? (int)threadIdx.x - 32 : wide_lane<SP>(c); }
  static __device__ __forceinline__ void bar() {
    if constexpr (!kHelpers) wide_bar<SP>();
    else if constexpr (kWarps > 1) asm volatile("bar.sync 4, %0;" ::"n"(32 * kWarps) : "memory");
    else __syncwarp();
  }
};
// main warp: publish the command and the scalar context the phase reads, then release the helpers
template <class SP>
__device__ __forceinline__ void wide_post(const Ctx& c, int cmd) {
  if constexpr (SP::kWide > 1) {
    WideBox& b = wide_box();
    if (c.lane == 0) { b.cmd = cmd; b.ncon = c.ncon; b.nlim = c.nlim; b.ndrow = c.ndrow; b.nefc = c.nefc; }
    wide_bar<SP>();
  }
}
// ... the same without waiting for the helpers (bar.arrive: the mailbox writes are visible to them once they pass)
template <class SP>
__device__ __forceinline__ void wide_post_async(const Ctx& c, int cmd) {
  static_assert(SP::kWide > 1, "a one-warp trajectory has no helpers to post to");
  WideBox& b = wide_box();
  if (c.lane == 0) { b.cmd = cmd; b.ncon = c.ncon; b.nlim = c.nlim; b.ndrow = c.ndrow; b.nefc = c.nefc; }
  asm volatile("bar.arrive 1, %0;" ::"n"(32 * SP::kWide) : "memory");
}
// main warp: wait until the helpers have finished the posted phase; helpers: report it finished
template <class SP>
__device__ __forceinline__ void wide_join() { asm volatile("bar.sync 3, %0;" ::"n"(32 * SP::kWide) : "memory"); }
template <class SP>
__device__ __forceinline__ void wide_done() { asm volatile("bar.arrive 3, %0;" ::"n"(32 * SP::kWide) : "memory"); }
// main warp: meet a phase that is still in flight (an assembly the solve no longer needs is left running while the step
// ends; this is called before the next step touches what it reads or writes, and before the helpers are released)
template <class SP>
__device__ __forceinline__ void wide_settle(Ctx& c) {
  if constexpr (SP::kWide > 1) {
    if (c.wide_pending) { wide_join<SP>(); c.wide_pending = 0; }
  }
}

// ---------------------------------------------------------------------------------------- co-resident pairs
// At 256 candidates 124 of the H100's 132 SMs run two candidates, and the measured cost of sharing an SM is instruction
// fetch: two candidates at different places of the 124 KB-per-step code evict each other's lines, while two that
// run the SAME code at the same time cost each other almost nothing (profiles/icache_probe.py).  The main warps of
// the two candidates of an SM therefore keep in step through a 128-byte record in HBM (they are different CTAs):
// they start every time step together; the one that needs more Newton iterations finishes its solve while the other
// waits at the next meeting point - and a waiting warp fetches nothing.
// Timing only: no data crosses, results are bitwise those of unsynchronised runs; every wait is bounded (partner
// finished / time-out), so nothing can deadlock.  Meeting at every Newton iteration as well was measured and is slower
// (an HBM flag round trip per iteration plus the waits), profiles/ab_pairsync.py.
//   record words: [0] registration count | [8 + 8 s + {0, 1}] alive flag, meeting-point sequence number of slot s
constexpr long long kPairTimeout = 400000;   // SM cycles (shorter time-outs were measured: strict waiting is best)
__device__ __forceinline__ unsigned ld_vol(const unsigned* p) {
  unsigned v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_vol(unsigned* p, unsigned v) { asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void pair_sync_init(Ctx& c, unsigned* table) {
  c.sync = nullptr; c.sync_slot = -1;
  if (!table) return;
  unsigned smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  c.sync = table + 32 * (smid & 255u);
  if (c.lane == 0) {
    const unsigned slot = atomicAdd(c.sync, 1u);
    c.sync_slot = slot < 2u ? (int)slot : -1;
    if (c.sync_slot >= 0) st_vol(c.sync + 8 + 8 * c.sync_slot, 1u);   // alive
  }
}
__device__ __forceinline__ void pair_sync_done(Ctx& c) {   // the SM's other candidate stops waiting for this one
  if (c.sync && c.lane == 0 && c.sync_slot >= 0) st_vol(c.sync + 8 + 8 * c.sync_slot, 0u);
}
// meeting point number seq (increasing along the trajectory): wait until the partner has reached it too (or is gone)
__device__ __noinline__ void pair_sync_meet(Ctx& c, int seq) {
  if (!c.sync) return;
  if (c.lane == 0 && c.sync_slot >= 0) {
    unsigned* me = c.sync + 8 + 8 * c.sync_slot;
    const unsigned* ot = c.sync + 8 + 8 * (1 - c.sync_slot);
    st_vol(me + 1, (unsigned)seq);
    if (seq > 0 && ld_vol(c.sync) >= 2u) {
      const long long t0 = clock64();
      while (ld_vol(ot + 1) < (unsigned)seq && ld_vol(ot) != 0u && clock64() - t0 < kPairTimeout) __nanosleep(200);
    }
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------------------- small math
__device__ __forceinline__ float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ void cross3(float* r, const float* a, const float* b) {
  float x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ float norm3(const float* a) { return sqrtf(dot3(a, a)); }
__device__ __forceinline__ float normalize3(float* a) {
  float n = norm3(a);
  if (n < kMinVal) { a[0] = 1; a[1] = 0; a[2] = 0; return n; }
  a[0] /= n; a[1] /= n; a[2] /= n;
  return n;
}
__device__ __forceinline__ void quat_mul(float* r, const float* a, const float* b) {
  float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  float x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  float z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
__device__ __forceinline__ void quat_normalize(float* q) {
  float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < kMinVal) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
__device__ __forceinline__ void quat2mat(float* m, const float* q) {
  float w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
__device__ __forceinline__ void rot_vec(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2],
        z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ void rot_vec_T(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2],
        z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
__device__ __forceinline__ void axis_angle_quat(float* q, const float* axis, float angle) {
  float s, co;
  sincosf(angle * 0.5f, &s, &co);
  q[0] = co; q[1] = axis[0] * s; q[2] = axis[1] * s; q[3] = axis[2] * s;
}
__device__ __forceinline__ void quat_integrate(float* q, const float* w, float h) {
  float ax[3] = {w[0], w[1], w[2]};
  float n = norm3(ax);
  if (n < kMinVal) return;
  ax[0] /= n; ax[1] /= n; ax[2] /= n;
  float dq[4], r[4];
  axis_angle_quat(dq, ax, n * h);
  quat_mul(r, q, dq);
  quat_normalize(r);
  q[0] = r[0]; q[1] = r[1]; q[2] = r[2]; q[3] = r[3];
}
__device__ __forceinline__ void cross_motion(float* r, const float* v, const float* m) {
  float a[3], b[3], cc[3];
  cross3(a, v, m); cross3(b, v, m + 3); cross3(cc, v + 3, m);
  for (int k = 0; k < 3; k++) { r[k] = a[k]; r[3 + k] = b[k] + cc[k]; }
}
__device__ __forceinline__ void cross_force(float* r, const float* v, const float* f) {
  float a[3], b[3], cc[3];
  cross3(a, v, f); cross3(b, v + 3, f + 3); cross3(cc, v, f + 3);
  for (int k = 0; k < 3; k++) { r[k] = a[k] + b[k]; r[3 + k] = cc[k]; }
}
__device__ __forceinline__ void mul_inert_vec(float* r, const float* I, const float* v) {
  const float* w = v; const float* l = v + 3; const float* mo = I + 6;
  float a[3], b[3];
  cross3(a, mo, l); cross3(b, mo, w);
  r[0] = I[0] * w[0] + I[3] * w[1] + I[4] * w[2] + a[0];
  r[1] = I[3] * w[0] + I[1] * w[1] + I[5] * w[2] + a[1];
  r[2] = I[4] * w[0] + I[5] * w[1] + I[2] * w[2] + a[2];
  r[3] = I[9] * l[0] - b[0]; r[4] = I[9] * l[1] - b[1]; r[5] = I[9] * l[2] - b[2];
}
__device__ __forceinline__ void make_frame(float* f) {
  float* x = f; float* y = f + 3; float* z = f + 6;
  if (x[1] > -0.5f && x[1] < 0.5f) { y[0] = 0; y[1] = 1; y[2] = 0; } else { y[0] = 0; y[1] = 0; y[2] = 1; }
  float dd = dot3(x, y);
  for (int k = 0; k < 3; k++) y[k] -= dd * x[k];
  normalize3(y);
  cross3(z, x, y);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int n = __shfl_up_sync(kFull, v, o);
    if (lane >= o) v += n;
  }
  return v;
}

// ---- warp-cooperative dense Cholesky (left-looking), A = L L^T in place (lower), n x n row-major in
// shared memory; inv[n] receives 1/L[i][i].  All 32 lanes must call.
__device__ __noinline__ void warp_chol(float* A, float* inv, int n, int lane) {
  for (int j = 0; j < n; j++) {
    float piv = 0.f;
    for (int base = j; base < n; base += 32) {
      int i = base + lane;
      float s = 0.f;
      if (i < n) {
        s = A[i * n + j];
        for (int k = 0; k < j; k++) s -= A[i * n + k] * A[j * n + k];
      }
      if (base == j) {
        piv = __shfl_sync(kFull, s, 0);
        if (piv < kMinVal) piv = kMinVal;
        piv = sqrtf(piv);
      }
      if (i < n) A[i * n + j] = (i == j) ? piv : s / piv;
    }
    if (lane == 0) inv[j] = 1.0f / piv;
    __syncwarp();
  }
}
// solve L L^T x = b; x and b in shared memory (may alias); n <= 64
__device__ __noinline__ void warp_chol_solve(float* x, const float* Lm, const float* inv, const float* b, int n,
                                             int lane) {
  float r0 = lane < n ? b[lane] : 0.f;
  float r1 = lane + 32 < n ? b[lane + 32] : 0.f;
  for (int i = 0; i < n; i++) {  // forward: L y = b
    float yi = __shfl_sync(kFull, i < 32 ? r0 : r1, i & 31) * inv[i];
    if (lane == (i & 31)) { if (i < 32) r0 = yi; else r1 = yi; }
    if (lane > i && lane < n) r0 -= Lm[lane * n + i] * yi;
    if (lane + 32 > i && lane + 32 < n) r1 -= Lm[(lane + 32) * n + i] * yi;
  }
  for (int i = n - 1; i >= 0; i--) {  // backward: L^T x = y
    float xi = __shfl_sync(kFull, i < 32 ? r0 : r1, i & 31) * inv[i];
    if (lane == (i & 31)) { if (i < 32) r0 = xi; else r1 = xi; }
    if (lane < i) r0 -= Lm[i * n + lane] * xi;
    if (lane + 32 < i) r1 -= Lm[i * n + lane + 32] * xi;
  }
  if (lane < n) x[lane] = r0;
  if (lane + 32 < n) x[lane + 32] = r1;
  __syncwarp();
}
// select by bit masks (exactly one of the conditions holds): never compiled into a branch
__device__ __forceinline__ float mask_pick(float a, bool ma, float b, bool mb) {
  return __int_as_float((__float_as_int(a) & (ma ? -1 : 0)) | (__float_as_int(b) & (mb ? -1 : 0)));
}
__device__ __forceinline__ float mask_pick3(float a, bool ma, float b, bool mb, float c2, bool mc) {
  return __int_as_float((__float_as_int(a) & (ma ? -1 : 0)) | (__float_as_int(b) & (mb ? -1 : 0)) | (__float_as_int(c2) & (mc ? -1 : 0)));
}
// ---- register-resident variant for compile-time N <= 32: lane i keeps row i of the matrix in registers,
// columns are broadcast with shuffles (N(N-1)/2 SHFL + FMA), then L is written back to shared memory and
// L L^T x = b is solved (forward substitution from registers, backward substitution from shared memory rows).
template <int N>
__device__ __forceinline__ void warp_chol_factor_solve_reg(float* A, float* x, const float* b, int lane) {
  float row[N], il[N];
  const int li = lane < N ? lane : N - 1;
#pragma unroll
  for (int k = 0; k < N; k++) row[k] = A[li * N + k];
  float y = b[li];
  __syncwarp();   // lanes >= N read row N-1 / b[N-1], which lane N-1 (and x == b callers) overwrite below
  // The factorisation is a chain of N dependent (broadcast pivot -> scale column -> broadcast column -> update) steps
  // and the warp has the issue port to itself: the forward substitution L y = b rides along as one more "column"
  // (y is updated by column j as soon as that column exists) instead of a second N-step chain of its own.
#pragma unroll
  for (int j = 0; j < N; j++) {
    float p = __shfl_sync(kFull, row[j], j);
    if (p < kMinVal) p = kMinVal;
    const float l = sqrtf(p);   // (rsqrt instead of sqrt + reciprocal was measured: no change in kernel time)
    il[j] = 1.0f / l;
    const float yj = __shfl_sync(kFull, y, j) * il[j];
    // (bit-mask selection: written with ?: the compiler makes a divergent branch region of every column step)
    const float scaled = row[j] * il[j];
    row[j] = mask_pick(l, lane == j, scaled, lane != j);
    y = mask_pick3(yj, lane == j, y - scaled * yj, lane > j, y, lane < j);
#pragma unroll
    for (int k = j + 1; k < N; k++) {
      const float lkj = __shfl_sync(kFull, row[j], k);
      row[k] -= row[j] * lkj;
    }
  }
  if (lane < N) {
#pragma unroll
    for (int k = 0; k < N; k++)
      if (k <= lane) A[lane * N + k] = row[k];
  }
  __syncwarp();
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {  // backward: L^T x = y
    const float xi = __shfl_sync(kFull, y, i) * il[i];
    if (lane == i) y = xi;
    if (lane < i) y -= A[i * N + lane] * xi;
  }
  if (lane < N) x[lane] = y;
  __syncwarp();
}

// ---- leaves-first factorisation along the dof tree, for matrices whose non-zeros all pair a dof with an ancestor (qM,
// qM + h diag(damping), and the Newton Hessian when every contact is against a body without dofs).  Eliminating a dof
// only couples its ancestors, which are already coupled, so nothing fills in; dofs in different branches are
// independent, and the dependent chain is the tree's height instead of nv (Quadruped: 9 levels instead of 18 columns).
//   A = G G^T, G upper triangular: G[a][j] = A'[a][j] / l_j for every ancestor a of j (A' the matrix as updated by the
//   eliminations of j's descendants), G[j][j] = l_j.
// Lane a (< N) holds column a of A's lower triangle (A[k][a], k >= a); lane N holds b as one more row: it is an
// ancestor of every dof, and its entry j ends as y_j, the solution of G y = b (the forward substitution is part of the
// elimination and has no dependent chain of its own).  G^T x = y is then solved root-to-leaves on every lane, from G
// gathered by shuffles off the chain.  Every register access has a compile-time index (no local memory) and every
// dependence between columns is a real one, so the scheduler overlaps the branches.
// Tr: the compile-time tree of N dofs (DofTree below): anc(j) bit mask of j's ancestors, col(t) the t-th column
// eliminated (by height above the leaves, leaves first).  A is read only.  Pivots below kMinVal are clamped as in the
// dense factor.
template <int J, int B, class Tr, int N>
__device__ __forceinline__ void tree_update(float (&row)[N]) {
  if constexpr (((Tr::anc(J) >> B) & 1u) != 0u) row[B] -= row[J] * __shfl_sync(kFull, row[J], B);
}
template <int T, class Tr, int N, int... B>
__device__ __forceinline__ void tree_column(float (&row)[N], float (&il)[N], std::integer_sequence<int, B...>) {
  constexpr int J = Tr::col(T);
  float p = __shfl_sync(kFull, row[J], J);
  if (p < kMinVal) p = kMinVal;
  const float l = sqrtf(p);
  il[J] = 1.0f / l;
  row[J] *= il[J];
  (tree_update<J, B, Tr>(row), ...);
}
template <int J, int I, class Tr, int N>
__device__ __forceinline__ void tree_back_update(float& t, const float (&row)[N], const float (&xs)[N]) {
  if constexpr (((Tr::anc(J) >> I) & 1u) != 0u) t -= __shfl_sync(kFull, row[J], I) * xs[I];
}
template <int J, class Tr, int N, int... I>
__device__ __forceinline__ void tree_back(const float (&row)[N], float (&xs)[N], const float (&il)[N], std::integer_sequence<int, I...>) {
  float t = xs[J];
  (tree_back_update<J, I, Tr>(t, row, xs), ...);
  xs[J] = t * il[J];
}
template <class Tr, int N, int... T>
__device__ __forceinline__ void tree_solve(const float* A, float* x, const float* b, int lane, std::integer_sequence<int, T...> seq) {
  static_assert(N < 32, "lane N carries the right-hand side");
  float row[N], il[N], xs[N];
  const int li = lane < N ? lane : N - 1;
#pragma unroll
  for (int k = 0; k < N; k++) row[k] = lane == N ? b[k] : A[k * N + li];
  __syncwarp();   // x may alias b
  (tree_column<T, Tr>(row, il, seq), ...);
  // G^T x = y, root to leaves (a dof's ancestors have smaller indices): x_j = (y_j - sum_{i anc j} G[i][j] x_i) / l_j
#pragma unroll
  for (int j = 0; j < N; j++) xs[j] = __shfl_sync(kFull, row[j], N);
  (tree_back<T, Tr>(row, xs, il, seq), ...);
  // every lane holds all of x: same-value stores from all lanes (picking x[lane] out of xs would index it by lane,
  // which puts xs in local memory)
#pragma unroll
  for (int k = 0; k < N; k++) x[k] = xs[k];
  __syncwarp();
}
// solve A x = b (x may alias b) for a matrix with Tr's tree pattern.  ONE out-of-line copy per tree: every kernel
// instance of a model, helper-warp or one-warp, runs this same code.
template <class Tr>
__device__ __noinline__ void warp_tree_factor_solve(const float* A, float* x, const float* b, int lane) {
  tree_solve<Tr, Tr::kN>(A, x, b, lane, std::make_integer_sequence<int, Tr::kN>{});
}

// factor A (destroyed, holds L afterwards) and solve A x = b; dispatches to the register variant for the
// dof counts of the built-in models
// NS > 0: the size is a compile-time constant of a static spec (register-resident path, no dispatch)
template <int NS>
__device__ __noinline__ void warp_chol_factor_solve(float* A, float* inv, float* x, const float* b, int n, int lane) {
  if constexpr (NS > 0 && NS <= 32) { warp_chol_factor_solve_reg<NS>(A, x, b, lane); return; }
  if (n == 18) { warp_chol_factor_solve_reg<18>(A, x, b, lane); return; }
  if (n == 2) { warp_chol_factor_solve_reg<2>(A, x, b, lane); return; }
  warp_chol(A, inv, n, lane);
  warp_chol_solve(x, A, inv, b, n, lane);
}
#endif  // __CUDACC__

}  // namespace mjpc_dev
