// rollout_kernels.cuh - the CUDA kernels of the hot path (sm_90a).
//
//   rollout_kernel      one candidate trajectory per CTA: one warp (generic) or main + helper warps (static instances)
//                       (Trajectory::Rollout / RolloutDiscrete,
//                       mjpc/trajectory.cc:92-309) incl. policy, mj_step restatement, residual, cost, return
//   rank_kernel         order of each problem's candidates by return (partial_sort, sampling/planner.cc:184-188)
//   ensemble_score_kernel  each candidate's score over the member models of a model ensemble (set_model_ensemble)
//   step_batch_kernel   independent single forward+Euler steps through the same device functions (parity hooks)
//   plant_step_kernel   one step of every closed-loop plant, its state kept in device memory (plant_bank.h)
//   fd_*_kernel         finite-difference transition/residual Jacobians (model_derivatives.cc:45-165)
//
// Shared memory per CTA: [model pack (floats | ints)] [header copies] [the candidate's data]
// The model pack is staged with ONE 1-D TMA bulk copy (cp.async.bulk -> SASS UBLKCP) signalled on an mbarrier.
// Trajectory outputs are written time-major per candidate with lane-strided (coalesced) stores.
#pragma once
#include "dev_physics.cuh"
#include "dev_task.cuh"
#include "spec_quadruped.h"
#include "spec_humanoid_track.h"

namespace mjpc_dev {

// A launch holds nprob independent planning problems of nper candidates each; candidate `cand` (flat index, N = nprob *
// nper in total) belongs to problem cand / nper.  The per-problem arrays below are read once, in the prologue.
struct RolloutArgs {
  DevModel M;
  DevLayout L;
  const float* pack;        // device: nf floats followed by ni ints
  // model variants (set_model_variants): problem prob stages the block pack + pack_index[prob] * pack_stride instead;
  // pack_stride 0: every problem the one pack (pack_index unread)
  int pack_stride;
  const int* pack_index;    // [nprob]
  int nprob, nper;
  const float* state;       // [nprob][dim_state]
  const float* mocap;       // [nprob][7*nmocap]
  const float* task_state;  // [nprob][task_state_size] (times rebased to the problem's start) or nullptr
  const float* weight;      // [nprob][num_term] or nullptr (the packed Task::weight)
  const float* parameters;  // [nprob][num_parameters] or nullptr (the packed Task::parameters)
  const float* knots;       // [N][P][nu]
  const float* knot_times;  // [nprob][P], relative to the problem's start
  const PolicyInterval* iv; // [nprob][H]: each step's absolute time and its place among the policy's nodes
  double timestep;          // the step table's clock step in double: the recorded times accumulate it
  FeedbackArgs fb;
  const float* step_sizes;  // [N] for the feedback policy
  int policy_kind;          // 0 spline, 1 feedback
  float xfrc_std, xfrc_rate;   // NoisyRollout (trajectory.cc:100-210): OU force noise, std 0 = off
  unsigned noise_seed;
  int cand0;                // global index of this launch's first candidate (multi-GPU shards): noise stream = cand0 + local index
  // [nprob] or nullptr: per-problem noise keys.  Given, problem prob draws with key noise_seeds[prob] and its
  // problem-local candidate index as the stream, which is what a launch of that problem alone with that seed draws.
  const unsigned* noise_seeds;
  int P, interp, N, H;
  float* states; float* actions; double* times; float* residual; float* costs; float* trace;
  float* returns; unsigned char* failure;
  unsigned* pair_sync;      // HBM [256][32] zeroed before the launch, or nullptr: co-resident pair synchronisation (dev_data.cuh)
  long long* stats;         // [N][12]: cycles, Newton iterations, contacts, constraint rows (summed over steps), 8 phase timers
};

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// Stage the model pack into shared memory with a TMA bulk copy; all threads of the CTA must call.
__device__ __forceinline__ void stage_model_pack(float* dst, const float* src, unsigned bytes) {
  __shared__ __align__(8) unsigned long long bar;
  const unsigned bar_a = smem_u32(&bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_a), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(bar_a) : "memory");
  }
  unsigned done = 0;
  while (!done) {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done) : "r"(bar_a), "r"(0) : "memory");
  }
  __syncthreads();
}

// shared-memory words taken by the pack + header copies (must match engine.cu smem_bytes)
__host__ __device__ inline int smem_header_words(const DevModel& M) {
  return M.nf + M.ni + (int)((sizeof(DevModel) + 15) / 16) * 4 + (int)((sizeof(DevLayout) + 15) / 16) * 4;
}

// the model block a CTA of problem `prob` stages: the pack, or with model variants the problem's variant block
__device__ __forceinline__ const float* problem_pack(const float* pack, int stride, const int* index, int prob) {
  return stride ? pack + (size_t)index[prob] * stride : pack;
}

// copy the DevModel / DevLayout kernel parameters behind the pack and set up this warp's context.  `pack` is the block
// the CTA staged; with model variants (stride != 0) the last word of the variant's block is its meaninertia, which
// replaces the header's (the one float of the header a variant may change)
__device__ __forceinline__ void init_ctx(Ctx& c, const DevModel* M, const DevLayout* L, float* smem, int lane,
                                         const float* pack, int stride = 0) {
  const int hdr = M->nf + M->ni;
  const int lay = hdr + (int)((sizeof(DevModel) + 15) / 16) * 4;
  const int data0 = lay + (int)((sizeof(DevLayout) + 15) / 16) * 4;
  {
    const int* srcM = reinterpret_cast<const int*>(M);
    const int* srcL = reinterpret_cast<const int*>(L);
    int* dst = reinterpret_cast<int*>(smem);
    constexpr int kMeanInertia = (int)(offsetof(DevModel, meaninertia) / 4);
    for (int i = threadIdx.x; i < (int)(sizeof(DevModel) / 4); i += blockDim.x)
      dst[hdr + i] = stride && i == kMeanInertia ? __float_as_int(pack[stride - 1]) : srcM[i];
    for (int i = threadIdx.x; i < (int)(sizeof(DevLayout) / 4); i += blockDim.x) dst[lay + i] = srcL[i];
  }
  __syncthreads();
  c.hdr = hdr; c.lay = lay; c.ibase = M->nf;
  c.dbase = data0;
  c.lane = lane;
  c.gkey = pack + M->nf + M->ni;   // the keyframe table follows the staged part of the pack in HBM
  c.ncon = 0; c.npseudo = 0; c.xfrc_on = 0; c.nefc = 0; c.ndrow = 0; c.nitem = 0; c.niter = 0; c.nlim = 0; c.warn = 0; c.time = 0.f;
  c.sync = nullptr; c.sync_slot = -1; c.wide_pending = 0;
#ifdef MJPC_PHASE_TIMING
  for (int k = 0; k < 9; k++) c.tph[k] = 0;
  c.tlast = clock64();
#endif
}

// row `prob` of a problem's task snapshot over the CTA's shared-memory copy of the pack; a NULL array keeps the packed
// values.  The copy is per CTA and a CTA holds one candidate, so every warp of it may write the same values.
template <class SP>
__device__ __forceinline__ void load_task(Ctx& c, int prob, const float* task_state, const float* weight,
                                          const float* parameters) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  if (task_state) {
    float* ts = const_cast<float*>(MF(task_state));
    for (int i = lane; i < M.task_state_size; i += 32) ts[i] = task_state[(size_t)prob * M.task_state_size + i];
  }
  if (weight) {
    float* w = const_cast<float*>(MF(task_weight));
    for (int i = lane; i < M.num_term; i += 32) w[i] = weight[(size_t)prob * M.num_term + i];
  }
  if (parameters) {
    float* pr = const_cast<float*>(MF(task_parameters));
    for (int i = lane; i < M.num_parameters; i += 32) pr[i] = parameters[(size_t)prob * M.num_parameters + i];
  }
}

// the state a single step starts from: qpos, qvel, ctrl, the warm start (NULL: zeros) and the mocap poses ([nmocap][7]
// split into pos and quat); qM is zeroed
template <class SP>
__device__ __forceinline__ void load_state(Ctx& c, const float* qpos, const float* qvel, const float* ctrl,
                                           const float* warmstart, const float* mocap) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  for (int i = lane; i < M.nq; i += 32) DF(qpos)[i] = qpos[i];
  for (int i = lane; i < nv; i += 32) { DF(qvel)[i] = qvel[i]; DF(qacc_warmstart)[i] = warmstart ? warmstart[i] : 0.f; }
  for (int i = lane; i < M.nu; i += 32) DF(ctrl)[i] = ctrl[i];
  for (int i = lane; i < 7 * M.nmocap; i += 32) {
    const int k = i / 7, q = i - 7 * k;
    if (q < 3) DF(mocap_pos)[3 * k + q] = mocap[i]; else DF(mocap_quat)[4 * k + q - 3] = mocap[i];
  }
  for (int i = lane; i < nv * nv; i += 32) DF(qM)[i] = 0;
}

// write the trace points (GetTraces, mjpc/utilities.cc:268-285)
template <class SP>
__device__ __forceinline__ void write_traces(Ctx& c, float* out) {
  auto&& M = SP::model(c);
  const int *ty = MI(task_trace_objtype), *id = MI(task_trace_objid);
  for (int w = c.lane; w < 3 * M.num_trace; w += 32) {
    const int k = w / 3, q = w - 3 * k;
    const float* src = ty[k] == OBJ_SITE ? DF(site_xpos) : ty[k] == OBJ_GEOM ? DF(geom_xpos) : ty[k] == OBJ_XBODY ? DF(xpos) : DF(xipos);
    out[w] = src[3 * id[k] + q];
  }
}

// A standard normal from Philox4x32-10 with key (k0, k1) on counter (c0, c1, c2, c3), Box-Muller on the first two
// output words.  Key word 1 names the stream's owner: 0 the knots (host), 1 the rollouts' force noise, 2 the plants'
// disturbances and measurement noise, 3 the initial-state ensembles (belief_kernels.cuh), so no two of them ever draw
// the same numbers.
__device__ __forceinline__ float philox_normal(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0,
                                               unsigned k1) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const unsigned n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  // log u1, u1 = (c0 + 0.5) 2^-32, without rounding c0 to 24 bits where that matters: above 2^31 as log1p of minus the
  // complement (~c0 + 0.5) 2^-32, so the top counters keep their distance from u1 = 1 (fp32 u1 would round to 1 and
  // give z = 0 for the top 128 counters); below it u1 <= 1/2 and logf's relative error is what a rounded c0 adds.
  // -use_fast_math remaps logf to __logf, not log1pf.
  const float l1 = c0 >= 0x80000000u ? log1pf(-((float)(~c0) + 0.5f) * 2.3283064365386963e-10f)
                                     : logf(((float)c0 + 0.5f) * 2.3283064365386963e-10f);
  const float u2 = ((float)c1 + 0.5f) * 2.3283064365386963e-10f;
  return sqrtf(-2.0f * l1) * cospif(2.0f * u2);
}

// The Ornstein-Uhlenbeck coefficients of a noise of stationary std `std_` and time constant `rate` seconds over a step
// dt: n <- r n + s z with r = exp(-dt / rate) and s = std sqrt(1 - r^2), written as 1 + expm1 and sqrt(-expm1) so that
// neither cancels when rate >> dt (1 - r r in fp32 loses s entirely from rate ~ 1e6 dt), and r <= 1 always.
// -use_fast_math does not remap expm1f; the division is the correctly rounded one.
struct OUCoefficients { float r, s; };
__device__ __forceinline__ OUCoefficients ou_coefficients(float dt, float std_, float rate) {
  const float x = __fdiv_rn(-dt, rate);
  return {1.f + expm1f(x), std_ * sqrtf(-expm1f(2.f * x))};
}

// Injected noise of NoisyRollout: key (seed, 1), counter (step, stream, element, 'XFRC') - the definition of
// oracle/rollout.h (xfrc_normal), evaluated in fp32 here.
__device__ __forceinline__ float xfrc_normal(unsigned seed, unsigned step, unsigned stream, unsigned element) {
  return philox_normal(step, stream, element, 0x58465243u, seed, 1u);
}

// The task warp of a rollout CTA (StaticSpec<K, W, 1>): per step, between the main warp's fork / join barriers,
//   fork .. join 1 : composite inertia, velocities, smooth forces  (main: collision + constraint rows)
//   join 1 .. join 2: residual, trace, cost, the next step's spline action  (main: reference + Newton solve)
// None of these reads anything the main warp writes in the same interval (the arrays are listed per function in
// DESIGN.md section 5); every value is computed by the same code on the same inputs as in the one-warp order.
template <class SP>
__device__ __noinline__ void task_warp_loop(Ctx& c, const RolloutArgs& A, int cand) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nu = M.nu, nr = M.num_residual, ntr = 3 * M.num_trace, H = A.H;
  (void)nu;
  c.xfrc_on = A.xfrc_std > 0.f ? 1 : 0;
  float* o_res = A.residual + (size_t)cand * H * nr;
  float* o_trace = A.trace + (size_t)cand * H * ntr;
  const PolicyInterval* iv = A.iv + (size_t)(cand / A.nper) * H;
#ifdef MJPC_PHASE_TIMING
  long long fork_cycles = 0;   // timer mapping 2: this warp's fork intervals, reported by the main warp
#endif
  for (int t = 0; t < H; t++) {
    const bool last = t == H - 1;
    task_bar();   // fork (the main warp has written the state, the action and the poses of step t)
    if (wide_box().task_exit) return;
    // step t+1's interval (the last step's twice), issued here, right after the fork, so that the load has landed by
    // the end of the step where the spline reads it
    int next_upper, next_frac_bits;
    asm volatile("ld.global.nc.v2.s32 {%0, %1}, [%2];" : "=r"(next_upper), "=r"(next_frac_bits) : "l"(&iv[min(t + 1, H - 1)].upper));
    const float next_frac = __int_as_float(next_frac_bits);
#ifdef MJPC_PHASE_TIMING
    const long long t_fork = clock64();
#endif
    k_crb<SP>(c);
    k_com_vel<SP>(c);
    k_smooth_forces<SP>(c);
#ifdef MJPC_PHASE_TIMING
    fork_cycles += clock64() - t_fork;
    if (lane == 0) wide_box().task_fork_cycles = fork_cycles;
#endif
    task_bar();   // join 1
    k_residual<SP>(c);
    for (int i = lane; i < nr; i += 32) o_res[(size_t)t * nr + i] = DF(residual)[i];
    write_traces<SP>(c, o_trace + (size_t)t * ntr);
    const float cost = k_cost_value<SP>(c);
    if (lane == 0) { wide_box().task_cost = cost; wide_box().task_warn = c.warn; }   // (a residual can raise a warning)
    if (!last) {
      c.time += CM(c).timestep;   // the same sum k_euler forms on the main warp
      if (A.policy_kind == 0 && t + 1 < H - 1) k_policy_spline<SP>(c, A.P, A.interp, next_upper, next_frac);
    }
    task_bar();   // join 2
  }
}

template <class SP>
__device__ __forceinline__ void rollout_body(const RolloutArgs& A) {
  float* smem = g_smem;
  // (blockIdx.x is the candidate in every instance: the one-warp ones have one warp)
  const float* pack = problem_pack(A.pack, A.pack_stride, A.pack_index, (int)blockIdx.x / A.nper);
  stage_model_pack(smem, pack, (unsigned)((A.M.nf + A.M.ni) * 4));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // the CTA is ONE candidate (SP::kWide > 1: warp 0 runs the pipeline, the others help with the wide phases).  The
  // one-warp instances add their warp index, 0: with blockIdx.x alone the Humanoid Track one is compiled to 128
  // registers and spills.
  const int cand = (SP::kWide > 1 || SP::kTask > 0) ? (int)blockIdx.x : (int)blockIdx.x + warp;
  Ctx c;
  init_ctx(c, &A.M, &A.L, smem, lane, pack, A.pack_stride);
  if (cand >= A.N) return;
  if (SP::kWide > 1 && warp > 0 && warp < SP::kWide) { wide_helper_loop<SP>(c); return; }
  if (SP::kTask > 0 && warp == SP::kWide) { task_warp_loop<SP>(c, A, cand); return; }
  constexpr bool kTask = SP::kTask > 0;
  if (kTask && lane == 0) wide_box().task_exit = 0;
  if constexpr (SP::kWide > 1) pair_sync_init(c, A.pair_sync);
  auto&& M = SP::model(c);
  const int nq = M.nq, nv = M.nv, nu = M.nu, ds = nq + nv, nr = M.num_residual, ntr = 3 * M.num_trace, H = A.H;
  // this candidate's problem: its inputs are resolved here, the step loop below only sees Ctx, the step table and the outputs
  const int prob = cand / A.nper;
  const PolicyInterval* iv = A.iv + (size_t)prob * A.H;
  const float* state = A.state + (size_t)prob * ds;
  const float* mocap = A.mocap + (size_t)prob * 7 * M.nmocap;
  // the problem's task snapshot (task state time-rebased) overrides the packed copy.  With a task warp this happens
  // before its first fork, where it starts to read them.
  load_task<SP>(c, prob, A.task_state, A.weight, A.parameters);
  // ---- initial conditions (trajectory.cc:108-137)
  // (written out rather than through load_state: through the helper the rollout kernels compile to different SASS)
  for (int i = lane; i < nq; i += 32) DF(qpos)[i] = state[i];
  for (int i = lane; i < nv; i += 32) { DF(qvel)[i] = state[nq + i]; DF(qacc_warmstart)[i] = 0; }
  for (int i = lane; i < 7 * M.nmocap; i += 32) {
    const int k = i / 7, q = i - 7 * k;
    if (q < 3) DF(mocap_pos)[3 * k + q] = mocap[i]; else DF(mocap_quat)[4 * k + q - 3] = mocap[i];
  }
  for (int i = lane; i < nv * nv; i += 32) DF(qM)[i] = 0;
  const bool noisy = A.xfrc_std > 0.f;
  const OUCoefficients ou = noisy ? ou_coefficients(CM(c).timestep, A.xfrc_std, A.xfrc_rate) : OUCoefficients{0.f, 0.f};
  const float ou_rate = ou.r, ou_scale = ou.s;
  // the noise key and stream of this candidate: kept in shared memory rather than in registers across the step loop:
  // two more live registers there made the Quadruped one-warp and Humanoid Track helper-warp instances spill
  __shared__ unsigned noise_ks[2];
  if (noisy && lane == 0) {   // (published to the warp by the __syncwarp below)
    noise_ks[0] = A.noise_seeds ? A.noise_seeds[prob] : A.noise_seed;
    noise_ks[1] = A.noise_seeds ? (unsigned)(cand - prob * A.nper) : (unsigned)(A.cand0 + cand);
  }
  for (int i = lane; i < 6 * M.nbody; i += 32) DF(xfrc)[i] = 0;
  c.xfrc_on = noisy ? 1 : 0;
  float step_size = 0.f;
  if (A.policy_kind == 0) {
    for (int i = lane; i < A.P * nu; i += 32) DF(knots)[i] = A.knots[(size_t)cand * A.P * nu + i];
    for (int i = lane; i < A.P; i += 32) DF(knot_times)[i] = A.knot_times[(size_t)prob * A.P + i];
  } else {
    step_size = A.step_sizes[cand];
  }
  __syncwarp();
  float* o_states = A.states + (size_t)cand * H * ds;
  float* o_actions = A.actions + (size_t)cand * H * nu;
  double* o_times = A.times + (size_t)cand * H;
  float* o_res = A.residual + (size_t)cand * H * nr;
  float* o_costs = A.costs + (size_t)cand * H;
  float* o_trace = A.trace + (size_t)cand * H * ntr;
  for (int i = lane; i < ds; i += 32) o_states[i] = state[i];
  // T[t], the reference's rollout clock, accumulated in double as the step table's (c.time is its fp32 relative twin)
  double time = iv[0].time;
  if (lane == 0) o_times[0] = time;
  int next_upper = iv[0].upper;   // the spline's interval of the coming step
  float next_frac = iv[0].frac;
  float total = 0.f;
  bool failed = false;
  const long long clk0 = clock64();
  long long n_newton = 0, n_con = 0, n_efc = 0;
  for (int t = 0; t < H; t++) {
    const bool last = t == H - 1;
    if constexpr (SP::kWide > 1) pair_sync_meet(c, t);
    // (with a task warp the spline action of step t > 0 was evaluated by it during step t-1's constraint solve)
    if (!last) {
      if (A.policy_kind == 0) {
        const int upper = next_upper;
        const float frac = next_frac;
        if (!kTask) { next_upper = iv[t + 1].upper; next_frac = iv[t + 1].frac; }   // read a step ahead
        if (!kTask || t == 0) k_policy_spline<SP>(c, A.P, A.interp, upper, frac);
      }
      else k_policy_feedback<SP>(c, A.fb, step_size, t, cand);
    }
    // action record (the last row repeats the previous action; H == 1 -> zeros; trajectory.cc:190-196)
    for (int i = lane; i < nu; i += 32) {
      if (H == 1) DF(ctrl)[i] = 0;
      o_actions[(size_t)t * nu + i] = DF(ctrl)[i];
    }
    if (!last && (k_bad(c, DF(qpos), nq) || k_bad(c, DF(qvel), nv))) {
      failed = true;
      if (kTask) { if (lane == 0) wide_box().task_exit = 1; task_bar(); }   // the task warp waits at the fork
      break;
    }
    if (noisy && !last) {   // Ornstein-Uhlenbeck perturbation in discrete time (trajectory.cc:147-155)
      float* xf = DF(xfrc);
      for (int i = lane; i < 6 * M.nbody; i += 32)
        xf[i] = ou_rate * xf[i] + ou_scale * xfrc_normal(noise_ks[0], (unsigned)t, noise_ks[1], (unsigned)i);
      __syncwarp();
    }
    float cost;
    if constexpr (kTask) {
      // the step as a fork / join graph (the one-warp order is k_forward, dev_physics.cuh):
      //   main: kinematics, com | collision, constraint rows        | reference, Newton solve           | Euler
      //   task:                 | CRB, velocities, smooth forces    | residual, cost, next spline action |
      PHASE(c, 7); PHASE_AT(c, 2, 7);
      wide_settle<SP>(c);   // the last step's abandoned Hessian assembly reads poses, cdof, qM and the contacts
      k_kinematics<SP>(c);
      k_com_pos<SP>(c);
      PHASE(c, 0); PHASE_AT(c, 2, 0);
      task_bar();   // fork
      k_collision<SP>(c);
      PHASE(c, 1); PHASE_AT(c, 2, 1);
      k_make_constraint<SP>(c);
      PHASE(c, 2); PHASE_AT(c, 2, 2);
      task_bar();   // join: qM, qfrc_smooth, qacc_smooth are in place
      PHASE_AT(c, 2, 3);
      k_reference<SP>(c);
      PHASE(c, 3);
      k_solve<SP>(c);
      PHASE(c, 4); PHASE_AT(c, 2, 4);
      n_newton += c.niter; n_con += c.ncon - c.npseudo; n_efc += c.nefc;
      if (!last && k_bad(c, DF(qacc), nv)) c.warn = 1;
      task_bar();   // join: residual, trace and cost of this step are written, ctrl holds the next action
      cost = wide_box().task_cost;
      if (wide_box().task_warn) c.warn = 1;
    } else {
      k_forward<SP>(c);
      n_newton += c.niter; n_con += c.ncon - c.npseudo; n_efc += c.nefc;
      k_residual<SP>(c);
      if (!last && k_bad(c, DF(qacc), nv)) c.warn = 1;
      for (int i = lane; i < nr; i += 32) o_res[(size_t)t * nr + i] = DF(residual)[i];
      write_traces<SP>(c, o_trace + (size_t)t * ntr);
    }
    if (c.warn) {
      failed = true;
      if (kTask && !last) { if (lane == 0) wide_box().task_exit = 1; task_bar(); }
      break;
    }
    if constexpr (!kTask) cost = k_cost_value<SP>(c);
    if (lane == 0) o_costs[t] = cost;
    total += cost;
    if (last) break;
    for (int i = lane; i < nv; i += 32) DF(qacc_warmstart)[i] = DF(qacc)[i];
    k_euler<SP>(c);
    for (int i = lane; i < nq; i += 32) o_states[(size_t)(t + 1) * ds + i] = DF(qpos)[i];
    for (int i = lane; i < nv; i += 32) o_states[(size_t)(t + 1) * ds + nq + i] = DF(qvel)[i];
    time += A.timestep;
    if (lane == 0) o_times[t + 1] = time;
  }
  pair_sync_done(c);
  wide_settle<SP>(c);
  wide_post<SP>(c, WIDE_EXIT);   // releases the helper warps
  if (lane == 0) {
    A.returns[cand] = failed ? 1.0e6f : total / (float)max(H, 1);
    A.failure[cand] = failed ? 1 : 0;
    if (A.stats) {
      A.stats[12 * cand] = clock64() - clk0; A.stats[12 * cand + 1] = n_newton;
      A.stats[12 * cand + 2] = n_con; A.stats[12 * cand + 3] = n_efc;
#if defined(MJPC_PHASE_TIMING) && MJPC_PHASE_MAP == 2
      if constexpr (kTask) c.tph[5] = wide_box().task_fork_cycles;
#endif
      for (int k = 0; k < 8; k++) {
#ifdef MJPC_PHASE_TIMING
        A.stats[12 * cand + 4 + k] = c.tph[k];
#else
        A.stats[12 * cand + 4 + k] = 0;
#endif
      }
#ifndef MJPC_PHASE_TIMING
      // placement diagnostics (profiles/placement.py): which SM and which hardware warp slot ran this candidate
      unsigned smid, warpid;
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
      asm volatile("mov.u32 %0, %%warpid;" : "=r"(warpid));
      A.stats[12 * cand + 4] = smid; A.stats[12 * cand + 5] = warpid;
#endif
    }
  }
}

extern "C" __global__ void __launch_bounds__(32) rollout_kernel(const __grid_constant__ RolloutArgs A) {
  rollout_body<DynSpec>(A);
}
// statically specialised instance for the Quadruped (flat) task model (spec_quadruped.h); one warp per CTA
// Static instances: the shipped one holds kRolloutWide + kRolloutTask warps per candidate (main warp, Hessian helper warps,
// task warp: DESIGN.md section 5 "helper warps"; 7 + 1 since the Hessian runs on the helpers alone: 6 helpers cover the
// 171 Hessian entries of the A1 in one round, measured faster than 6 + 1 at 256 candidates).  The *_plain instance is
// the same source with ONE warp per candidate: the reference the helper-warp kernel must equal bit for bit
// (tests/test_gpu_parity.py, MJPC_B200_SHAPE=plain) and the baseline of the profiles.
constexpr int kRolloutWide = 7, kRolloutTask = 1, kRolloutThreads = 32 * (kRolloutWide + kRolloutTask);
extern "C" __global__ void __launch_bounds__(kRolloutThreads) rollout_kernel_quadruped(const __grid_constant__ RolloutArgs A) {
  rollout_body<StaticSpec<SpecQuadruped, kRolloutWide, kRolloutTask>>(A);
}
extern "C" __global__ void __launch_bounds__(32) rollout_kernel_quadruped_plain(const __grid_constant__ RolloutArgs A) {
  rollout_body<StaticSpec<SpecQuadruped, 1, 0>>(A);
}
// ... and for the Humanoid Track task model (spec_humanoid_track.h)
extern "C" __global__ void __launch_bounds__(kRolloutThreads) rollout_kernel_humanoid_track(const __grid_constant__ RolloutArgs A) {
  rollout_body<StaticSpec<SpecHumanoidTrack, kRolloutWide, kRolloutTask>>(A);
}
extern "C" __global__ void __launch_bounds__(32) rollout_kernel_humanoid_track_plain(const __grid_constant__ RolloutArgs A) {
  rollout_body<StaticSpec<SpecHumanoidTrack, 1, 0>>(A);
}

// host: do the live model header / state layout / dof tree equal the table a static kernel was compiled from?
// (float options are not part of the comparison: static kernels read them from the live header)
template <class K>
inline bool spec_matches(const DevModel& M, const DevLayout& L, const int* dof_parent) {
  if (K::kNumModelWords != (int)(sizeof(DevModel) / 4) || K::kNumLayout != (int)D_COUNT) return false;
  const int* w = K::kModelWords;
#define X(n) if (w[offsetof(DevModel, n) / 4] != M.n) return false;
  MJPC_M_INTS(X)
#undef X
  for (int i = 0; i < F_COUNT; i++) if (w[offsetof(DevModel, fo) / 4 + i] != M.fo[i]) return false;
  for (int i = 0; i < I_COUNT; i++) if (w[offsetof(DevModel, io) / 4 + i] != M.io[i]) return false;
  for (int i = 0; i < D_COUNT; i++) if (K::kLayoutOff[i] != L.off[i]) return false;
  for (int i = 0; i < M.nv; i++) if (K::kDofParent[i] != dof_parent[i]) return false;
  return true;
}

// nseg segments of N returns: order[b][rank] = i, the index within segment b, ascending return, ties broken by index,
// NaN after every number and NaNs among themselves by index (numpy's stable argsort), so every segment is a permutation
extern "C" __global__ void rank_kernel(const float* __restrict__ ret, int N, int nseg, int* __restrict__ order) {
  for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < nseg * N; g += gridDim.x * blockDim.x) {
    const int b = g / N, i = g - b * N;
    const float* r = ret + (size_t)b * N;
    const float ri = r[i];
    int rank = 0;
    for (int j = 0; j < N; j++) {
      const float rj = r[j];
      rank += (rj < ri) || (rj == ri && j < i) || (ri != ri && (rj == rj || j < i));
    }
    order[(size_t)b * N + rank] = i;
  }
}

// The score of each candidate of a launch rolled out on K member models (set_model_ensemble): one warp per candidate
// (b, i) of B problems x N candidates, lane k holding member k, which the rollout left at [(b K + k) N + i].  The member
// returns are sorted in descending order (ties to the lower member, NaN first), the first `worst` summed left to right
// in double and divided once by worst: ret [B][N].  A candidate that failed on any member fails with return 1e6.
// mjpc_b200_host_ensemble_score is the host definition, bit for bit.
extern "C" __global__ void ensemble_score_kernel(const float* __restrict__ member_ret,
                                                 const unsigned char* __restrict__ member_fail, int B, int K, int N,
                                                 int worst, float* __restrict__ ret, unsigned char* __restrict__ failure) {
  const int lane = threadIdx.x & 31;
  const int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (c >= B * N) return;   // (the whole warp)
  const int b = c / N, i = c - b * N;
  const bool member = lane < K;
  const size_t at = ((size_t)b * K + lane) * N + i;
  const float r = member ? member_ret[at] : 0.f;
  const unsigned failed = __ballot_sync(~0u, member && member_fail[at]);
  int rank = 0;   // the members sorted before this one
  for (int j = 0; j < K; j++) {
    const float rj = __shfl_sync(~0u, r, j);
    rank += (rj > r) || (rj == r && j < lane) || (rj != rj && (r == r || j < lane));
  }
  double sum = 0.0;
  for (int p = 0; p < worst; p++) {
    const int src = __ffs(__ballot_sync(~0u, member && rank == p)) - 1;
    sum = __dadd_rn(sum, (double)__shfl_sync(~0u, r, src));
  }
  if (lane == 0) {
    ret[c] = failed ? 1.0e6f : __double2float_rn(__ddiv_rn(sum, (double)worst));
    failure[c] = failed ? 1 : 0;
  }
}

// Single-step parity hook: B independent (qpos, qvel, ctrl, warm start, time) tuples, each advanced by ONE mj_step
// through the same device functions - and the same static / generic instances - the rollout kernel runs.
// Teacher-forced per-step parity tests feed it the oracle's own states, so a mismatch cannot be blamed on trajectory
// divergence.
struct StepBatchArgs {
  DevModel M;
  DevLayout L;
  const float* pack;
  const float* qpos; const float* qvel; const float* ctrl; const float* warmstart;   // [B][nq|nv|nu|nv]
  const float* mocap; const float* task_state;
  const float* time;    // [B], relative to the rollout start the task state was rebased to
  int B;
  float* qacc; float* next_qpos; float* next_qvel; float* residual; float* cost; int* counts;   // counts [B][4]
  // optional (NULL: not written): qM [B][nv nv], efc_force [B][maxefc], contact [B][maxcon][8] = dist, pos[3],
  // normal[3], dim of the geometric contacts
  float* qM; float* efc_force; float* contact;
  // optional (NULL: not evaluated): the measurement sensors sensors[0, nsensor) (k_sensors), sensordata [B][sensor_dim]
  // from address sensor_adr0 on
  const DevSensor* sensors; int nsensor, sensor_adr0, sensor_dim; float* sensordata;
  // row b's mocap poses start at mocap + b mocap_stride: 0 shares one set, 7 nmocap gives each row its own
  int mocap_stride;
  // model variants: row b steps on variant pack_index[b / pack_rows] (problem_pack); pack_stride 0: the one pack
  int pack_stride, pack_rows;
  const int* pack_index;
};

template <class SP>
__device__ __forceinline__ void step_batch_body(const StepBatchArgs& A) {
  float* smem = g_smem;
  const int b = blockIdx.x;
  const float* pack = problem_pack(A.pack, A.pack_stride, A.pack_index, A.pack_stride ? b / A.pack_rows : 0);
  stage_model_pack(smem, pack, (unsigned)((A.M.nf + A.M.ni) * 4));
  Ctx c;
  init_ctx(c, &A.M, &A.L, smem, threadIdx.x, pack, A.pack_stride);
  auto&& M = SP::model(c);
  const int lane = c.lane, nq = M.nq, nv = M.nv, nu = M.nu, nr = M.num_residual;
  if (b >= A.B) return;
  load_task<SP>(c, 0, A.task_state, nullptr, nullptr);
  load_state<SP>(c, A.qpos + (size_t)b * nq, A.qvel + (size_t)b * nv, A.ctrl + (size_t)b * nu,
                 A.warmstart ? A.warmstart + (size_t)b * nv : nullptr, A.mocap + (size_t)b * A.mocap_stride);
  for (int i = lane; i < 6 * M.nbody; i += 32) DF(xfrc)[i] = 0;
  c.time = A.time[b];
  __syncwarp();
  k_forward<SP>(c);
  k_residual<SP>(c);
  if (k_bad(c, DF(qacc), nv)) c.warn = 1;
  const float cost = k_cost_value<SP>(c);
  const int ncon = c.ncon - c.npseudo;
  for (int i = lane; i < nv; i += 32) A.qacc[(size_t)b * nv + i] = DF(qacc)[i];
  for (int i = lane; i < nr; i += 32) A.residual[(size_t)b * nr + i] = DF(residual)[i];
  if (lane == 0) {
    A.cost[b] = cost;
    A.counts[4 * b] = ncon; A.counts[4 * b + 1] = c.nefc; A.counts[4 * b + 2] = c.niter; A.counts[4 * b + 3] = c.warn;
  }
  if (A.qM)
    for (int i = lane; i < nv * nv; i += 32) A.qM[(size_t)b * nv * nv + i] = DF(qM)[i];
  if (A.efc_force)
    for (int i = lane; i < c.nefc; i += 32) A.efc_force[(size_t)b * M.maxefc + i] = DF(efc_force)[i];
  if (A.contact)
    for (int i = lane; i < ncon; i += 32) {
      float* o = A.contact + ((size_t)b * M.maxcon + i) * 8;
      o[0] = DF(con_dist)[i];
      for (int q = 0; q < 3; q++) { o[1 + q] = DF(con_pos)[3 * i + q]; o[4 + q] = DF(con_frame)[9 * i + q]; }
      const int d = DI(con_dim)[i];   // the pyramidal constraint phase rewrites it as the row count 2 (dim - 1)
      o[7] = (float)(M.cone == CONE_PYRAMIDAL && d > 1 ? d / 2 + 1 : d);
    }
  if (A.sensordata) k_sensors<SP>(c, A.sensors, A.nsensor, A.sensor_adr0, A.sensordata + (size_t)b * A.sensor_dim);
  for (int i = lane; i < nv; i += 32) DF(qacc_warmstart)[i] = DF(qacc)[i];
  k_euler<SP>(c);
  for (int i = lane; i < nq; i += 32) A.next_qpos[(size_t)b * nq + i] = DF(qpos)[i];
  for (int i = lane; i < nv; i += 32) A.next_qvel[(size_t)b * nv + i] = DF(qvel)[i];
}
extern "C" __global__ void __launch_bounds__(32) step_batch_kernel(const __grid_constant__ StepBatchArgs A) {
  step_batch_body<DynSpec>(A);
}
// The one-step entry points (step_batch, and step_sensors: the estimators' sigma-point and finite-difference steps) and
// the plant steps, which must equal them, keep the dense factor: the Kalman filter differentiates these steps with 1e-3 differences, and through a hard contact solve
// a rounding change can move where the Newton iteration stops by its tolerance, which those differences amplify.
extern "C" __global__ void __launch_bounds__(32) step_batch_kernel_quadruped(const __grid_constant__ StepBatchArgs A) {
  step_batch_body<StaticSpec<SpecQuadruped, 1, 0, true>>(A);
}
extern "C" __global__ void __launch_bounds__(32) step_batch_kernel_humanoid_track(const __grid_constant__ StepBatchArgs A) {
  step_batch_body<StaticSpec<SpecHumanoidTrack, 1, 0, true>>(A);
}

// Closed-loop plants (plant_bank.h): B plants whose state stays in device memory, each advanced by ONE mj_step per
// launch through the device functions and the order of step_batch_body, on its own model variant and task rows.  The
// step of a running plant whose next qpos, qvel and qacc are finite is committed in place (state, warm start carried
// as MuJoCo's qacc_warmstart, time, cost sum, step and warning counts); otherwise the plant becomes PLANT_DIVERGED and
// keeps what it had.  A plant that is not running is not stepped.  The outputs of a plant that did not step hold its
// state and time, cost 0 and zero sensors; its applied ctrl is the ctrl its step was given (commanded + control noise),
// or the commanded ctrl when it is not running.  The disturbances' OU states advance only with a committed step.
enum PlantStatus { PLANT_RUNNING = 0, PLANT_DIVERGED = 1, PLANT_IDLE = 2 };

// A plant's disturbances (mjpc_b200_plant_set_disturbance / _set_xfrc / _set_sensor_noise): Ornstein-Uhlenbeck control
// noise and body-force noise (std 0: off; the rate is the time constant in seconds), the key of its noise stream,
// whether it holds a non-zero wrench and whether any of its sensor-noise stds is > 0
struct PlantDisturbance {
  float ctrl_std, ctrl_rate, xfrc_std, xfrc_rate;
  unsigned seed;
  int held;
  int sens;
};

// Plant noise: Philox key (seed, 2), counter (committed step count, 0, element, tag)
constexpr unsigned kPlantTagCtrl = 0x4354524Cu;   // 'CTRL'
constexpr unsigned kPlantTagXfrc = 0x58465243u;   // 'XFRC'
constexpr unsigned kPlantTagSens = 0x53454E53u;   // 'SENS'
__device__ __forceinline__ float plant_normal(unsigned seed, unsigned step, unsigned element, unsigned tag) {
  return philox_normal(step, 0u, element, tag, seed, 2u);
}

struct PlantArgs {
  DevModel M;
  DevLayout L;
  const float* pack;
  int pack_stride;          // model variants: plant b stages its variant block (problem_pack); 0: the one pack
  const int* pack_index;
  int B;
  double timestep;
  // the bank, read and committed in place
  float* qpos; float* qvel; float* warm;   // [B][nq|nv|nv]
  double* time; double* cost_sum;          // [B]
  int* steps; int* warnings; int* status;  // [B]
  // this step's upload: ctrl [B][nu], mocap [B][7 nmocap], and the task rows with the task state rebased to each plant's
  // time: task_state [B][size] (nullptr when empty), weight [B][num_term], parameters [B][num_parameters] (nullptr: none)
  const float* ctrl; const float* mocap; const float* task_state; const float* weight; const float* parameters;
  // this step's outputs: state [B][nq+nv], time [B], cost [B] (the pre-step residual's), status [B]
  float* state_out; double* time_out; float* cost_out; int* status_out;
  // optional (sensordata NULL: not evaluated): sensors [0, nsensor) of the pre-step state, [B][sensor_dim]
  const DevSensor* sensors; int nsensor, sensor_adr0, sensor_dim; float* sensordata;
  // disturbances: settings dist [B]; OU states ctrl_noise [B][nu] and xfrc_noise [B][6 nbody]; the held wrench
  // xfrc_held [B][6 nbody]; noise_next [B][nu + 6 nbody], this step's OU states until the step is committed
  const PlantDisturbance* dist; float* ctrl_noise; float* xfrc_noise; const float* xfrc_held; float* noise_next;
  float* ctrl_out;   // output: the applied ctrl [B][nu] (commanded + control noise)
  const float* sensor_std;   // measurement noise std [B][sensor_dim] (read only for a plant whose dist.sens is set)
};

// The disturbances of plant b's coming step, between load_state and k_forward (app.cc:291-304, 95-101, 323-352):
// control noise n <- r n + s z (r = exp(-timestep / rate), s = std sqrt(1 - r^2), ou_coefficients) added to the ctrl, which actuation
// clamps as any ctrl; xfrc = the held wrench + the force noise's state under the same recursion.  The advanced states go
// to noise_next; the applied ctrl is written out.
template <class SP>
__device__ __forceinline__ void plant_disturb(Ctx& c, const PlantArgs& A, int b) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nu = M.nu, nx = 6 * M.nbody;
  const PlantDisturbance& d = A.dist[b];
  const unsigned step = (unsigned)A.steps[b];
  float* next = A.noise_next + (size_t)b * (nu + nx);
  if (d.ctrl_std > 0.f) {
    const OUCoefficients ou = ou_coefficients(CM(c).timestep, d.ctrl_std, d.ctrl_rate);
    const float r = ou.r, s = ou.s;
    const float* n = A.ctrl_noise + (size_t)b * nu;
    for (int i = lane; i < nu; i += 32) {
      const float v = r * n[i] + s * plant_normal(d.seed, step, (unsigned)i, kPlantTagCtrl);
      next[i] = v;
      DF(ctrl)[i] += v;
    }
  }
  for (int i = lane; i < nu; i += 32) A.ctrl_out[(size_t)b * nu + i] = DF(ctrl)[i];
  const float* held = A.xfrc_held + (size_t)b * nx;
  if (d.xfrc_std > 0.f) {
    const OUCoefficients ou = ou_coefficients(CM(c).timestep, d.xfrc_std, d.xfrc_rate);
    const float r = ou.r, s = ou.s;
    const float* n = A.xfrc_noise + (size_t)b * nx;
    for (int i = lane; i < nx; i += 32) {
      const float v = r * n[i] + s * plant_normal(d.seed, step, (unsigned)i, kPlantTagXfrc);
      next[nu + i] = v;
      DF(xfrc)[i] = held[i] + v;
    }
    c.xfrc_on = 1;
  } else if (d.held) {
    for (int i = lane; i < nx; i += 32) DF(xfrc)[i] = held[i];
    c.xfrc_on = 1;
  }
}

// a committed step advances plant b's OU states to noise_next (each lane copies what it wrote in plant_disturb)
__device__ __forceinline__ void plant_commit_noise(const PlantArgs& A, int b, int lane) {
  const PlantDisturbance& d = A.dist[b];
  const int nu = A.M.nu, nx = 6 * A.M.nbody;
  const float* next = A.noise_next + (size_t)b * (nu + nx);
  if (d.ctrl_std > 0.f)
    for (int i = lane; i < nu; i += 32) A.ctrl_noise[(size_t)b * nu + i] = next[i];
  if (d.xfrc_std > 0.f)
    for (int i = lane; i < nx; i += 32) A.xfrc_noise[(size_t)b * nx + i] = next[nu + i];
}

// The measurement noise of plant b's committed step, after the step is committed: sensordata[e] += std[e] z on counter
// (the committed step count before this step, 0, e, 'SENS').  Elements whose std is 0 are not touched.  Only the
// returned measurement changes.
__device__ __forceinline__ void plant_sensor_noise(const PlantArgs& A, int b, int lane) {
  const unsigned seed = A.dist[b].seed, step = (unsigned)A.steps[b] - 1u;
  const float* sd = A.sensor_std + (size_t)b * A.sensor_dim;
  float* out = A.sensordata + (size_t)b * A.sensor_dim;
  for (int e = lane; e < A.sensor_dim; e += 32)
    if (sd[e] > 0.f) out[e] += sd[e] * plant_normal(seed, step, (unsigned)e, kPlantTagSens);
}

template <class SP>
__device__ __forceinline__ void plant_body(const PlantArgs& A) {
  float* smem = g_smem;
  const int b = blockIdx.x;
  if (b >= A.B) return;
  const bool running = A.status[b] == PLANT_RUNNING;
  bool stepped = false;
  float cost = 0.f;
  Ctx c;
  if (running) {
    // (a state set or reset to non-finite values diverges before it is stepped)
    const float* pack = problem_pack(A.pack, A.pack_stride, A.pack_index, b);
    stage_model_pack(smem, pack, (unsigned)((A.M.nf + A.M.ni) * 4));
    init_ctx(c, &A.M, &A.L, smem, threadIdx.x, pack, A.pack_stride);
    auto&& M = SP::model(c);
    const int lane = c.lane, nq = M.nq, nv = M.nv;
    load_task<SP>(c, b, A.task_state, A.weight, A.parameters);
    load_state<SP>(c, A.qpos + (size_t)b * nq, A.qvel + (size_t)b * nv, A.ctrl + (size_t)b * M.nu,
                   A.warm + (size_t)b * nv, A.mocap + (size_t)b * 7 * M.nmocap);
    for (int i = lane; i < 6 * M.nbody; i += 32) DF(xfrc)[i] = 0;
    plant_disturb<SP>(c, A, b);
    __syncwarp();   // c.time stays 0: the task state was rebased to the plant's time
    if (!(k_bad(c, DF(qpos), nq) || k_bad(c, DF(qvel), nv))) {
      // step_batch_body's sequence (written out again: through one shared function the step_batch instances compile
      // to different SASS)
      k_forward<SP>(c);
      k_residual<SP>(c);
      if (k_bad(c, DF(qacc), nv)) c.warn = 1;
      cost = k_cost_value<SP>(c);
      if (A.sensordata) k_sensors<SP>(c, A.sensors, A.nsensor, A.sensor_adr0, A.sensordata + (size_t)b * A.sensor_dim);
      for (int i = lane; i < nv; i += 32) DF(qacc_warmstart)[i] = DF(qacc)[i];
      k_euler<SP>(c);
      stepped = !(k_bad(c, DF(qpos), nq) || k_bad(c, DF(qvel), nv) || k_bad(c, DF(qacc), nv));
    }
    if (stepped) {
      plant_commit_noise(A, b, lane);
      for (int i = lane; i < nq; i += 32) A.qpos[(size_t)b * nq + i] = DF(qpos)[i];
      for (int i = lane; i < nv; i += 32) { A.qvel[(size_t)b * nv + i] = DF(qvel)[i]; A.warm[(size_t)b * nv + i] = DF(qacc)[i]; }
      if (lane == 0) {
        A.time[b] += A.timestep;
        A.cost_sum[b] += (double)cost;
        A.steps[b] += 1;
        A.warnings[b] += c.warn;
      }
    } else if (lane == 0) {
      A.status[b] = PLANT_DIVERGED;
    }
    __syncwarp();
  }
  const int lane = threadIdx.x, nq = A.M.nq, ds = nq + A.M.nv;
  if (!running)
    for (int i = lane; i < A.M.nu; i += 32) A.ctrl_out[(size_t)b * A.M.nu + i] = A.ctrl[(size_t)b * A.M.nu + i];
  for (int i = lane; i < ds; i += 32)
    A.state_out[(size_t)b * ds + i] = i < nq ? A.qpos[(size_t)b * nq + i] : A.qvel[(size_t)b * A.M.nv + i - nq];
  if (A.sensordata && !stepped)
    for (int i = lane; i < A.sensor_dim; i += 32) A.sensordata[(size_t)b * A.sensor_dim + i] = 0.f;
  // (the __syncwarp above made the committed step count and k_sensors' values visible to every lane)
  if (stepped && A.dist[b].sens) plant_sensor_noise(A, b, lane);
  if (lane == 0) {
    A.time_out[b] = A.time[b];
    A.cost_out[b] = stepped ? cost : 0.f;
    A.status_out[b] = A.status[b];
  }
}
extern "C" __global__ void __launch_bounds__(32) plant_step_kernel(const __grid_constant__ PlantArgs A) {
  plant_body<DynSpec>(A);
}
extern "C" __global__ void __launch_bounds__(32) plant_step_kernel_quadruped(const __grid_constant__ PlantArgs A) {
  plant_body<StaticSpec<SpecQuadruped, 1, 0, true>>(A);
}
extern "C" __global__ void __launch_bounds__(32) plant_step_kernel_humanoid_track(const __grid_constant__ PlantArgs A) {
  plant_body<StaticSpec<SpecHumanoidTrack, 1, 0, true>>(A);
}

}  // namespace mjpc_dev
