/* mjpc_b200.h - C ABI of the H100 (sm_90a) rollout engine (libmjpc_b200.so).
 *
 * The engine replaces the data-parallel hot path of MJPC and nothing else.  std::function policies and
 * virtual ResidualFn objects cannot cross to the device, so every entry point takes *data* and sits exactly
 * where the reference fans work out over its ThreadPool:
 *
 *   mjpc_b200_rollout_spline    <- SamplingPlanner::Rollouts            mjpc/planners/sampling/planner.cc:355-393
 *                                  (+ Trajectory::Rollout/NoisyRollout  mjpc/trajectory.cc:92-210,
 *                                     SamplingPolicy::Action            mjpc/planners/sampling/policy.cc:52-59,
 *                                     UpdateReturn                      mjpc/trajectory.cc:312-326,
 *                                     partial_sort by return            mjpc/planners/sampling/planner.cc:184-188)
 *   mjpc_b200_rollout_feedback  <- iLQGPlanner::FeedbackRollouts / ActionRollouts
 *                                                                       mjpc/planners/ilqg/planner.cc:630-724
 *                                  (+ iLQGPolicy::Action                mjpc/planners/ilqg/policy.cc:82-161,
 *                                     Trajectory::RolloutDiscrete       mjpc/trajectory.cc:213-309)
 *   mjpc_b200_model_derivatives <- ModelDerivatives::Compute            mjpc/planners/model_derivatives.cc:45-165
 *   mjpc_b200_cost_derivatives  <- CostDerivatives::Compute             mjpc/planners/cost_derivatives.cc:112-230
 *   mjpc_b200_backward_pass     <- RiccatiStep recursion                mjpc/planners/ilqg/planner.cc:429-520,
 *                                                                       mjpc/planners/ilqg/backward_pass.cc:65-250
 *   mjpc_b200_*_batched         <- the calls above for B independent problems in one launch (rollout_spline,
 *                                  rollout_feedback, model_derivatives, cost_derivatives, backward_pass)
 *   mjpc_b200_gradient_batched  <- Gradient::Compute with its derivatives   mjpc/planners/gradient/gradient.cc:76-107
 *                                  (the two derivative sweeps, then the gradient recursion, all on the device)
 *   mjpc_b200_set_task          <- residual_fn_ snapshot per PlanIteration  mjpc/agent.cc:316-319, task.cc:112-128
 *   mjpc_b200_fetch_trajectory  <- fills a mjpc::Trajectory             mjpc/trajectory.h:74-86
 *   create / destroy            <- Planner::Initialize/Allocate + ResizeMjData  mjpc/planners/planner.cc:23-33;
 *                                  precedent for a C surface: mjpc/interface.h:44-49
 *
 * Conventions: all pointers are HOST memory owned by the caller; the handle owns every device buffer and
 * stream.  All calls come from the single plan thread (as Agent::PlanIteration does today).  Functions return
 * 0 on success or a negative mjpc_b200_error; they never throw or abort.  Per-candidate divergence is
 * reported through failure[i] (= Trajectory::failure) with returns[i] = 1e6 (mjpc/trajectory.cc:29,169-173).
 * Arithmetic on the device is fp32; time is carried relative to the rollout start and returned as double.
 */
#ifndef MJPC_B200_H_
#define MJPC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mjpc_b200 mjpc_b200_t;

typedef enum {
  MJPC_B200_OK = 0,
  MJPC_B200_ERR_BAD_ARGUMENT = -1,
  MJPC_B200_ERR_BAD_BLOB = -2,
  MJPC_B200_ERR_CAPACITY = -3,   /* N / H above what create() reserved, or model too large for shared memory */
  MJPC_B200_ERR_CUDA = -4,       /* no device, launch or copy failure: the engine has NO CPU fallback */
  MJPC_B200_ERR_UNSUPPORTED = -5 /* model feature outside the implemented subset */
} mjpc_b200_error;

/* Flat model + task description (field names = mjModel's); written by mujoco_mpc_b200/blob.py, or by a
 * maintainer from an mjModel* (INTEGRATION.md).  The engine copies what it needs during create(). */
typedef struct {
  const void* data;
  size_t nbytes;
} mjpc_model_blob;

/* Live task snapshot (BaseResidualFn::Update, mjpc/task.cc:112-123). NULL members keep the current value. */
typedef struct {
  const double* weight;      /* [num_term]                         Task::weight        */
  const double* parameters;  /* [num_parameters]                   Task::parameters    */
  const double* task_state;  /* residual-specific state block (e.g. quadruped mode/gait/phase), see DESIGN.md */
  double risk;               /* Task::risk                                              */
} mjpc_task_desc;

typedef struct {
  int nq, nv, nu, na, nmocap, nuserdata;
  int dim_state;        /* nq + nv + na   */
  int dim_dstate;       /* 2*nv + na      */
  int num_residual, num_term, num_trace, num_parameters, task_state_size;
  int max_candidates, max_horizon;
  int device;           /* CUDA device ordinal in use */
  int smem_bytes_per_warp;
} mjpc_b200_info;

/* interp: 0 zero-order, 1 linear, 2 cubic (mjpc/spline/spline.h SplineInterpolation) */
/* feedback mode: 0/1/2 time-indexed with that interpolation (iLQGPolicy::representation), 3 step-indexed */

const char* mjpc_b200_version(void);
const char* mjpc_b200_last_error(void);

int mjpc_b200_create(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                     mjpc_b200_t** out);
void mjpc_b200_destroy(mjpc_b200_t* h);
int mjpc_b200_get_info(const mjpc_b200_t* h, mjpc_b200_info* info);

int mjpc_b200_set_task(mjpc_b200_t* h, const mjpc_task_desc* task);

/* Planning-model overrides of Agent::PlanIteration (agent.cc:288-289): opt.timestep = agent_timestep, opt.integrator =
 * agent_integrator, for the following calls of this handle.  Only the Euler integrator (0) is implemented: any other value
 * returns MJPC_B200_ERR_UNSUPPORTED. */
int mjpc_b200_set_options(mjpc_b200_t* h, double timestep, int integrator);

/* MakeDifferentiable (mjpc/utilities.cc:60-75) for the following calls of this handle: on != 0 zeroes solimp[0] of every
 * joint and geom in the model the kernels read, 0 restores the model's values - what Agent::PlanIteration does around
 * OptimizePolicy for gradient-based planners (agent.cc:296-309,346-356; default on for iLQG / iLQS / Gradient,
 * agent.cc:158-164).  The C++ iLQG planner switches it on unless iLQGSettings::differentiable is cleared. */
int mjpc_b200_set_differentiable(mjpc_b200_t* h, int on);

/* N candidate splines -> N rollouts of H steps. knots [N][P][nu]; knot_times [P] (absolute seconds).
 * candidate_offset: global index of this handle's first candidate (multi-GPU sharding; only used for bookkeeping).
 * returns [N], failure [N]; order [N] = candidate indices sorted by return (ties: lower index first), may be NULL. */
int mjpc_b200_rollout_spline(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                             const float* userdata, const float* knots, const double* knot_times, int interp,
                             int P, int N, int H, float* returns, uint8_t* failure, int* order);

/* B independent planning problems of N candidates each in ONE rollout launch (mjpc_b200_rollout_spline is the case
 * B = 1).  Every problem has its own start state, absolute start time, mocap, task snapshot and knots; N, P, interp and
 * H are common.  Candidate i of problem b has the flat index b*N + i.
 *   states [B][dim_state], times [B] (absolute), mocaps [B][7 nmocap], knots [B][N][P][nu], knot_times [B][P] (absolute)
 *   weights [B][num_term], parameters [B][num_parameters], task_states [B][task_state_size]: each may be NULL, which
 *     stands for the handle's set_task value in every problem; the time-like task-state entries are rebased by times[b].
 *     Risk is the handle's (Task::risk).
 *   returns [B][N], failure [B][N]; order [B][N] (may be NULL): order[b] ranks problem b's candidates by return with
 *     indices local to the problem (0..N-1, ties: lower index first).
 * B*N must not exceed max_candidates (MJPC_B200_ERR_CAPACITY); B, N, H >= 1, H <= max_horizon and P <= 64, otherwise an
 * error is returned and the handle stays usable.  After a batched launch, fetch_trajectory, fetch_all and fetch_stats
 * take the flat index, last_kernel_ms / last_kernel_static describe the one launch, and NoisyRollout force noise
 * (set_xfrc_noise) draws with the flat index as its candidate counter. */
int mjpc_b200_rollout_spline_batched(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                                     const double* weights, const double* parameters, const double* task_states,
                                     const float* knots, const double* knot_times, int interp, int P, int N, int H,
                                     float* returns, uint8_t* failure, int* order);

/* NoisyRollout (mjpc/trajectory.cc:100-210, used by the Robust planner): the following rollouts of this handle add
 * Ornstein-Uhlenbeck noise to xfrc_applied of every body (stationary std xfrc_std, correlation time xfrc_rate
 * seconds), drawn from Philox4x32-10 with key (seed, 1) and counter (step, candidate, element, 'XFRC') - the
 * reference's absl::BitGen cannot be seeded.  xfrc_std = 0 switches the noise off (the default).  Clears the
 * per-problem keys of set_xfrc_noise_batched. */
int mjpc_b200_set_xfrc_noise(mjpc_b200_t* h, double xfrc_std, double xfrc_rate, uint32_t seed);

/* The same noise with one key per problem: the following rollout launches must hold exactly B problems (a launch of
 * another B returns MJPC_B200_ERR_BAD_ARGUMENT and leaves the handle usable; a single-problem launch is B = 1), and
 * problem b draws with key seeds[b] and its problem-local candidate index as the counter - bitwise what a launch of
 * problem b alone draws after set_xfrc_noise(seeds[b]).  seeds [B].  mjpc_b200_rollout_spline_sharded refuses
 * per-problem keys (MJPC_B200_ERR_UNSUPPORTED); set_xfrc_noise clears them. */
int mjpc_b200_set_xfrc_noise_batched(mjpc_b200_t* h, double xfrc_std, double xfrc_rate, int B, const uint32_t* seeds);

/* Per-problem model variants: problem b of the following batched launches runs on models[b] instead of the handle's
 * model, bitwise what a handle created from models[b] computes.  Each variant is a full blob (its own MJCF through
 * mjcf.py, or its own mjModel after mj_setConst); derived constants are taken from it, never recomputed.  Every
 * variant must equal the handle's model, as created, in: every integer header field (sizes, option flags, task
 * dimensions), the whole int section of the pack (so a frictionloss set to 0, a contype change or an extra geom are
 * refused), timestep, impratio, tolerance, ls_tolerance, gravity and task_risk, the task arrays (task_weight,
 * task_norm_parameter, task_parameters, task_state), actuator_ctrlrange and the measurement-sensor table; and it must
 * pass create's own refusals.  The other float arrays (body, joint, dof, geom, site, actuator and tendon parameters,
 * qpos0, qpos_spring, key_qpos), meaninertia and the keyframe table may differ.  A mismatch is
 * MJPC_B200_ERR_BAD_ARGUMENT (last_error names the variant and the first field that differs) and leaves the handle as
 * it was.  set_options, set_differentiable and set_task still apply to the whole handle (set_task to every variant).
 * count = 0 (or models NULL) clears the variants.  While variants are set:
 *   rollout_*_batched, model_derivatives_batched, gradient_batched and a filter bank's update must hold exactly count
 *     problems (MJPC_B200_ERR_BAD_ARGUMENT otherwise, before anything is staged) - or the B of select_model_variants;
 *   the single-problem calls, rollout_spline_sharded, step_debug*, step_batch and step_sensors return
 *     MJPC_B200_ERR_UNSUPPORTED naming the call;
 *   cost_derivatives_batched and backward_pass_batched read only what variants share, and take any B. */
int mjpc_b200_set_model_variants(mjpc_b200_t* h, const mjpc_model_blob* models, int count);
/* With variants set: the following launches hold B problems, problem j running on variant index[j] in [0, count)
 * (index NULL: problem j on variant j, B = count).  For planners that plan a subset of their problems in one launch.
 * Without variants there is nothing to select: returns 0 and changes nothing. */
int mjpc_b200_select_model_variants(mjpc_b200_t* h, const int* index, int B);

/* A model ensemble: every spline launch of this handle (rollout_spline, rollout_spline_batched, upload_spline_inputs +
 * launch_resident) scores each candidate on K member models.  Candidate i of problem b is rolled out once per member,
 * and its return is the mean of its `worst` largest member returns (worst = K: the expected return; worst = 1: the
 * worst case): the member returns sorted in descending order (ties to the lower member), the first `worst` summed left
 * to right in double, divided once by worst and rounded to float.  If any member fails, the candidate fails and its
 * return is exactly 1e6.  returns, failure and order of the launch describe these scores ([B][N], order ranks them), and
 * fetch_trajectory / fetch_all (flat index b*N + i) return member 0's trajectories; fetch_stats returns the rows of
 * every launched trajectory [B][K][N].
 *   Members follow the rule of set_model_variants, with its error naming the member and the first field that differs;
 *   set_task rewrites every member's task.  1 <= K <= 32 and 1 <= worst <= K, else MJPC_B200_ERR_BAD_ARGUMENT; the
 *   handle is unchanged on any refusal.  K = 0 (or models NULL) clears the ensemble.
 *   The launch holds B*K*N trajectories (member k of problem b is launch problem b*K + k); B*N is still bounded by
 *   max_candidates: the call grows the per-trajectory device buffers to K x max_candidates (never shrinks them;
 *   MJPC_B200_ERR_CUDA, handle unchanged, if that fails).
 *   While an ensemble is set, set_model_variants (count > 0), rollout_feedback*, model_derivatives*, gradient_batched,
 *   rollout_spline_sharded, step_debug*, step_batch, step_sensors, the plant calls, a filter bank's update and a spline
 *   launch with force noise (set_xfrc_noise*) return MJPC_B200_ERR_UNSUPPORTED naming the call; set_model_ensemble
 *   while variants are set likewise. */
int mjpc_b200_set_model_ensemble(mjpc_b200_t* h, const mjpc_model_blob* models, int K, int worst);
/* The member returns [B][K][N] and failure flags [B][K][N] of the last launch, an ensemble launch (either may be
 * NULL); MJPC_B200_ERR_BAD_ARGUMENT after any other launch. */
int mjpc_b200_fetch_ensemble(mjpc_b200_t* h, float* member_returns, uint8_t* member_failure);
/* Candidate (flat b*N + i) of the last launch as member `member` rolled it out (fetch_trajectory's arrays);
 * fetch_trajectory is member 0.  After a launch without an ensemble only member 0 exists. */
int mjpc_b200_fetch_trajectory_member(mjpc_b200_t* h, int candidate, int member, float* states, float* actions,
                                      double* times, float* residual, float* costs, float* trace);
/* The score of one candidate from its K member returns [K] and failure flags [K] on the host, bit for bit what the
 * device computes (for tests).  Nothing is written unless 1 <= K <= 32 and 1 <= worst <= K. */
void mjpc_b200_host_ensemble_score(const float* member_returns, const uint8_t* member_failure, int K, int worst,
                                   float* score, uint8_t* failure);
/* Test hooks: the device's candidate ranking and ensemble score on caller data, with the launch shapes of a rollout
 * launch, on the handle's stream; the last launch's returns, order and trajectories are untouched.
 * debug_rank: returns [nseg][N] -> order [nseg][N], each segment's indices by ascending return (ties to the lower
 *   index, NaN last); order is filled with -1 before the launch, so a slot the ranking misses reads -1.
 * debug_ensemble_score: member_returns / member_failure [B][K][N] -> returns / failure [B][N], the score of
 *   set_model_ensemble with `worst`.
 * nseg, N, B < 1, K outside [1, 32], worst outside [1, K] or a NULL pointer: MJPC_B200_ERR_BAD_ARGUMENT, nothing
 * launched and the handle usable. */
int mjpc_b200_debug_rank(mjpc_b200_t* h, const float* returns, int nseg, int N, int* order);
int mjpc_b200_debug_ensemble_score(mjpc_b200_t* h, const float* member_returns, const uint8_t* member_failure, int B,
                                   int K, int N, int worst, float* returns, uint8_t* failure);

/* An initial-state ensemble: rollout_spline_batched with every candidate scored over K initial states drawn from each
 * problem's state covariance, so that a candidate that does well only from the exact mean state does not win when the
 * state estimate is uncertain.  Arguments as rollout_spline_batched, plus:
 *   covariances [B][n][n] (double, n = 2 nv: the filters' tangent space, positions then velocities), K members per
 *   problem, worst (the score is the mean of the `worst` largest member returns: set_model_ensemble's rule, with its
 *   failure rule), and seed / iteration of the draws.
 * Member 0 of problem b starts from states[b] itself; member k >= 1 from states[b] (+) L_b z_{b,k}, where L_b is the
 * lower Cholesky factor of (P_b + P_b') / 2 and (+) is mj_integratePos for the position half (free and ball joints:
 * the quaternion times exp(w / 2), normalised; a rotation of exactly zero keeps the quaternion bit for bit) and addition
 * for the velocity half (a zero entry keeps the coordinate bit for bit).  z is a standard normal: Philox4x32-10 with key
 * (seed + b, 3) and counter (iteration, k, element, 'BELF'), Box-Muller in double on the first two words; key word 3 is
 * used by no candidate-noise or plant-noise draw.  The factor, L z and (+) are computed in double on the device (one
 * CTA per problem), and the member states are written as float straight into the launch's state rows.  A pivot of
 * exactly 0 whose column below is all zero gives a zero column, so a zero covariance gives K copies of the mean and
 * scores equal to the plain launch's returns.
 * The launch holds B*K*N trajectories, member k of problem b as launch problem b*K + k (the model ensemble's layout):
 * returns / failure / order are the scores [B][N], fetch_ensemble gives the member returns [B][K][N],
 * fetch_trajectory_member any member's trajectory and fetch_trajectory / fetch_all member 0's.  With model variants
 * set (B must then be their count or select_model_variants' B), every member row of problem b runs on problem b's
 * variant.  The launch does not become the resident one (launch_resident refuses until the next upload).
 * Refusals, each before anything is staged and with the handle unchanged: K outside [1, 32], worst outside [1, K], a
 * non-finite covariance entry (last_error names the problem) or bad sizes: MJPC_B200_ERR_BAD_ARGUMENT; B*N above
 * max_candidates (or H, P above capacity): MJPC_B200_ERR_CAPACITY; a model ensemble or force noise (set_xfrc_noise*)
 * set on the handle: MJPC_B200_ERR_UNSUPPORTED naming the call.  As set_model_ensemble does, the call grows the
 * per-trajectory device buffers to K x max_candidates trajectories (never shrinks them; MJPC_B200_ERR_CUDA if that
 * fails), so the launch holds up to K x max_candidates trajectories; it also allocates its own tables once.  A
 * covariance whose factorisation fails (a pivot < 0,
 * a zero pivot with a non-zero column below, or a non-finite pivot) returns MJPC_B200_ERR_BAD_ARGUMENT with last_error
 * naming the problem, and no rollout is launched and no returns are written; the handle stays usable. */
int mjpc_b200_rollout_spline_belief_batched(mjpc_b200_t* h, int B, int K, int worst, uint32_t seed, uint32_t iteration,
                                            const float* states, const double* covariances, const double* times,
                                            const float* mocaps, const double* weights, const double* parameters,
                                            const double* task_states, const float* knots, const double* knot_times,
                                            int interp, int P, int N, int H, float* returns, uint8_t* failure,
                                            int* order);
/* Member `member` (0..31) of problem `problem` of a belief launch on the host, in double (for tests): out [nq + nv] is
 * state (+) L z with the launch's factor, draw and (+), summed in the same order; the device's member states are this
 * rounded to float, up to fp64 contractions.  MJPC_B200_ERR_BAD_ARGUMENT for a non-finite covariance or a failed
 * factorisation (out then holds state), MJPC_B200_ERR_BAD_BLOB for a bad blob. */
int mjpc_b200_host_state_member(const mjpc_model_blob* model, const double* state, const double* covariance,
                                uint32_t seed, uint32_t iteration, int problem, int member, double* out);

/* K line-search rollouts of the iLQG policy. u_nom [H][nu], x_nom [H][dim_state], t_nom [H] (absolute),
 * gains [H][nu][dim_dstate], du [H][nu] (may be NULL), step_sizes [K]. */
int mjpc_b200_rollout_feedback(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                               const float* userdata, const float* u_nom, const float* x_nom, const double* t_nom,
                               const float* gains, const float* du, const float* step_sizes, int mode, int K, int H,
                               float* returns, uint8_t* failure, int* order);

/* B independent problems of K line-search rollouts each in ONE launch (mjpc_b200_rollout_feedback is the case B = 1).
 * Conventions as mjpc_b200_rollout_spline_batched: states [B][dim_state], times [B] (absolute), mocaps [B][7 nmocap],
 * weights / parameters / task_states [B][..] or NULL for the handle's set_task values; per problem u_nom [B][H][nu],
 * x_nom [B][H][dim_state], t_nom [B][H] (absolute; rebased to times[b]), gains [B][H][nu][dim_dstate], du [B][H][nu]
 * (may be NULL), step_sizes [B][K]; mode, K and H are common.  returns / failure / order [B][K], order local to the
 * problem.  B*K > max_candidates or H > max_horizon: MJPC_B200_ERR_CAPACITY.  fetch_* then take the flat index b*K + i. */
int mjpc_b200_rollout_feedback_batched(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                                       const double* weights, const double* parameters, const double* task_states,
                                       const float* u_nom, const float* x_nom, const double* t_nom, const float* gains,
                                       const float* du, const float* step_sizes, int mode, int K, int H, float* returns,
                                       uint8_t* failure, int* order);

/* Copy candidate i of the last rollout into Trajectory-shaped host arrays (any pointer may be NULL):
 * states [H][dim_state], actions [H][nu], times [H], residual [H][num_residual], costs [H], trace [H][3*num_trace] */
int mjpc_b200_fetch_trajectory(mjpc_b200_t* h, int candidate, float* states, float* actions, double* times,
                               float* residual, float* costs, float* trace);
/* Bulk variant: every candidate of the last rollout ([N] leading dimension). */
int mjpc_b200_fetch_all(mjpc_b200_t* h, float* states, float* actions, double* times, float* residual,
                        float* costs, float* trace);

/* Finite-difference transition / residual Jacobians along a trajectory (ModelDerivatives::Compute,
 * model_derivatives.cc:45-165).  x [H][dim_state], u [H][nu], t [H]; A [H][n][n], B [H][n][nu], C [H][nr][n],
 * D [H][nr][nu], n = dim_dstate, nr = num_residual (the rows CostDerivatives reads).
 *   skip  derivative_skip: only every (skip+1)-th step plus H-2 and H-1 is differentiated, the rest is linearly
 *         interpolated between its evaluated neighbours (model_derivatives.cc:56-72,109-164); 0 = every step
 *   tol   finite-difference step (ilqg/settings.h:23, reference default 1e-6 in double; fp32 wants ~1e-3)
 *   mode  0 one-sided, 1 centred (ilqg/settings.h:24 fd_mode -> mjd_transitionFD flg_centered)
 * Row H-1 of A, B, D is left zero (model_derivatives.cc:89-93). */
int mjpc_b200_model_derivatives(mjpc_b200_t* h, const float* x, const float* u, const double* t,
                                const float* mocap, int H, int skip, float tol, int mode, float* A, float* B,
                                float* C, float* D);

/* Gauss-Newton cost derivatives. residual [H][nr], C, D as above -> cx [H][n], cu [H][nu], cxx [H][n][n],
 * cuu [H][nu][nu], cxu [H][n][nu]. */
int mjpc_b200_cost_derivatives(mjpc_b200_t* h, const float* residual, const float* C, const float* D, int H,
                               float* cx, float* cu, float* cxx, float* cuu, float* cxu);

/* One Riccati sweep at fixed regularisation. status_out: 1 success, 0 failure (caller scales mu and retries).
 * reg_type 0 control, 1 state-control, 2 value, 3 none; limits 1 = box-QP within ctrlrange - action.
 * Outputs: K [H][nu][n], du [H][nu], dV[2], and (optional, may be NULL) Vx [H][n], Vxx [H][n][n]. */
int mjpc_b200_backward_pass(mjpc_b200_t* h, const float* A, const float* B, const float* cx, const float* cu,
                            const float* cxx, const float* cxu, const float* cuu, const float* actions, int H,
                            float mu, int reg_type, int limits, float* K, float* du, float* dV, float* Vx,
                            float* Vxx, int* status_out);

/* The three iLQG sweeps for B independent problems in one launch each (the single-problem calls above are B = 1).
 * Every per-problem array gains a leading [B] dimension; H, skip, tol, mode, reg_type and limits are common, the risk
 * is the handle's.  weights [B][num_term], parameters [B][num_parameters], task_states [B][task_state_size] may each
 * be NULL for the handle's set_task values; problem b's time-like task state is rebased to its own t[b][0].
 * backward_pass_batched: mu [B], dV [B][2], status [B] (1 success, 0 failure; a failure ends only that problem's
 * sweep); Vx / Vxx may be NULL.  B < 1 or a NULL required pointer: MJPC_B200_ERR_BAD_ARGUMENT; H > max_horizon:
 * MJPC_B200_ERR_CAPACITY.  The handle's iLQG buffers grow on demand to the largest B seen. */
int mjpc_b200_model_derivatives_batched(mjpc_b200_t* h, int B, const float* x, const float* u, const double* t,
                                        const float* mocaps, const double* weights, const double* parameters,
                                        const double* task_states, int H, int skip, float tol, int mode, float* A,
                                        float* B_, float* C, float* D);
int mjpc_b200_cost_derivatives_batched(mjpc_b200_t* h, int B, const double* weights, const float* residual, const float* C,
                                       const float* D, int H, float* cx, float* cu, float* cxx, float* cuu, float* cxu);
int mjpc_b200_backward_pass_batched(mjpc_b200_t* h, int B, const float* A, const float* B_, const float* cx,
                                    const float* cu, const float* cxx, const float* cxu, const float* cuu,
                                    const float* actions, int H, const float* mu, int reg_type, int limits, float* K,
                                    float* du, float* dV, float* Vx, float* Vxx, int* status);
/* Gradient::Compute (gradient.cc:76-107) for B problems: the FD derivative sweep of mjpc_b200_model_derivatives_batched
 * and the cost derivatives of mjpc_b200_cost_derivatives_batched on the same inputs, then the gradient recursion, all on
 * the device; A, B, C, D and the cost derivatives never leave it.  Inputs as model_derivatives_batched, plus
 * residual [B][H][nr].  k [B][H][nu] (row H-1 repeats row H-2), dV0 [B], both double, bitwise what
 * mjpc_b200_host_gradient_sweep computes from the A, B, cx and cu the two batched calls return.  B < 1, H < 2, a NULL
 * required pointer, a bad skip / mode / tol or missing mocaps: MJPC_B200_ERR_BAD_ARGUMENT; H > max_horizon:
 * MJPC_B200_ERR_CAPACITY.  last_kernel_ms spans the call's kernels (the residual upload between them included). */
int mjpc_b200_gradient_batched(mjpc_b200_t* h, int B, const float* x, const float* u, const double* t,
                               const float* mocaps, const double* weights, const double* parameters,
                               const double* task_states, const float* residual, int H, int skip, float tol, int mode,
                               double* k, double* dV0);

/* Debug / parity hook: one forward-dynamics evaluation + Euler step for a single state through the same
 * device code the rollout kernel runs. qacc[nv], residual[nr], next_qpos[nq], next_qvel[nv], counts[4] =
 * {ncon, nefc, solver iterations, warning}. */
int mjpc_b200_step_debug(mjpc_b200_t* h, const float* qpos, const float* qvel, const float* ctrl,
                         const float* mocap, double time, const float* warmstart, float* qacc, float* residual,
                         float* next_qpos, float* next_qvel, float* qM, float* efc_force, int* counts);

/* The geometric contacts of the last mjpc_b200_step_debug call (tendon-limit pseudo-contacts excluded), in the
 * order the narrow phase emitted them (pair order): contact [n][8] = {dist, pos[3], normal (frame row 0)[3], dim}
 * for the first min(ncon, capacity) of them, *ncon = their number.  Debug / parity hook only. */
int mjpc_b200_step_debug_contacts(mjpc_b200_t* h, int capacity, float* contact, int* ncon);

/* Batched variant for teacher-forced per-step parity at full planner sizes: B independent (qpos, qvel, ctrl, warm start,
 * absolute time) tuples are each advanced by one mj_step (mjpc/trajectory.cc:158) through the same kernel instance the
 * rollout uses.  The task state is rebased to time0 as for a rollout starting there.  warmstart may be NULL (zeros).
 * Outputs (any may be NULL): qacc [B][nv], next_qpos [B][nq], next_qvel [B][nv], residual [B][nr], cost [B],
 * counts [B][4] = {ncon, nefc, solver iterations, warning}. */
int mjpc_b200_step_batch(mjpc_b200_t* h, int B, const float* qpos, const float* qvel, const float* ctrl,
                         const float* warmstart, const float* mocap, double time0, const double* times, float* qacc,
                         float* next_qpos, float* next_qvel, float* residual, float* cost, int* counts);

/* The sigma-point step of a state estimator: B states [B][dim_state], all from the same ctrl [nu], mocap and absolute
 * time, are each advanced by one mj_step through the kernel instance mjpc_b200_step_batch runs, and the measurement
 * sensors [sensor_start, sensor_start + nsensor) of each PRE-step state are evaluated after the constraint solve
 * (positions, velocities and touch forces of the state the step starts from, as mj_step's sensor stage sees them).
 * Evaluated: jointpos / jointvel of slide and hinge joints; the frame sensors framepos, framequat, framexaxis /
 * frameyaxis / framezaxis, framelinvel / frameangvel and framelinacc / frameangacc (world frame, no reference frame) of a
 * site, body (inertial frame), xbody or geom; subtreecom / subtreelinvel / subtreeangmom of a body; touch with a sphere
 * site zone; accelerometer / velocimeter / gyro of a site (in the site frame); ballquat / ballangvel of a ball joint;
 * jointactuatorfrc of a slide or hinge joint; actuatorpos / actuatorvel (joint or fixed-tendon transmission) and
 * actuatorfrc; tendonpos / tendonvel of a fixed tendon; magnetometer of a site (site_xmat' opt.magnetic, the blob's
 * opt_magnetic or MuJoCo's default 0 -0.5 0); rangefinder of a site (mj_ray along the site's z axis over the geoms not
 * of the site's body whose alpha, the blob's geom_alpha, is not 0: the least distance, or -1; refused when such a geom
 * is a height field or another type rays are not cast against).  Not evaluated (MJPC_B200_ERR_UNSUPPORTED, the last
 * error naming the sensor): user, force, torque, camprojection, limit and constraint force,
 * energy and clock sensors, touch with another zone, and any sensor with a cutoff.  The same set and refusals hold for
 * plant_init's sensor range and for the estimators' (unscented_create, kalman_create, batch_estimator_create).
 * warmstart [B][nv] may be NULL (zeros); mocap [7 nmocap] is required when
 * nmocap > 0.  Outputs: next_states [B][dim_state], sensordata [B][dim] (dim = the range's total sensor dimension),
 * and, when not NULL, qacc [B][nv] and counts [B][4] = {ncon, nefc, solver iterations, warning}, all equal to what
 * mjpc_b200_step_batch returns for the same inputs.  last_kernel_ms times the launch.  A range outside the model's
 * sensors: MJPC_B200_ERR_BAD_ARGUMENT; a sensor in it that is not evaluated: MJPC_B200_ERR_UNSUPPORTED;
 * B > max_candidates: MJPC_B200_ERR_CAPACITY.  Device and pinned buffers are the handle's (no allocation per call
 * once the largest B has been seen). */
int mjpc_b200_step_sensors(mjpc_b200_t* h, int B, const float* states, const float* ctrl, const float* warmstart,
                           const float* mocap, double time, int sensor_start, int nsensor, float* next_states,
                           float* sensordata, float* qacc, int* counts);

/* ---- Closed-loop plants: num_plants plants on an engine handle, each an mjData-like state (qpos, qvel, warm start,
 * time) kept in device memory with its running cost sum, step count and warning count, its own mocap and task rows
 * (weight, parameters, task state in absolute time) and, with model variants set, its own model: plant b steps on
 * variant b, bitwise what a handle created from that variant steps.  mjpc_b200_plant_step advances every running plant
 * by one mj_step in one launch, through the device functions and the kernel instance mjpc_b200_step_batch runs: plant
 * b's step equals step_batch's with time0 = the plant's time, its task rows and its warm start.  The ctrl is applied
 * as step_batch applies it.  The warm start carries from step to step (qacc_warmstart across mj_step calls).
 *
 * A step is committed only when the next qpos, qvel and qacc are finite: the state, the warm start (= qacc), time +=
 * timestep (double), cost sum += the step's cost (the pre-step residual's CostValue), steps += 1, warnings += the
 * step's warning (contact or constraint buffer full).  Otherwise the plant's status becomes MJPC_B200_PLANT_DIVERGED
 * and nothing is committed.  Unlike MuJoCo, which would call mj_resetData, a plant is never reset silently: it is
 * skipped by later steps until plant_reset.  A plant is MJPC_B200_PLANT_IDLE from plant_init until its first reset.
 *
 * Every call returns MJPC_B200_ERR_BAD_ARGUMENT for a NULL handle, a handle without plants (plant_init) or a plant
 * index outside [0, num_plants), and leaves the bank unchanged on any refusal.  Disturbances (control noise, body-force
 * noise, a held wrench) are set per plant below plant_get. */
enum { MJPC_B200_PLANT_RUNNING = 0, MJPC_B200_PLANT_DIVERGED = 1, MJPC_B200_PLANT_IDLE = 2 };

/* The handle's plants (replacing any earlier ones), every plant idle, with the handle's set_task values as task rows.
 * nsensor = 0: no sensors; else plant_step returns the measurement sensors [sensor_start, sensor_start + nsensor) of
 * each pre-step state (the range rules of mjpc_b200_step_sensors: BAD_ARGUMENT outside the model's sensors,
 * UNSUPPORTED for a sensor the engine does not evaluate).  num_plants above max_candidates: MJPC_B200_ERR_CAPACITY. */
int mjpc_b200_plant_init(mjpc_b200_t* h, int num_plants, int sensor_start, int nsensor);
/* Start an episode of plant `plant` (mj_resetData + setting the state): qpos [nq], qvel [nv], time, mocap [7 nmocap]
 * (required when nmocap > 0).  Warm start, cost sum, steps and warnings become 0 and the plant runs. */
int mjpc_b200_plant_reset(mjpc_b200_t* h, int plant, const float* qpos, const float* qvel, double time,
                          const float* mocap);
/* What a Task::Transition writes into mjData between steps; NULL keeps the current value.  Warm start, time, sums and
 * status are kept. */
int mjpc_b200_plant_set(mjpc_b200_t* h, int plant, const float* qpos, const float* qvel, const float* mocap);
/* The plant's task rows for the following steps (task state in absolute time); NULL keeps the current row. */
int mjpc_b200_plant_set_task(mjpc_b200_t* h, int plant, const double* weight, const double* parameters,
                             const double* task_state);
/* One step of every running plant from ctrl [num_plants][nu].  Outputs (any may be NULL), per plant after the step:
 * state [num_plants][nq+nv], time [num_plants], cost [num_plants] (the step's cost; 0 for a plant that did not step),
 * sensordata [num_plants][dim] (the pre-step sensors of plant_init's range; zeros for a plant that did not step) and
 * status [num_plants].  With model variants set, their count (or select_model_variants' B) must be num_plants
 * (MJPC_B200_ERR_BAD_ARGUMENT otherwise).  last_kernel_ms times the launch. */
int mjpc_b200_plant_step(mjpc_b200_t* h, const float* ctrl, float* state_out, double* time_out, float* cost_out,
                         float* sensordata_out, int* status_out);
/* Plant `plant`'s fields; any pointer may be NULL: state [nq+nv], warmstart [nv], time, cost_sum, steps, warnings,
 * status. */
int mjpc_b200_plant_get(mjpc_b200_t* h, int plant, float* state, float* warmstart, double* time, double* cost_sum,
                        int* steps, int* warnings, int* status);

/* Disturbances (the reference app's control noise and force perturbations, app.cc:95-101, 291-304, 323-352).  Before
 * each step of a running plant:
 *   control noise  n <- r n + s z per actuator, r = exp(-timestep / ctrl_rate), s = ctrl_std sqrt(1 - r^2), added to the
 *                  commanded ctrl; actuation clamps the sum to ctrlrange as it clamps any ctrl
 *   force noise    the same recursion (xfrc_std, xfrc_rate) over the 6 nbody entries of xfrc_applied, as the Robust
 *                  planner's rollouts draw it
 *   xfrc_applied   = the held wrench + the force noise: per body force 3 then torque 3, world frame, at the body's
 *                  centre of mass
 * z is a standard normal: Philox4x32-10 with key (seed, 2) and counter (the plant's committed step count, 0, element,
 * 'CTRL' or 'XFRC'), Box-Muller on the first two words.  A plant's noise depends on its seed and its own history only.
 * The OU states advance only with a committed step.  plant_reset zeroes them (with the step count: the episode replays
 * its seed's sequence) and keeps the settings and the held wrench; plant_init starts every plant undisturbed.  A plant
 * without disturbances steps bitwise as before.  Every call below is refused with MJPC_B200_ERR_UNSUPPORTED while a
 * model ensemble is set. */
/* Plant `plant`'s noise (std 0: off) and seed; zeroes its OU states.  BAD_ARGUMENT: a negative or non-finite std, or a
 * rate <= 0 or non-finite where its std is > 0. */
int mjpc_b200_plant_set_disturbance(mjpc_b200_t* h, int plant, double ctrl_std, double ctrl_rate, double xfrc_std,
                                    double xfrc_rate, uint32_t seed);
/* The wrench xfrc [nbody][6] held on plant `plant` until changed (ApplyForcePerturbations headless); NULL clears it.
 * BAD_ARGUMENT: a non-finite value. */
int mjpc_b200_plant_set_xfrc(mjpc_b200_t* h, int plant, const float* xfrc);
/* Measurement noise of plant `plant`: std [nsensordata] (one entry per element of plant_init's sensor range; NULL
 * clears it).  Each committed step of the running plant returns sensordata[e] + std[e] z, z a standard normal from
 * Philox4x32-10 with key (seed, 2) and counter (the committed step count before the step, 0, e, 'SENS'): it depends on
 * the plant's seed (set_disturbance) and its own history only, never on its index or the other plants, never repeats
 * the control or force noise, and plant_reset replays it.  Quaternion sensors (framequat, ballquat) get the noise
 * added to each component, without renormalisation.  Only the returned measurement changes: the plant's state, cost
 * and warm start are bitwise what they are without noise, elements whose std is 0 are bitwise unchanged, and a plant
 * whose stds are all 0 steps exactly as one without the call.  BAD_ARGUMENT: a negative or non-finite entry (the plant
 * is then unchanged). */
int mjpc_b200_plant_set_sensor_noise(mjpc_b200_t* h, int plant, const float* std);
/* Plant `plant`'s OU states; either pointer may be NULL: ctrl_noise [nu], xfrc_noise [nbody][6]. */
int mjpc_b200_plant_get_disturbance(mjpc_b200_t* h, int plant, float* ctrl_noise, float* xfrc_noise);
/* The ctrl every plant applied in the last plant_step, [num_plants][nu]: commanded + control noise (the commanded ctrl,
 * bit for bit, without control noise; the commanded ctrl of a plant that was not running; zeros before any step). */
int mjpc_b200_plant_last_ctrl(mjpc_b200_t* h, float* ctrl_out);

/* ---- State estimators (csrc/host/estimator.h, the reference's Estimator base mjpc/estimators/estimator.h): a single
 * filter is the batched estimators' bank of one filter below, on an engine handle it owns, with the same device
 * arithmetic.  Each kind has its own create (its settings); every other call is one of the generic
 * mjpc_b200_estimator_* below, which take a filter of any kind and return MJPC_B200_ERR_BAD_ARGUMENT for a NULL one
 * (last_error: "").  create measures the sensors [sensor_start, sensor_start + nsensor) of the blob; a range outside
 * the model's sensors returns MJPC_B200_ERR_BAD_ARGUMENT and a sensor the engine does not evaluate
 * MJPC_B200_ERR_UNSUPPORTED.  Settings are explicit (timestep = estimator_timestep or opt.timestep, noise
 * scales 1e-4 by default).
 *   reset      state NULL -> the model's first keyframe, else qpos0 and zero qvel; covariance = covariance_scale I,
 *              diagonal process / sensor noise
 *   set_noise  process [ndstate], sensor [nsensordata] (NULL keeps one)
 *   set        state, covariance [ndstate^2] (NULL keeps one) and time
 *   update     one filter update from ctrl [nu], the measured sensor slice [nsensordata] and mocap [7 nmocap] or NULL
 *              (the model's).  A failed factorisation (a pivot below 1e-15 or not finite) or a new state or
 *              covariance that would not be finite returns MJPC_B200_ERR_BAD_ARGUMENT and leaves state, covariance
 *              and time untouched; last_error names the factor, or says "non-finite result".
 * reset, set_noise, set and update refuse a value that is not finite with MJPC_B200_ERR_BAD_ARGUMENT and change
 * nothing.
 *   get        state [nq+nv], covariance, time and the kind's scalars (any pointer may be NULL) */
typedef struct mjpc_b200_estimator mjpc_b200_estimator_t;
int mjpc_b200_estimator_destroy(mjpc_b200_estimator_t* f);
int mjpc_b200_estimator_reset(mjpc_b200_estimator_t* f, const double* state, double time, double covariance_scale,
                              double process_scale, double sensor_scale);
int mjpc_b200_estimator_set_noise(mjpc_b200_estimator_t* f, const double* process, const double* sensor);
int mjpc_b200_estimator_set(mjpc_b200_estimator_t* f, const double* state, const double* covariance, double time);
int mjpc_b200_estimator_update(mjpc_b200_estimator_t* f, const double* ctrl, const double* sensor, const float* mocap);
int mjpc_b200_estimator_get(const mjpc_b200_estimator_t* f, double* state, double* covariance, double* time,
                            double* scalars);
const char* mjpc_b200_estimator_last_error(const mjpc_b200_estimator_t* f);

/* MJPC's Unscented state estimator (mjpc/estimators/unscented.cc, kind 2 of class mjpc_b200_host::Estimator in
 * csrc/host/estimator.h): its 2 ndstate + 1 sigma-point steps are one launch (alpha 1, beta 2 by default).  update can
 * fail on the covariance or the sensor-covariance factor.  get: scalars[5] = {ndstate, nsigma, nsensordata, sigma-point
 * steps that raised a warning since reset, timestep}. */
int mjpc_b200_unscented_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                               double alpha, double beta, int device, mjpc_b200_estimator_t** out);

/* MJPC's Kalman state estimator (mjpc/estimators/kalman.cc, kind 1 of class mjpc_b200_host::Estimator): its
 * finite-difference Jacobians are one launch each (the centre state and its ndstate tangent-space perturbations
 * x (+) eps e_i, then x (+) -eps e_i when centered).  The reference's finite differences are 1e-6 one-sided, an fp64
 * setting: mujoco_mpc_b200.estimator.KALMAN_EPSILON / KALMAN_CENTERED are the engine's.  update_measurement (the same
 * arguments as update): C and the predicted sensors from one launch at the current state, then the gain, correction and
 * covariance update; it can fail on the sensor-covariance factor.  update_prediction: A and the next state from one
 * launch with the ctrl and mocap of the last successful measurement (zeros and the model's mocap after reset),
 * P = A P A' + diag(process noise), time += timestep.  update: both.  Both return MJPC_B200_ERR_BAD_ARGUMENT for a
 * filter that is not a Kalman filter.  get: scalars[6] = {ndstate, states per launch, nsensordata, steps that raised a warning
 * since reset, timestep, epsilon}. */
int mjpc_b200_kalman_create(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep,
                            double epsilon, int centered, int device, mjpc_b200_estimator_t** out);
int mjpc_b200_kalman_update_measurement(mjpc_b200_estimator_t* f, const double* ctrl, const double* sensor,
                                        const float* mocap);
int mjpc_b200_kalman_update_prediction(mjpc_b200_estimator_t* f);

/* ---- Batched state estimators (csrc/host/estimator.{h,cc}): num_filters independent filters of one kind on ONE
 * engine handle, each with its own state, covariance, time, noise, warm start, ctrl, sensors and mocap.  kind is the
 * reference's `estimator` numeric: 1 Kalman (settings {epsilon, centered}), 2 Unscented (settings {alpha, beta}).
 * Every update runs on the device: the filter arithmetic in fp64 (csrc/estimator_kernels.cuh) around one step launch of
 * all filters' rows per sigma-point set / Jacobian (Unscented one, Kalman two), the instance mjpc_b200_step_batch runs.
 * The host uploads ctrl, sensors and mocap once and downloads one status per filter; state and covariance stay on the
 * device until get.  Filter b computes what the single filter of its kind computes from the same state, covariance,
 * time, noise and warm start (bitwise: the single filter is the same code), with the same documented differences from
 * the reference.
 *   create     refuses what the single creates refuse: a bad argument or a sensor range outside the model's sensors
 *              (MJPC_B200_ERR_BAD_ARGUMENT), a bad blob (MJPC_B200_ERR_BAD_BLOB), a sensor the engine does not
 *              evaluate (MJPC_B200_ERR_UNSUPPORTED); and num_filters x rows per filter above 65536 step rows
 *              (MJPC_B200_ERR_CAPACITY; rows: Unscented 2 ndstate + 1, Kalman ndstate + 1, or 2 ndstate + 1 centred).
 *              Every filter starts as reset (NULL state, time 0, scales 1e-4) leaves it.
 *   reset      filter b as mjpc_b200_estimator_reset, zero warm start and warnings
 *   set_noise  filter b's process [ndstate] / sensor [nsensordata] noise (NULL keeps one)
 *   set        filter b's state, covariance [ndstate^2] (NULL keeps one) and time
 *   update     every filter from ctrl [num_filters][nu], sensor [num_filters][nsensordata] and mocap
 *              [num_filters][7 nmocap] (NULL: the model's for every filter).  status [num_filters]: 0, or
 *              MJPC_B200_ERR_BAD_ARGUMENT where a factorisation failed or the new state or covariance would not be
 *              finite, which leaves that filter's state, covariance, time, warm start and warnings untouched; the
 *              other filters update normally.  A ctrl, sensor or mocap value that is not finite refuses the whole call
 *              (MJPC_B200_ERR_BAD_ARGUMENT, nothing changed), as reset, set_noise and set refuse theirs
 *   get        filter b's state [nq+nv], covariance, time and the scalars of the single filter of its kind (Unscented
 *              5, Kalman 6; any pointer may be NULL)
 * Calls that take a filter index return MJPC_B200_ERR_BAD_ARGUMENT when it is outside [0, num_filters), and every call
 * returns it for a NULL handle (last_error: ""). */
int mjpc_b200_batch_estimator_create(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start,
                                     int nsensor, double timestep, const double* settings, int device, void** out);
int mjpc_b200_batch_estimator_destroy(void* f);
int mjpc_b200_batch_estimator_reset(void* f, int filter, const double* state, double time, double covariance_scale,
                                    double process_scale, double sensor_scale);
int mjpc_b200_batch_estimator_set_noise(void* f, int filter, const double* process, const double* sensor);
int mjpc_b200_batch_estimator_set(void* f, int filter, const double* state, const double* covariance, double time);
int mjpc_b200_batch_estimator_update(void* f, const double* ctrl, const double* sensor, const float* mocap,
                                     int* status);
int mjpc_b200_batch_estimator_get(void* f, int filter, double* state, double* covariance, double* time,
                                  double* scalars);
/* Test hooks: the bank's own kernels on the caller's data, with the bank's launch shape and stream.  phase: 0 the
 * Unscented sigma points, 1 the Kalman measurement, 2 the Kalman prediction (another phase than the kind's:
 * MJPC_B200_ERR_BAD_ARGUMENT).  status [num_filters] is the raw filter status: 0 updated, 1 sensor-covariance factor
 * failed, 2 covariance factor failed, 3 non-finite result.
 *   debug_rows    stages ctrl [num_filters][nu] and mocap (NULL: the model's) as update does and runs the row kernel:
 *                 qpos [num_filters rows][nq], qvel [num_filters rows][nv] and warm [num_filters rows][nv] are the step
 *                 launch's input rows and warm starts; phases 0 and 1 set status, phase 2 leaves the last one
 *   debug_finish  stages sensor [num_filters][nsensordata] (phase 2: may be NULL), clears every status, writes
 *                 next_qpos, next_qvel, qacc [num_filters rows][nv], sensordata [num_filters rows][nsensordata] and
 *                 counts [num_filters rows][4] where the step launch writes them and runs the phase's update kernel,
 *                 which commits into the filters as update does */
int mjpc_b200_batch_estimator_debug_rows(void* f, int phase, const double* ctrl, const float* mocap, float* qpos,
                                         float* qvel, float* warm, int* status);
int mjpc_b200_batch_estimator_debug_finish(void* f, int phase, const double* sensor, const float* next_qpos,
                                           const float* next_qvel, const float* qacc, const float* sensordata,
                                           const int* counts, int* status);
/* Filter b runs on models[b] from now on: mjpc_b200_set_model_variants on the bank's engine handle, with its rule and
 * refusals; a NULL-state reset and a NULL mocap then use filter b's model's first keyframe / qpos0 and mocap poses.
 * count must be num_filters, or 0 to run every filter on the bank's model again.  The filters' states are kept. */
int mjpc_b200_batch_estimator_set_models(void* f, const mjpc_model_blob* models, int count);
const char* mjpc_b200_batch_estimator_last_error(const void* f);

/* Per-candidate execution statistics of the last rollout, stats [N][12] = {SM cycles, Newton iterations, contacts,
 * constraint rows (summed over steps), 8 per-phase cycle counters (zero unless built with -DMJPC_PHASE_TIMING)}. */
int mjpc_b200_fetch_stats(mjpc_b200_t* h, int64_t* stats);

/* Number of CUDA kernels this handle has launched so far (bench.py reports it as gpu_launches). */
int64_t mjpc_b200_launch_count(const mjpc_b200_t* h);
/* Device time (ms, CUDA events on the engine's stream) of the kernels of the last call. */
float mjpc_b200_last_kernel_ms(const mjpc_b200_t* h);
/* Non-zero if the last rollout launch used a statically specialised kernel instance (model == a shipped task model,
 * csrc/spec_*.h): 1 = the shipped instance (one CTA per candidate: main warp + Hessian helper warps + task warp),
 * 2 = its one-warp-per-candidate twin (same source, selected only by MJPC_B200_SHAPE=plain: the bitwise reference of
 * the tests and the baseline of the profiles); 0 = the generic kernel (MJPC_B200_NO_STATIC=1 forces it).
 * The shipped instance keeps the two candidates that share an SM in step, meeting once per time step, when
 * #SMs < N <= 2 #SMs; MJPC_B200_PAIR_SYNC=0 disables this (a scheduling aid: it never changes a result). */
int mjpc_b200_last_kernel_static(const mjpc_b200_t* h);
/* Host-only: header + state-layout words of a model ({n_model, n_layout, model words, layout offsets}); what
 * mujoco_mpc_b200/gen_spec.py writes into csrc/spec_*.h.  Returns the number of ints written or <0. */
int mjpc_b200_spec_words(const mjpc_model_blob* model, int* out, int capacity);

/* Resident-input path used for the device-timed bench value: upload once, then launch repeatedly. */
int mjpc_b200_upload_spline_inputs(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                                   const float* userdata, const float* knots, const double* knot_times, int interp,
                                   int P, int N, int H);
int mjpc_b200_launch_resident(mjpc_b200_t* h);          /* async on the engine stream; refused after a set_options timestep change (upload again) */
int mjpc_b200_sync(mjpc_b200_t* h);
int mjpc_b200_read_returns(mjpc_b200_t* h, float* returns, uint8_t* failure, int* order);
/* ---- Multi-GPU: ONE planning problem, its candidates sharded over the ranks of an NCCL communicator owned by the
 * handle (one process per GPU).  Rank g owns the contiguous candidate range [g*N/G, (g+1)*N/G) (the first N % G ranks
 * one more); candidate 0, the un-noised nominal (sampling/planner.cc:374), lives on rank 0.  The single exchange per
 * planning iteration - per-candidate returns + failure flags - is one ncclAllGather enqueued on the engine stream
 * behind the rollout kernel; ranking runs on the device on the gathered vector, so every rank sees the same
 * returns / failure / order for all N candidates (north_star: "a single NCCL all-reduce of per-candidate returns").
 * NCCL is bound with dlopen("libnccl.so.2") at the first call; without it these return MJPC_B200_ERR_UNSUPPORTED.
 *   comm_unique_id: rank 0 generates the 128-byte ncclUniqueId, the caller distributes it (MPI / torch.distributed / file)
 *   comm_init:      collective over all ranks (ncclCommInitRank)                                                     */
int mjpc_b200_comm_unique_id(void* out, size_t nbytes);
int mjpc_b200_comm_init(mjpc_b200_t* h, int nranks, int rank, const void* unique_id, size_t nbytes);
int mjpc_b200_comm_info(const mjpc_b200_t* h, int* nranks, int* rank);
/* Same arguments on every rank (knots [N][P][nu] for ALL candidates; inputs are replicated, a few KB).  N may be up to
 * nranks * max_candidates.  returns [N], failure [N], order [N] are global and identical on every rank. */
int mjpc_b200_rollout_spline_sharded(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                                     const float* userdata, const float* knots, const double* knot_times, int interp,
                                     int P, int N, int H, float* returns, uint8_t* failure, int* order);
/* Trajectory of GLOBAL candidate index on every rank (ncclBroadcast from its owner); collective. */
int mjpc_b200_fetch_trajectory_sharded(mjpc_b200_t* h, int candidate, float* states, float* actions, double* times,
                                       float* residual, float* costs, float* trace);

/* Raw stream / device pointers for multi-GPU plumbing (NCCL all-gather of returns runs on this stream). */
void* mjpc_b200_stream(mjpc_b200_t* h);
float* mjpc_b200_device_returns(mjpc_b200_t* h);

/* ---- C++ host layer above the ABI (csrc/host): the reference's planners with its method names; these C wrappers are
 * what ctypes / a test harness binds.
 * mjpc_b200_host_spline_sample = TimeSpline::Sample (mjpc/spline/spline.cc:103-156), usable without a GPU. */
void mjpc_b200_host_spline_sample(const double* times, const double* values, int P, int dim, int interp, double t,
                                  double* out);
/* The step table a rollout launch builds per problem to place its policy in time, usable without a GPU: the rollout
 * time times[t] (time0 plus t timesteps, accumulated in double as mj_step does), upper[t] = the first of the `count`
 * non-decreasing absolute node times (spline knot times or the feedback policy's nominal times) above times[t], and
 * frac[t] = the fraction of times[t] between nodes upper[t] - 1 and upper[t], in double rounded to float (0 when
 * upper[t] is 0 or count).  The spline samples and FindInterval's bounds of every step follow from upper[t]. */
void mjpc_b200_host_policy_intervals(const double* nodes, int count, double time0, double timestep, int H, double* times,
                                     int* upper, float* frac);
double mjpc_b200_host_philox_normal(uint32_t seed, uint32_t iteration, uint32_t candidate, uint32_t knot, uint32_t dof);

/* ---- Planners (csrc/host/planner.h, the reference's Planner interface mjpc/planners/planner.h:33-77).  Each kind has
 * its own create (its settings) and get_result (its result shape), and the sampling and iLQS planners a
 * set_exploration; these return MJPC_B200_ERR_BAD_ARGUMENT for a NULL handle or one of another kind.  Every other call
 * is one of the generic mjpc_b200_planner_* below, which take a planner of any kind and return
 * MJPC_B200_ERR_BAD_ARGUMENT for a NULL one.
 *   reset               Planner::Reset to horizon steps; initial_repeated_action [nu] may be NULL
 *   set_state           state [dim_state], absolute time, mocap [7 nmocap] (NULL keeps the previous one)
 *   optimize_policy     Planner::OptimizePolicy: <0 on error.  The sampling, Cross-Entropy, Sample Gradient and Robust
 *                       planners return 0; iLQG and iLQS 1 when the policy was updated, 0 when the iteration was
 *                       rejected; Gradient 1 when the return improved, 0 when the nominal was kept
 *   nominal_trajectory  Planner::NominalTrajectory, what planning does while it is disabled
 *   action_from_policy  action [nu] of the policy at `time`.  state [dim_state] (may be NULL: open loop) is read by the
 *                       iLQG policy (iLQG, iLQS); use_previous != 0 reads the previous policy of the sampling-based
 *                       planners (the others ignore it)
 *   set_fd              finite-difference settings of the derivative-based planners (ilqg/settings.h:23-24,
 *                       iLQGPlanner::derivative_skip_): tolerance <= 0 / mode < 0 / skip < 0 keep the current value.
 *                       Defaults 3e-4, centred, 0 (the reference's 1e-6 one-sided is an fp64 setting, ilqg_planner.h).
 *                       Gradient, iLQG and the iLQG half of iLQS; the others return MJPC_B200_ERR_UNSUPPORTED */
typedef struct mjpc_b200_planner mjpc_b200_planner_t;
int mjpc_b200_planner_destroy(mjpc_b200_planner_t* p);
int mjpc_b200_planner_reset(mjpc_b200_planner_t* p, int horizon, const double* initial_repeated_action);
int mjpc_b200_planner_set_state(mjpc_b200_planner_t* p, const double* state, double time, const double* mocap);
int mjpc_b200_planner_optimize_policy(mjpc_b200_planner_t* p, int horizon);
int mjpc_b200_planner_nominal_trajectory(mjpc_b200_planner_t* p, int horizon);
int mjpc_b200_planner_action_from_policy(mjpc_b200_planner_t* p, double* action, const double* state, double time,
                                         int use_previous);
int mjpc_b200_planner_set_fd(mjpc_b200_planner_t* p, double tolerance, int mode, int derivative_skip);
/* Plan on a model ensemble: mjpc_b200_set_model_ensemble on the planner's handle, with its rule and refusals (K = 0 or
 * models NULL clears it).  The planner ranks by the scores; returns and improvement of its get_result are scores, and
 * the best trajectory is member 0's trajectory of the winner with the winner's score as its return.  Sampling,
 * Cross-Entropy and Sample Gradient; Robust, Gradient, iLQG and iLQS return MJPC_B200_ERR_UNSUPPORTED. */
int mjpc_b200_planner_set_ensemble(mjpc_b200_planner_t* p, const mjpc_model_blob* models, int K, int worst);
/* Plan over the state estimate's uncertainty: every spline launch of the planner becomes
 * mjpc_b200_rollout_spline_belief_batched with K members per problem, `worst`, `seed` and the planner's own iteration
 * counter, from the covariance of set_state_covariance.  The planner ranks by the scores, as with a model ensemble.
 * K = 0 clears it.  K outside [0, 32] or worst outside [1, K]: MJPC_B200_ERR_BAD_ARGUMENT.  Refused
 * (MJPC_B200_ERR_UNSUPPORTED) while a model ensemble is set, and set_ensemble (K > 0) is refused while a state ensemble
 * is set.  Sampling, Cross-Entropy and Sample Gradient; Robust, Gradient, iLQG and iLQS return
 * MJPC_B200_ERR_UNSUPPORTED. */
int mjpc_b200_planner_set_state_ensemble(mjpc_b200_planner_t* p, int K, int worst, uint32_t seed);
/* The state covariance [2 nv][2 nv] (double) the planner's state-ensemble launches draw from until the next call; NULL
 * is zero, as is a planner's covariance before the first call (its members then all equal the mean and its scores are
 * the plain returns).  A non-finite entry: MJPC_B200_ERR_BAD_ARGUMENT, nothing changed.  The kinds of
 * set_state_ensemble. */
int mjpc_b200_planner_set_state_covariance(mjpc_b200_planner_t* p, const double* covariance);
/* mjpc_b200_set_task on every engine handle the planner plans on (the task snapshot Agent gives it per iteration) */
int mjpc_b200_planner_set_task(mjpc_b200_planner_t* p, const mjpc_task_desc* task);

/* ---- Predictive Sampling (csrc/host/sampling_planner.{h,cc}; mjpc/planners/sampling/planner.h:40-160). */
int mjpc_b200_sampling_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points,
                                      int interpolation, double exploration, double timestep, const double* ctrlrange,
                                      uint32_t seed, int max_horizon, int device, mjpc_b200_planner_t** out);
/* noise_exploration[0..1] (sampling/planner.cc:85-88, 334-338): exploration2 > 0 replaces the std with probability 0.2 */
int mjpc_b200_sampling_planner_set_exploration(mjpc_b200_planner_t* p, double exploration, double exploration2);
/* winner, improvement, returns [num_trajectory], installed knots [P][nu] / times [P]; returns the number of knots */
int mjpc_b200_sampling_planner_get_result(mjpc_b200_planner_t* p, int* winner, double* improvement, float* returns,
                                          double* knots, double* knot_times);

/* ---- Cross-Entropy planner (csrc/host/cross_entropy_planner.{h,cc}; mjpc/planners/cross_entropy/planner.h:35-146).
 * One rollout launch covers the N noisy candidates and the un-noised nominal (candidate N); the elite mean and
 * variance are host arithmetic in double, as in the reference (planner.cc:201-262).  n_elite <= 0 selects the
 * reference default max(N/10, 2). */
int mjpc_b200_ce_planner_create(const mjpc_model_blob* model, int num_trajectory, int n_elite, int num_spline_points,
                                int interpolation, double std_initial, double std_min, double explore_fraction,
                                double timestep, const double* ctrlrange, uint32_t seed, int max_horizon, int device,
                                mjpc_b200_planner_t** out);
/* improvement, returns [N+1] (last = nominal), elite order [N], installed knots [P][nu] / times [P], variance [P][nu];
 * returns the number of spline points */
int mjpc_b200_ce_planner_get_result(mjpc_b200_planner_t* p, double* improvement, float* returns, int* order,
                                    double* knots, double* knot_times, double* variance);

/* ---- Sample Gradient planner (csrc/host/sample_gradient_planner.{h,cc}; mjpc/planners/sample_gradient/planner.cc).
 * One rollout launch covers candidate 0 (the resampled nominal), the noisy samples 1 .. N-G-1 (knot += exploration * z,
 * not scaled by the control range) and the G gradient candidates N-G .. N-1 computed by the previous iteration; the
 * fitness-shaped gradient estimate and the log-spaced steps (1e-3 .. 2) along it are host arithmetic in double.
 * num_gradient is clamped to N - 1 on every optimize_policy; nominal_trajectory rolls out the resampled nominal alone.
 * Requires num_trajectory >= 1, num_spline_points >= 2. */
int mjpc_b200_sg_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_gradient, int num_spline_points,
                                int interpolation, double exploration, double gradient_filter, double timestep,
                                const double* ctrlrange, uint32_t seed, int max_horizon, int device,
                                mjpc_b200_planner_t** out);
/* winner, winner_type (0 nominal, 1 noisy, 2 gradient), improvement, returns [N], order [N] (as trajectory_order holds
 * it: the ranking of all N, or of the N-G noisy samples in its first N-G entries on the call that computed the
 * fitness weights), installed knots [P][nu] / times [P], gradient candidates' knots [G][P][nu] as the next iteration
 * resamples and rolls them out, gradient [P][nu].  Any pointer may be NULL; returns the number of installed knots. */
int mjpc_b200_sg_planner_get_result(mjpc_b200_planner_t* p, int* winner, int* winner_type, double* improvement,
                                    float* returns, int* order, double* knots, double* knot_times,
                                    double* gradient_knots, double* gradient);

/* ---- Robust planner (csrc/host/robust_planner.{h,cc}; mjpc/planners/robust/robust_planner.cc:40-160) over the
 * sampling planner: the best `ncandidates` of the clean launch are re-rolled `nrepetitions` times each with
 * NoisyRollout force perturbations (one launch on a second handle) and the best mean score is installed.
 * ncandidates = -1 -> num_trajectory / nrepetitions, nrepetitions <= 0 -> 5 (the reference's defaults). */
int mjpc_b200_robust_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points,
                                    int interpolation, double exploration, double timestep, const double* ctrlrange,
                                    uint32_t seed, int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate,
                                    int max_horizon, int device, mjpc_b200_planner_t** out);
/* winner, robust scores [ncandidates], clean returns [num_trajectory], installed knots/times; returns #scores */
int mjpc_b200_robust_planner_get_result(mjpc_b200_planner_t* p, int* winner, double* scores, float* returns,
                                        double* knots, double* knot_times);

/* ---- Task::Transition of the config tasks on the host (csrc/host/task_transition.{h,cc}): the state machines that
 * produce the task-state block the kernels consume (QuadrupedFlat::TransitionLocked quadruped.cc:228-395,
 * Tracking::TransitionLocked tracking.cc:218-267).  Host only - no device, no handle.
 * quadruped ids[14] = {p_gait, p_gait_switch, p_cadence, p_amplitude, p_duty, p_walk_speed, p_walk_turn,
 *                      w_upright, w_height, w_position, w_gait, w_balance, w_effort, w_posture};
 * view[24] = {time, torso_subtreelinvel[3], torso_xmat[9], torso_xpos[3], torso_xquat[4], head_site_xpos[3],
 *             ground height under the torso subtree com (read when the Flip mode starts)}. */
void* mjpc_b200_quadruped_transition_create(const int* ids, const double* parameters, int nparam, const double* weight,
                                            int nweight, const double* task_state, int nstate, const double* goal_pos);
void mjpc_b200_quadruped_transition_destroy(void* transition);
/* caller / GUI edits of Task::parameters and Task::weight between transitions (either may be NULL) */
void mjpc_b200_quadruped_transition_set(void* transition, const double* parameters, const double* weight);
void mjpc_b200_quadruped_transition_step(void* transition, int* mode_inout, const double* view, double* parameters,
                                         double* weight, double* task_state, double* goal_pos);
void* mjpc_b200_track_transition_create(int nq, int nv, int nmocap, int nkey, const double* key_qpos,
                                        const double* key_qvel, const double* key_mpos);
void mjpc_b200_track_transition_destroy(void* transition);
void mjpc_b200_track_transition_step(void* transition, int mode, double time, double* qpos, double* qvel,
                                     double* mocap_pos, double* task_state);

/* ShadowReorient::TransitionLocked (hand.cc:90-119): cube at rest on the floor -> back into the hand.  Returns 1 on a reset. */
void* mjpc_b200_shadow_transition_create(int cube_qposadr, int cube_dofadr, const double* qpos0_cube /*[7]*/);
void mjpc_b200_shadow_transition_destroy(void* transition);
int mjpc_b200_shadow_transition_step(void* transition, double* qpos, double* qvel, int on_floor, const double* cube_linvel);

/* ---- iLQG planner (csrc/host/ilqg_planner.{h,cc}; mjpc/planners/ilqg/planner.h, planner.cc:156-740).
 * OptimizePolicy = NominalTrajectory (feedback-scaling line search) + Iteration (model derivatives, cost derivatives,
 * backward pass with the regularisation retry loop, K action rollouts, winner, regularisation update); each sweep is
 * one call of the ABI above.  fd_tolerance <= 0 keeps the default (set_fd).  action_from_policy is iLQGPolicy::Action
 * (ilqg/policy.cc:82-161): with a state the time-varying feedback feedback_scaling * K (state (-) x_nominal) is added
 * before clamping. */
int mjpc_b200_ilqg_planner_create(const mjpc_model_blob* model, int num_rollouts, int representation, double fd_tolerance,
                                  int max_horizon, int device, mjpc_b200_planner_t** out);
/* iLQGPolicy::Action, stateless and host only: u_nom [H][nu], x_nom [H][dim_state], t_nom [H], gains [H][nu][2 nv] */
int mjpc_b200_host_ilqg_policy_action(const mjpc_model_blob* model, const float* u_nom, const float* x_nom,
                                      const double* t_nom, const float* gains, int horizon, int representation,
                                      double feedback_scaling, const double* state, double time, double* action);
/* scalars[6] = {total_return, regularization, improvement, expected, surprise, winner}; nominal states [H][dim_state],
 * actions [H][nu], times [H] (any pointer may be NULL); returns H */
int mjpc_b200_ilqg_planner_get_result(mjpc_b200_planner_t* p, double* scalars, float* states, float* actions,
                                      double* times);

/* ---- Gradient planner (csrc/host/gradient_planner.{h,cc}; mjpc/planners/gradient/planner.cc:159-383, gradient.cc:44-107,
 * spline_mapping.cc): ResamplePolicy, nominal rollout, {model derivatives, cost derivatives, gradient sweep, total derivative
 * through the spline mapping, K line-search rollouts (ONE mjpc_b200_rollout_spline launch)} x max_rollout.
 * fd_tolerance <= 0 keeps the default (set_fd). */
int mjpc_b200_gradient_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int representation,
                                      double fd_tolerance, double timestep, const double* ctrlrange, int max_horizon, int device,
                                      mjpc_b200_planner_t** out);
/* scalars[6] = {total_return, winner, action_step, expected, improvement, surprise}; parameters [P][nu], times [P] */
int mjpc_b200_gradient_planner_get_result(mjpc_b200_planner_t* p, double* scalars, double* parameters, double* times);
/* SplineMapping::Compute (gradient/spline_mapping.cc) as scalar weights W [num_output][num_input]; host only */
void mjpc_b200_host_spline_mapping(int representation, const double* input_times, int num_input, const double* output_times,
                                   int num_output, double* W);
/* Gradient::Compute's recursion on the host in fp64 (the single planner's GradientSweep); host only.  A [T][n][n],
 * B [T][n][m], cx [T][n], cu [T][m] -> k [T][m] (row T-1 repeats row T-2), *dV0.  The reference of
 * mjpc_b200_gradient_batched. */
void mjpc_b200_host_gradient_sweep(const float* A, const float* B, const float* cx, const float* cu, int n, int m, int T,
                                   double* k, double* dV0);

/* ---- iLQS planner (csrc/host/gradient_planner.{h,cc}; mjpc/planners/ilqs/planner.cc:87-215): Predictive Sampling first;
 * when it does not improve, one iLQG iteration seeded with the sampling nominal; when sampling follows iLQG the trajectory
 * policy is converted to spline parameters through the least-squares inverse of the spline mapping. */
int mjpc_b200_ilqs_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                                  double exploration, double timestep, const double* ctrlrange, uint32_t seed,
                                  int ilqg_num_rollouts, int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                                  mjpc_b200_planner_t** out);
int mjpc_b200_ilqs_planner_set_exploration(mjpc_b200_planner_t* p, double exploration);   /* its sampling half */
/* scalars[4] = {active_policy (0 sampling, 1 iLQG), sampling winner return, iLQG total_return, sampling winner}; returns active_policy */
int mjpc_b200_ilqs_planner_get_result(mjpc_b200_planner_t* p, double* scalars);

/* ---- Batch planners (csrc/host/batch_planner.h): num_problems independent planners of one kind on ONE engine handle
 * (two for the Robust and iLQS batches, as their single planners have), each problem with its own seed, state, mocap,
 * task snapshot and policy.  An iteration runs the kind's one iteration over every problem, one batched launch per
 * sweep, so each problem's result equals that of the kind's single planner with the same seed and inputs.  Settings are
 * common to a batch.  Each kind has its own create (the single planner's create arguments plus num_problems, and
 * seeds [num_problems] in place of seed) and get_result (the single planner's get_result of one problem), the iLQS
 * batch a set_exploration and the iLQG batch a nominal_trajectory; these return MJPC_B200_ERR_BAD_ARGUMENT for a NULL
 * handle or one of another kind.  Every other call is one of the generic mjpc_b200_batch_planner_* below, which take a
 * batch of any kind and return MJPC_B200_ERR_BAD_ARGUMENT for a NULL one (destroy ignores it).  A call that takes a
 * problem index returns MJPC_B200_ERR_BAD_ARGUMENT when it is outside [0, num_problems).
 *   reset               mjpc_b200_planner_reset of one problem
 *   set_state           mjpc_b200_planner_set_state of one problem; state must not be NULL
 *   set_task            one problem's task snapshot (weight, parameters, task state), which starts as the model's; NULL
 *                       members keep the current value
 *   set_models          problem b plans on models[b] from now on: mjpc_b200_set_model_variants, with its rule and
 *                       refusals, on every engine handle the batch owns.  count must be num_problems, or 0 to plan every
 *                       problem on the batch's model again.  Valid between planning iterations (after an online system
 *                       identification, for example).  The planners' settings and ctrlrange stay the batch's: variants
 *                       must share actuator_ctrlrange
 *   optimize_policy     Planner::OptimizePolicy of every problem: <0 on error.  codes [num_problems] (may be NULL)
 *                       receives what each problem's single planner's optimize_policy returns: 0 for Sampling,
 *                       Cross-Entropy, Sample Gradient and Robust, 1 / 0 for Gradient, iLQG and iLQS; all 0 after an
 *                       error
 *   action_from_policy  mjpc_b200_planner_action_from_policy of one problem: state (may be NULL) is read by the iLQG
 *                       policy (iLQG, iLQS)
 *   set_fd              mjpc_b200_planner_set_fd of every problem: Gradient, iLQG and iLQS; the others return
 *                       MJPC_B200_ERR_UNSUPPORTED
 *   set_ensemble        every problem plans on the same model ensemble: mjpc_b200_planner_set_ensemble's kinds and
 *                       refusals, on the batch's handle
 *   set_state_ensemble  every problem plans over its state covariance with the same K, worst and seed:
 *                       mjpc_b200_planner_set_state_ensemble's kinds and refusals; the batch's one launch draws problem
 *                       b with key seed + b (so problem b of a batch draws what a single planner with seed + b draws)
 *                       and the iteration counter of problem 0 (the problems iterate together)
 *   set_state_covariance  problem `problem`'s covariance: mjpc_b200_planner_set_state_covariance */
typedef struct mjpc_b200_batch_planner mjpc_b200_batch_planner_t;
void mjpc_b200_batch_planner_destroy(mjpc_b200_batch_planner_t* p);
int mjpc_b200_batch_planner_reset(mjpc_b200_batch_planner_t* p, int problem, int horizon,
                                  const double* initial_repeated_action);
int mjpc_b200_batch_planner_set_state(mjpc_b200_batch_planner_t* p, int problem, const double* state, double time,
                                      const double* mocap);
int mjpc_b200_batch_planner_set_task(mjpc_b200_batch_planner_t* p, int problem, const double* weight,
                                     const double* parameters, const double* task_state);
int mjpc_b200_batch_planner_set_models(mjpc_b200_batch_planner_t* p, const mjpc_model_blob* models, int count);
int mjpc_b200_batch_planner_optimize_policy(mjpc_b200_batch_planner_t* p, int horizon, int* codes);
int mjpc_b200_batch_planner_action_from_policy(mjpc_b200_batch_planner_t* p, int problem, double* action,
                                               const double* state, double time, int use_previous);
int mjpc_b200_batch_planner_set_fd(mjpc_b200_batch_planner_t* p, double tolerance, int mode, int derivative_skip);
int mjpc_b200_batch_planner_set_ensemble(mjpc_b200_batch_planner_t* p, const mjpc_model_blob* models, int K, int worst);
int mjpc_b200_batch_planner_set_state_ensemble(mjpc_b200_batch_planner_t* p, int K, int worst, uint32_t seed);
int mjpc_b200_batch_planner_set_state_covariance(mjpc_b200_batch_planner_t* p, int problem, const double* covariance);

/* Predictive Sampling: one mjpc_b200_rollout_spline_batched launch of B x N per iteration. */
int mjpc_b200_batch_sampling_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                            int num_spline_points, int interpolation, double exploration,
                                            double timestep, const double* ctrlrange, const uint32_t* seeds,
                                            int max_horizon, int device, mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_sampling_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, int* winner,
                                                double* improvement, float* returns, double* knots,
                                                double* knot_times);
/* Cross-Entropy: one launch of B x (N + 1). */
int mjpc_b200_batch_ce_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory, int n_elite,
                                      int num_spline_points, int interpolation, double std_initial, double std_min,
                                      double explore_fraction, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device,
                                      mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_ce_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, double* improvement,
                                          float* returns, int* order, double* knots, double* knot_times,
                                          double* variance);
/* Sample Gradient: one launch of B x N. */
int mjpc_b200_batch_sg_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                      int num_gradient, int num_spline_points, int interpolation, double exploration,
                                      double gradient_filter, double timestep, const double* ctrlrange,
                                      const uint32_t* seeds, int max_horizon, int device,
                                      mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_sg_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, int* winner, int* winner_type,
                                          double* improvement, float* returns, int* order, double* knots,
                                          double* knot_times, double* gradient_knots, double* gradient);
/* Robust: a clean launch of B x N, then one noisy launch of B x ncandidates x nrepetitions on a second handle, each
 * problem drawing its force noise with its own key seed + iteration (mjpc_b200_set_xfrc_noise_batched). */
int mjpc_b200_batch_robust_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                          int num_spline_points, int interpolation, double exploration, double timestep,
                                          const double* ctrlrange, const uint32_t* seeds, int ncandidates,
                                          int nrepetitions, double xfrc_std, double xfrc_rate, int max_horizon,
                                          int device, mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_robust_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, int* winner, double* scores,
                                              float* returns, double* knots, double* knot_times);
/* Gradient: per max_rollout iteration one spline launch of the B resampled nominals, one mjpc_b200_gradient_batched on
 * their trajectories and one spline launch of the B x num_trajectory line-search candidates. */
int mjpc_b200_batch_gradient_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                            int num_spline_points, int representation, double fd_tolerance,
                                            double timestep, const double* ctrlrange, int max_horizon, int device,
                                            mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_gradient_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, double* scalars,
                                                double* parameters, double* times);
/* iLQS: sampling on a handle of num_problems x num_trajectory, iLQG on one of num_problems x ilqg_num_rollouts.  Per
 * iteration at most one feedback launch of the iLQG nominals of the problems whose active policy was iLQG, one spline
 * launch of every problem's sampling, then, for the problems sampling did not settle, one batched derivative sweep, one
 * batched cost-derivative call, backward-pass rounds of the problems still failing and one action-rollout launch.
 * set_exploration sets every problem's. */
int mjpc_b200_batch_ilqs_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                        int num_spline_points, int interpolation, double exploration, double timestep,
                                        const double* ctrlrange, const uint32_t* seeds, int ilqg_num_rollouts,
                                        int ilqg_representation, double fd_tolerance, int max_horizon, int device,
                                        mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_ilqs_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, double* scalars);
int mjpc_b200_batch_ilqs_planner_set_exploration(mjpc_b200_batch_planner_t* p, double exploration);
/* iLQG: one batched launch per sweep for all problems; backward passes are retried in batches of the problems still
 * failing.  nominal_trajectory is every problem's iLQGPlanner::NominalTrajectory in one launch. */
int mjpc_b200_batch_ilqg_planner_create(const mjpc_model_blob* model, int num_problems, int num_rollouts,
                                        int representation, double fd_tolerance, int max_horizon, int device,
                                        mjpc_b200_batch_planner_t** out);
int mjpc_b200_batch_ilqg_planner_get_result(mjpc_b200_batch_planner_t* p, int problem, double* scalars, float* states,
                                            float* actions, double* times);
int mjpc_b200_batch_ilqg_planner_nominal_trajectory(mjpc_b200_batch_planner_t* p, int horizon);

/* ---- Agent::PlanIteration glue (csrc/host/agent.{h,cc}; mjpc/agent.cc:85-107,150-164,283-357): owns the planner selected
 * by agent_planner (0 Sampling, 1 Gradient, 2 iLQG, 3 iLQS, 4 Robust, 5 Cross-Entropy; mjpc/planners/include.h:26-34) and does
 * per iteration what the reference does around OptimizePolicy: steps_ = int(max(min(horizon / timestep + 1, 512), 1)),
 * timestep / integrator override, MakeDifferentiable for gradient-based planners (restored afterwards), SetState, the
 * residual snapshot (set_task on every engine handle of the planner), OptimizePolicy(steps_) - or NominalTrajectory when
 * planning is disabled.
 * settings[20] = {planner, horizon, timestep, integrator, differentiable (-1 = the reference default), num_trajectory,
 *   num_spline_points, representation, exploration, ilqg_num_rollouts, ilqg_representation, fd_tolerance, n_elite, std_min,
 *   explore_fraction, robust_candidates, robust_repetitions, robust_xfrc, robust_xfrc_rate, seed} */
/* agent_planner 6 is the Sample Gradient planner (above).  It takes settings[22]: the twenty entries above, then
 * settings[20] = sample_gradient_trajectories and settings[21] = sample_gradient_filter.  Those two are read only when
 * settings[0] == 6, so a caller of planners 0-5 may keep passing 20 values. */
int mjpc_b200_agent_steps(double horizon, double timestep);
int mjpc_b200_agent_create(const mjpc_model_blob* model, const double* settings, const double* ctrlrange, int device, void** out);
void mjpc_b200_agent_destroy(void* agent);
void mjpc_b200_agent_reset(void* agent, const double* initial_repeated_action);
void mjpc_b200_agent_set_state(void* agent, const double* state, double time, const double* mocap);
void mjpc_b200_agent_set_task(void* agent, const mjpc_task_desc* task);
void mjpc_b200_agent_set_plan_enabled(void* agent, int on);
int mjpc_b200_agent_plan_iteration(void* agent);
int mjpc_b200_agent_get_steps(void* agent);
void mjpc_b200_agent_action_from_policy(void* agent, double* action, const double* state, double time, int use_previous);

#ifdef __cplusplus
}
#endif
#endif /* MJPC_B200_H_ */
