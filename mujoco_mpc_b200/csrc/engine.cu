// engine.cu - host side of libmjpc_b200.so: the C ABI declared in include/mjpc_b200.h.
// Owns the device buffers, the stream and the pinned staging areas; validates arguments; launches the
// kernels in rollout_kernels.cuh / ilqg_kernels.cuh / estimator_kernels.cuh.  There is deliberately NO CPU fallback: without a
// usable CUDA device every entry point returns MJPC_B200_ERR_CUDA.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>   // types only: the NCCL entry points are bound with dlopen at comm_init (no link-time dependency)

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mjpc_b200.h"
#include "belief_kernels.cuh"
#include "device_memory.h"
#include "estimator_kernels.cuh"
#include "filter_bank.h"
#include "ilqg_kernels.cuh"
#include "plant_bank.h"
#include "rollout_kernels.cuh"

using namespace mjpc_dev;
using mjpc_mem::DeviceArray;
using mjpc_mem::PinnedArray;

namespace {
thread_local std::string g_last_error;
int fail(int code, const std::string& msg) { g_last_error = msg; return code; }

#define CUDA_TRY(expr)                                                                                     \
  do {                                                                                                     \
    cudaError_t e_ = (expr);                                                                               \
    if (e_ != cudaSuccess)                                                                                 \
      return fail(MJPC_B200_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));                 \
  } while (0)

// indices of task_state entries that hold absolute times (rebased to the rollout start before upload)
std::vector<int> time_like_state(int residual_id) {
  if (residual_id == RESIDUAL_QUADRUPED_FLAT) return {QS_MODE_START_TIME, QS_PHASE_START_TIME};
  if (residual_id == RESIDUAL_HUMANOID_TRACK) return {1};   // reference_time
  return {};
}

// The compiled kernel instances for one task model: the generic (DynSpec) ones, or those statically specialised for a
// model table (spec_*.h), which create() selects with spec_matches.
struct KernelSet {
  const void* rollout;         // shipped shape, rollout_threads threads per candidate
  const void* rollout_plain;   // one warp per candidate: the bitwise reference of the shipped shape
  const void* step;
  const void* fd_center;
  const void* fd_column;
  int rollout_threads;
  const void* plant;           // one step of every closed-loop plant (plant_bank.h)
};
const KernelSet kGenericKernels = {(const void*)rollout_kernel, (const void*)rollout_kernel, (const void*)step_batch_kernel,
                                   (const void*)fd_center_kernel, (const void*)fd_column_kernel, 32,
                                   (const void*)plant_step_kernel};
const KernelSet kQuadrupedKernels = {(const void*)rollout_kernel_quadruped, (const void*)rollout_kernel_quadruped_plain,
                                     (const void*)step_batch_kernel_quadruped, (const void*)fd_center_kernel_quadruped,
                                     (const void*)fd_column_kernel_quadruped, kRolloutThreads,
                                     (const void*)plant_step_kernel_quadruped};
// (no static fd instances: the Humanoid Track's derivative sweeps run the generic ones)
const KernelSet kHumanoidTrackKernels = {(const void*)rollout_kernel_humanoid_track,
                                         (const void*)rollout_kernel_humanoid_track_plain,
                                         (const void*)step_batch_kernel_humanoid_track, (const void*)fd_center_kernel,
                                         (const void*)fd_column_kernel, kRolloutThreads,
                                         (const void*)plant_step_kernel_humanoid_track};
}  // namespace

// The device filter bank of the state estimators (filter_bank.h): one allocation carved into the filters' fields, the
// per-update inputs, the rows of the step launch and its outputs, and the filters' scratch; pinned staging for the
// update's inputs and statuses.
struct FilterBank {
  FilterBankArgs a;
  int s0 = 0, nsens = 0, adr0 = 0, nsd = 0;
  DeviceArray<unsigned char> d_mem;
  float *d_rtime = nullptr, *d_task = nullptr, *d_res = nullptr, *d_cost = nullptr;
  unsigned char* d_in = nullptr;   // sensor [B][ny] doubles, ctrl [B][nu] and mocap [B][7 nmocap] floats
  PinnedArray<unsigned char> h_stage;
  size_t in_bytes = 0;
};

struct mjpc_b200 {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  ModelPack pack;
  int maxN = 0, maxH = 0, maxP = 64;
  int num_sms = 132;
  size_t smem_optin = 0;   // the device's opt-in limit of dynamic shared memory per block
  int max_term_dim = 1;    // widest cost term (task_dim_norm_residual): sizes cost_derivatives_kernel's scratch
  const KernelSet* kernels = &kGenericKernels;   // chosen at create: the model's static instances, if it has them
  DeviceArray<float> d_pack;
  // inputs: d_in holds the per-problem inputs and the knots of the last rollout launch (stage_problems)
  DeviceArray<float> d_in;
  // feedback policy of each problem of the last feedback launch ([fb_nprob][max_horizon][..]; grown on demand)
  DeviceArray<float> d_unom, d_xnom, d_tnom, d_gains, d_du, d_steps;
  int fb_nprob = 1;
  // outputs
  DeviceArray<float> d_states, d_actions, d_residual, d_costs, d_trace, d_returns;
  DeviceArray<double> d_times;
  DeviceArray<unsigned char> d_failure;
  DeviceArray<int> d_order;
  DeviceArray<long long> d_stats;
  DeviceArray<unsigned> d_pair_sync;   // [256][32]: per-SM records of the co-resident pair synchronisation (dev_data.cuh)
  // geometric contacts of the last step_debug (-1: none run yet) and their [maxcon][8] rows
  int dbg_ncon = -1;
  std::vector<float> dbg_contact;
  IlqgBuffers ilqg;
  std::unique_ptr<FilterBank> bank;   // the state estimators' filters (filter_bank.h), made by mjpc_b200_bank::Init
  std::unique_ptr<PlantBank> plants;  // the closed-loop plants (plant_bank.h), made by mjpc_b200_plant_init
  // pinned staging
  PinnedArray<float> h_in;
  size_t h_in_floats = 0;
  PinnedArray<unsigned char> h_out;
  size_t h_out_bytes = 0;
  // host copies of the live task
  std::vector<double> weight, parameters, task_state;
  double risk = 0;
  std::vector<int> time_idx;
  int lastN = 0, lastH = 0;
  int64_t launches = 0;
  float xfrc_std = 0.f, xfrc_rate = 1.f;   // NoisyRollout settings for the following rollouts (0 = off)
  unsigned noise_seed = 0;
  std::vector<unsigned> noise_seeds;   // set_xfrc_noise_batched: one key per problem of the following launches (else empty)
  int last_static = 0;
  float last_ms = 0;
  // multi-GPU: one NCCL communicator per handle; the per-iteration exchange (all-gather of returns + failure flags)
  // is enqueued on the engine stream right behind the rollout kernel
  ncclComm_t comm = nullptr;
  int nranks = 1, rank = 0;
  int totalN = 0, shard_lo = 0, shard_hi = 0;   // of the last sharded rollout
  DeviceArray<float> d_slot, d_gather, d_returns_all;
  DeviceArray<unsigned char> d_failure_all;
  DeviceArray<int> d_order_all;
  DeviceArray<float> d_bcast;
  size_t bcast_floats = 0;
  int maxTotal = 0;
  int nuserdata = 0;
  int differentiable = 0;   // MakeDifferentiable (utilities.cc:60-75) for the following launches (DevModel::differentiable)
  // measurement sensors (k_sensors): one table row per model sensor; sensor_why[i] is empty when sensor i is one the
  // device evaluates, else the reason it is not
  std::vector<DevSensor> sensors;
  std::vector<std::string> sensor_why;
  std::vector<int> sensor_geoms;   // the rangefinders' eligible geoms, uploaded right after the rows
  DeviceArray<DevSensor> d_sensors;
  // persistent scratch of step_impl: device buffer and its pinned host staging, grown on demand
  DeviceArray<float> d_step;
  PinnedArray<float> h_step;
  size_t step_words = 0;
  // model variants (set_model_variants): the model as created, which every variant is checked against; the variant
  // blocks [nvariants][variant_stride] floats in one allocation; and the variant each problem of the following launches
  // runs on, d_variant_index [nselected] (the identity over the variants unless select_model_variants chose others)
  DevModel M0;
  double timestep0 = 0;
  std::vector<float> f0;
  DeviceArray<float> d_variants;
  DeviceArray<int> d_variant_index;
  int nvariants = 0, variant_stride = 0, nselected = 0;
  // model ensemble (set_model_ensemble): the member blocks [nmembers][member_stride], laid out as the variant blocks;
  // the member of every launch problem, d_member_index [traj_factor x max_candidates] (problem j on member j % nmembers);
  // the members' returns and failure flags [B][K][N] of an ensemble launch.  The per-trajectory buffers hold
  // traj_factor x max_candidates trajectories (grown by set_model_ensemble, never shrunk).
  DeviceArray<float> d_members;
  DeviceArray<int> d_member_index;
  DeviceArray<float> d_member_returns;
  DeviceArray<unsigned char> d_member_failure;
  int nmembers = 0, member_stride = 0, worst = 0, traj_factor = 1;
  // the members of the resident and of the last launch (0: not an ensemble launch), and the last launch's N per problem
  int resident_members = 0, last_members = 0, last_nper = 0;
  // initial-state ensembles (rollout_spline_belief_batched): the covariances of the launch [cov_problems][n][n], the
  // joint table [3][njnt] (type, qposadr, dofadr), and d_belief [33 max_candidates]: each launch row's variant (up to
  // 32 rows per problem), then each problem's factorisation status
  DeviceArray<double> d_cov;
  int cov_problems = 0;
  DeviceArray<int> d_jnt;
  DeviceArray<int> d_belief;
  // resident-input launch description
  RolloutArgs resident;
  bool resident_ok = false;
  size_t smem_bytes(int P) const {
    DevLayout L = make_layout(pack.M, P);
    return ((size_t)smem_header_words(pack.M) + (size_t)L.total) * 4;
  }
  // the stream is idle here (mjpc_b200_destroy synchronised it; a failed create enqueued nothing on it), and the
  // owners free the memory after this
  ~mjpc_b200() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {

// the task floats of a pack: task_weight, task_norm_parameter, task_parameters and task_state lie back to back
size_t task_floats_begin(const DevModel& M) { return M.fo[F_task_weight]; }
size_t task_floats_count(const DevModel& M) { return M.fo[F_wrap_coef] - M.fo[F_task_weight]; }

int upload_task(mjpc_b200* h) {
  // weights / parameters / task_state live inside the model pack (float section), and inside every variant's block
  const DevModel& M = h->pack.M;
  std::vector<float>& f = h->pack.f;
  for (size_t i = 0; i < h->weight.size(); i++) f[M.fo[F_task_weight] + i] = (float)h->weight[i];
  for (size_t i = 0; i < h->parameters.size(); i++) f[M.fo[F_task_parameters] + i] = (float)h->parameters[i];
  for (size_t i = 0; i < h->task_state.size(); i++) f[M.fo[F_task_state] + i] = (float)h->task_state[i];
  h->pack.M.risk = (float)h->risk;
  CUDA_TRY(cudaMemcpyAsync(h->d_pack, f.data(), (size_t)(M.nf + M.ni) * 4, cudaMemcpyHostToDevice, h->stream));
  const size_t t0 = task_floats_begin(M), nt = task_floats_count(M);
  for (int v = 0; v < h->nvariants; v++)
    CUDA_TRY(cudaMemcpyAsync(h->d_variants + (size_t)v * h->variant_stride + t0, f.data() + t0, nt * 4,
                             cudaMemcpyHostToDevice, h->stream));
  for (int k = 0; k < h->nmembers; k++)
    CUDA_TRY(cudaMemcpyAsync(h->d_members + (size_t)k * h->member_stride + t0, f.data() + t0, nt * 4,
                             cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));  // f is pageable
  return 0;
}

// The model blocks a launch stages from, and their stride (pack_stride of the kernel arguments): the variants when
// set, else the one pack with stride 0
const float* launch_pack(const mjpc_b200* h) { return h->nvariants ? h->d_variants : h->d_pack; }
int launch_stride(const mjpc_b200* h) { return h->nvariants ? h->variant_stride : 0; }

// With model variants set, a launch that reads them holds one problem per selected variant; the calls without a
// problem index to choose a variant by (single-problem, sharded and step calls: B < 0 here) are refused.  0 otherwise.
int check_variants(const mjpc_b200* h, int B, const char* call) {
  if (!h->nvariants) return 0;
  if (B < 0)
    return fail(MJPC_B200_ERR_UNSUPPORTED, std::string(call) + ": not available while model variants are set " +
                                               "(set_model_variants); use the batched call");
  if (B != h->nselected)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": the launch has " + std::to_string(B) +
                                                " problems, the model variants are for " + std::to_string(h->nselected));
  return 0;
}

// With a model ensemble set, only the spline launches score on it: every other call that runs the model is refused
int check_ensemble(const mjpc_b200* h, const char* call) {
  if (!h->nmembers) return 0;
  return fail(MJPC_B200_ERR_UNSUPPORTED,
              std::string(call) + ": not available while a model ensemble is set (set_model_ensemble)");
}

// The measurement-sensor table of a blob: one row per model sensor; why[i] is empty when sensor i is one the device
// evaluates, else the reason it is not.  A blob without the sensor / site entries has no measurable sensors.
// ray_geoms gets the rangefinders' eligible-geom lists, which the device finds after the rows (DevSensor::geom0).
// opt_magnetic and geom_alpha are in the blob only when the model has a magnetometer or a rangefinder (MuJoCo's
// defaults otherwise: magnetic (0, -0.5, 0), every geom visible to rays).
void sensor_table(const Blob& b, std::vector<DevSensor>* sensors, std::vector<std::string>* why_out,
                  std::vector<int>* ray_geoms) {
  int dt, cnt; int64_t off;
  if (!b.find("nsensor", &dt, &cnt, &off) || !b.find("site_size", &dt, &cnt, &off)) return;
  const std::vector<int> ty = b.ints("sensor_type"), ot = b.ints("sensor_objtype"), oid = b.ints("sensor_objid"),
                         dim = b.ints("sensor_dim"), adr = b.ints("sensor_adr"), st = b.ints("site_type"),
                         jt = b.ints("jnt_type"), trntype = b.ints("actuator_trntype"),
                         trnid = b.ints("actuator_trnid");
  const std::vector<double> ss = b.reals("site_size");
  std::vector<double> cutoff(ty.size(), 0.0);
  if (b.find("sensor_cutoff", &dt, &cnt, &off)) cutoff = b.reals("sensor_cutoff");
  std::vector<double> magnetic = {0.0, -0.5, 0.0};
  if (b.find("opt_magnetic", &dt, &cnt, &off)) magnetic = b.reals("opt_magnetic");
  const std::vector<int> gtype = b.ints("geom_type"), gbody = b.ints("geom_bodyid"), sbody = b.ints("site_bodyid");
  std::vector<double> alpha(gtype.size(), 1.0);
  if (b.find("geom_alpha", &dt, &cnt, &off)) alpha = b.reals("geom_alpha");
  const int ns = b.i("nsensor");
  auto slide_or_hinge = [&](int j) { return jt[j] == JNT_SLIDE || jt[j] == JNT_HINGE; };
  for (int i = 0; i < ns; i++) {
    DevSensor S = {ty[i], ot[i], oid[i], adr[i], 0.f, {0.f, 0.f, 0.f}, 0, 0};
    std::string why;
    switch (ty[i]) {
      case SENS_JOINTPOS: case SENS_JOINTVEL:
        if (!slide_or_hinge(oid[i])) why = "jointpos / jointvel of a free or ball joint";
        break;
      case SENS_FRAMEPOS:
        if (ot[i] < OBJ_BODY || ot[i] > OBJ_SITE) why = "framepos of an unknown object type";
        break;
      case SENS_FRAMEQUAT: case SENS_FRAMEXAXIS: case SENS_FRAMEYAXIS: case SENS_FRAMEZAXIS: case SENS_FRAMELINVEL:
      case SENS_FRAMEANGVEL: case SENS_FRAMELINACC: case SENS_FRAMEANGACC:
        if (ot[i] < OBJ_BODY || ot[i] > OBJ_SITE) why = "frame sensor of an object other than a body, xbody, geom or site";
        break;
      case SENS_TOUCH:
        if (st[oid[i]] != GEOM_SPHERE) why = "touch zone other than a sphere site";
        S.radius = (float)ss[3 * oid[i]];
        break;
      case SENS_ACCELEROMETER: case SENS_VELOCIMETER: case SENS_GYRO:
        if (ot[i] != OBJ_SITE) why = "accelerometer / velocimeter / gyro of an object other than a site";
        break;
      case SENS_SUBTREECOM: case SENS_SUBTREELINVEL: case SENS_SUBTREEANGMOM:
        if (ot[i] != OBJ_BODY) why = "subtree sensor of an object other than a body";
        break;
      case SENS_BALLQUAT: case SENS_BALLANGVEL:
        if (jt[oid[i]] != JNT_BALL) why = "ballquat / ballangvel of a joint other than a ball joint";
        break;
      case SENS_JOINTACTUATORFRC:
        if (!slide_or_hinge(oid[i])) why = "jointactuatorfrc of a free or ball joint";
        break;
      case SENS_ACTUATORPOS: case SENS_ACTUATORVEL:
        // mjTRN_JOINT (0) on a slide or hinge joint, or mjTRN_TENDON (1): every tendon of the model is fixed
        if (!(trntype[oid[i]] == 1 || (trntype[oid[i]] == 0 && slide_or_hinge(trnid[oid[i]]))))
          why = "actuatorpos / actuatorvel of a transmission other than a slide or hinge joint or a fixed tendon";
        break;
      case SENS_ACTUATORFRC: case SENS_TENDONPOS: case SENS_TENDONVEL:
        break;
      case SENS_MAGNETOMETER:
        if (ot[i] != OBJ_SITE) why = "magnetometer of an object other than a site";
        for (int q = 0; q < 3; q++) S.field[q] = (float)magnetic[q];
        break;
      case SENS_RANGEFINDER: {
        if (ot[i] != OBJ_SITE) { why = "rangefinder of an object other than a site"; break; }
        // mj_ray's eligible geoms: not of the site's body, alpha not 0; every group, static geoms included
        S.geom0 = (int)ray_geoms->size();
        for (int g = 0; g < (int)gtype.size(); g++) {
          if (gbody[g] == sbody[oid[i]] || alpha[g] == 0.0) continue;
          if (gtype[g] != GEOM_PLANE && gtype[g] != GEOM_SPHERE && gtype[g] != GEOM_CAPSULE &&
              gtype[g] != GEOM_ELLIPSOID && gtype[g] != GEOM_CYLINDER && gtype[g] != GEOM_BOX) {
            why = "rangefinder: geom " + std::to_string(g) + " is of type " + std::to_string(gtype[g]) +
                  ", which rays are not cast against (only plane, sphere, capsule, ellipsoid, cylinder and box)";
            break;
          }
          ray_geoms->push_back(g);
        }
        S.ngeom = (int)ray_geoms->size() - S.geom0;
        break;
      }
      default:
        why = "sensor type " + std::to_string(ty[i]) +
              " (only jointpos, jointvel, framepos, framequat, framexaxis, frameyaxis, framezaxis, framelinvel, "
              "frameangvel, framelinacc, frameangacc, subtreecom, subtreelinvel, subtreeangmom, touch, accelerometer, "
              "velocimeter, gyro, magnetometer, rangefinder, ballquat, ballangvel, jointactuatorfrc, actuatorpos, "
              "actuatorvel, actuatorfrc, tendonpos and tendonvel are evaluated)";
    }
    if (why.empty() && dim[i] != sensor_dim(ty[i])) why = "unexpected sensor dimension";
    if (why.empty() && cutoff[i] != 0.0) why = "cutoff is not modelled";
    sensors->push_back(S);
    why_out->push_back(why);
  }
  // geom0 from the start of the list to the start of the row: the list follows the n rows
  const int row_words = (int)(sizeof(DevSensor) / sizeof(int));
  for (int i = 0; i < (int)sensors->size(); i++)
    if ((*sensors)[i].type == SENS_RANGEFINDER) (*sensors)[i].geom0 += ((int)sensors->size() - i) * row_words;
}

const char* const kFloatArrayNames[] = {
#define X(n) #n,
    MJPC_F_ARRAYS(X)
#undef X
};
const char* const kIntArrayNames[] = {
#define X(n) #n,
    MJPC_I_ARRAYS(X) MJPC_I_DERIVED(X)
#undef X
};

// set_model_variants' rule: the first field of variant V (packed, with its sensor table) that must equal the handle's
// model as created and does not, or "" when V may stand in for it.  Floats compare bitwise.
std::string variant_mismatch(const mjpc_b200* h, const ModelPack& V, const std::vector<DevSensor>& sensors,
                             const std::vector<std::string>& why, const std::vector<int>& geoms) {
  const DevModel &M = h->M0, &W = V.M;
#define X(n) if (W.n != M.n) return #n;
  MJPC_M_INTS(X)
#undef X
  for (int k = 0; k < F_COUNT; k++) if (W.fo[k] != M.fo[k]) return std::string("the layout of ") + kFloatArrayNames[k];
  for (int k = 0; k < I_COUNT; k++) if (W.io[k] != M.io[k]) return std::string("the layout of ") + kIntArrayNames[k];
  for (int k = 0; k < I_COUNT; k++) {
    const int a = M.io[k], e = k + 1 < I_COUNT ? M.io[k + 1] : M.ni;
    if (!std::equal(V.i.begin() + a, V.i.begin() + e, h->pack.i.begin() + a)) return kIntArrayNames[k];
  }
  auto same = [](const void* x, const void* y, size_t n) { return std::memcmp(x, y, n) == 0; };
  if (V.timestep != h->timestep0 || !same(&W.timestep, &M.timestep, 4)) return "timestep";
  if (!same(&W.impratio, &M.impratio, 4)) return "impratio";
  if (!same(&W.tolerance, &M.tolerance, 4)) return "tolerance";
  if (!same(&W.ls_tolerance, &M.ls_tolerance, 4)) return "ls_tolerance";
  if (!same(W.gravity, M.gravity, 12)) return "gravity";
  if (!same(&W.risk, &M.risk, 4)) return "task_risk";
  for (int k : {F_task_weight, F_task_norm_parameter, F_task_parameters, F_task_state, F_actuator_ctrlrange}) {
    const int a = M.fo[k], e = M.fo[k + 1];
    if (!same(V.f.data() + a, h->f0.data() + a, (size_t)(e - a) * 4)) return kFloatArrayNames[k];
  }
  if (sensors.size() != h->sensors.size()) return "the sensor table";
  for (size_t k = 0; k < sensors.size(); k++) {
    const DevSensor &x = sensors[k], &y = h->sensors[k];
    if (x.type != y.type || x.objtype != y.objtype || x.objid != y.objid || x.adr != y.adr ||
        !same(&x.radius, &y.radius, 4) || !same(x.field, y.field, 12) || x.geom0 != y.geom0 ||
        x.ngeom != y.ngeom || why[k] != h->sensor_why[k])
      return "sensor " + std::to_string(k);
  }
  if (geoms != h->sensor_geoms) return "the rangefinders' geoms";
  return "";
}

// The instance a launch runs from the handle's row, and what mjpc_b200_last_kernel_static reports for it (0 generic,
// 1 static, 2 static one-warp rollout).  Read per launch, so that tests and profiles can switch them on a live engine:
// MJPC_B200_NO_STATIC=1 forces the generic row, MJPC_B200_SHAPE=plain the one-warp rollout.
int pick_kernels(const mjpc_b200* h, const KernelSet** k) {
  const char* ns = std::getenv("MJPC_B200_NO_STATIC");
  const char* sh = std::getenv("MJPC_B200_SHAPE");
  if (h->kernels == &kGenericKernels || (ns && ns[0] == '1')) { *k = &kGenericKernels; return 0; }
  *k = h->kernels;
  return sh && sh[0] == 'p' && sh[1] == 'l' ? 2 : 1;
}

// src (NULL: the handle's task state) as floats, with its time-like entries made relative to t0.  The Quadruped's gait
// phase start is an absolute phase that grows at 2 pi cadence per second, so it is folded to t0 as well: the phase at
// t0 in double, less whole periods, and phase start time 0.  Periods come off only while the phase stays >= 2 pi: the
// gait's fmod(phase + pi - footphase, 2 pi) keeps the sign of its argument, which is negative early in an episode
// (phase < footphase - pi), and a phase of at least 2 pi keeps it positive.
void rebase_task_state(const mjpc_b200* h, const double* src, double t0, float* dst) {
  if (!src) src = h->task_state.data();
  for (int i = 0; i < h->pack.M.task_state_size; i++) {
    double v = src[i];
    if (std::find(h->time_idx.begin(), h->time_idx.end(), i) != h->time_idx.end()) v -= t0;
    dst[i] = (float)v;
  }
  if (h->pack.M.residual_id == RESIDUAL_QUADRUPED_FLAT) {
    const double period = 2 * M_PI;
    const double phase = src[QS_PHASE_START] + (t0 - src[QS_PHASE_START_TIME]) * src[QS_PHASE_VELOCITY];
    const double k = std::max(0.0, std::floor(phase / period) - 1);
    dst[QS_PHASE_START] = (float)(phase - k * period);
    dst[QS_PHASE_START_TIME] = 0.f;
  }
}

// floats of the per-problem block of stage_problems for B problems, P knots and H steps (knots excluded)
size_t problem_floats(const DevModel& M, int B, int P, int H) {
  return (size_t)B * (4 * (size_t)H + M.nq + M.nv + 7 * M.nmocap + M.task_state_size + M.num_term + M.num_parameters + P + 1);
}

// The policy step table of one problem (PolicyInterval, dev_task.cuh): T[0] = time0, T[t+1] = T[t] + timestep in double,
// and for each step the upper_bound of T[t] over the `count` absolute node times, with the interval fraction in double.
void build_policy_intervals(const double* nodes, int count, double time0, double timestep, int H, PolicyInterval* out) {
  double time = time0;
  for (int t = 0; t < H; t++) {
    const int upper = (int)(std::upper_bound(nodes, nodes + count, time) - nodes);
    double frac = 0;
    if (upper > 0 && upper < count) frac = (time - nodes[upper - 1]) / (nodes[upper] - nodes[upper - 1]);
    out[t].time = time; out[t].upper = upper; out[t].frac = (float)frac;
    time += timestep;
  }
}

// Stage the inputs of a rollout launch of B problems back to back in the pinned buffer and upload them with ONE copy
// into d_in; point A's per-problem inputs at them.  Layout (floats):
//   [step table B x H x 4][state B x ds][mocap B x 7 nmocap][task_state B x size][weight B x num_term, if given]
//   [parameters B x num_parameters, if given][knot_times B x P][knots B x N x P x nu]   (knot blocks: spline launches)
//   [noise keys B, if set_xfrc_noise_batched set them]
// The step table of problem b is built from its start time times[b] and its `count` absolute policy nodes nodes[b]
// (the knot times of a spline launch, the nominal times of a feedback launch).  A NULL task_states / weights /
// parameters stands for the handle's set_task values; the time-like task-state entries and the knot times are made
// relative to each problem's own start time.  *end: the first h_in float after the block.  Per-problem noise keys for
// another number of problems are refused before anything is staged.  R > 1 (a model ensemble of R members) stages
// each problem R times: launch problem b R + k holds problem b's inputs.
int stage_problems(mjpc_b200* h, int B, const float* states, const double* times, const float* mocaps,
                   const double* weights, const double* parameters, const double* task_states, const double* nodes,
                   int count, int H, const float* knots, int N, RolloutArgs* A, size_t* end, int R = 1) {
  if (int rc = check_variants(h, B, "rollout")) return rc;
  if (!h->noise_seeds.empty() && (int)h->noise_seeds.size() != B)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout: set_xfrc_noise_batched gave keys for " +
                                                std::to_string(h->noise_seeds.size()) + " problems, the launch has " +
                                                std::to_string(B));
  const DevModel& M = h->pack.M;
  const size_t ds = M.nq + M.nv, nm = 7 * (size_t)M.nmocap, nts = M.task_state_size, nw = M.num_term,
               np = M.num_parameters, nk = (size_t)N * count * M.nu;
  const int BR = B * R;
  float* in = h->h_in;
  PolicyInterval* iv = reinterpret_cast<PolicyInterval*>(in);
  for (int j = 0; j < BR; j++)
    build_policy_intervals(nodes + (size_t)(j / R) * count, count, times[j / R], h->pack.timestep, H, iv + (size_t)j * H);
  size_t o = 4 * (size_t)BR * H;
  const size_t o_state = o;
  for (int j = 0; j < BR; j++, o += ds) std::memcpy(in + o, states + (j / R) * ds, ds * 4);
  const size_t o_mocap = o;
  if (nm) for (int j = 0; j < BR; j++, o += nm) std::memcpy(in + o, mocaps + (j / R) * nm, nm * 4);
  const size_t o_ts = o;
  for (int j = 0; j < BR; j++, o += nts)
    rebase_task_state(h, task_states ? task_states + (j / R) * nts : nullptr, times[j / R], in + o);
  const size_t o_w = o;
  if (weights) for (int j = 0; j < BR; j++) for (size_t i = 0; i < nw; i++) in[o++] = (float)weights[(j / R) * nw + i];
  const size_t o_p = o;
  if (parameters)
    for (int j = 0; j < BR; j++) for (size_t i = 0; i < np; i++) in[o++] = (float)parameters[(j / R) * np + i];
  const size_t o_kt = o;
  if (knots) {
    for (int j = 0; j < BR; j++)
      for (int k = 0; k < count; k++) in[o++] = (float)(nodes[(size_t)(j / R) * count + k] - times[j / R]);
  }
  const size_t o_k = o;
  if (knots) for (int j = 0; j < BR; j++, o += nk) std::memcpy(in + o, knots + (j / R) * nk, nk * 4);
  const size_t o_seed = o;
  if (!h->noise_seeds.empty()) { std::memcpy(in + o, h->noise_seeds.data(), (size_t)B * 4); o += B; }
  CUDA_TRY(cudaMemcpyAsync(h->d_in, in, o * 4, cudaMemcpyHostToDevice, h->stream));
  float* d = h->d_in;
  A->nprob = BR; A->nper = N;
  A->iv = reinterpret_cast<const PolicyInterval*>(d);
  A->timestep = h->pack.timestep;
  A->state = d + o_state; A->mocap = d + o_mocap; A->task_state = d + o_ts;
  A->weight = weights ? d + o_w : nullptr; A->parameters = parameters ? d + o_p : nullptr;
  A->knot_times = knots ? d + o_kt : nullptr; A->knots = knots ? d + o_k : nullptr;
  A->noise_seeds = h->noise_seeds.empty() ? nullptr : reinterpret_cast<const unsigned*>(d + o_seed);
  *end = o;
  return 0;
}

// grow the pinned staging buffer to at least `floats` (never shrinks); on failure the old buffer stays
int reserve_h_in(mjpc_b200* h, size_t floats) {
  if (floats <= h->h_in_floats) return 0;
  PinnedArray<float> p;
  CUDA_TRY(p.alloc(floats));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // earlier copies may still read the old buffer
  h->h_in = std::move(p); h->h_in_floats = floats;
  return 0;
}

// grow the feedback-policy buffers to B problems (never shrinks); on failure the old buffers stay
int reserve_feedback(mjpc_b200* h, int B) {
  if (B <= h->fb_nprob) return 0;
  const DevModel& M = h->pack.M;
  const size_t H = h->maxH, ds = M.nq + M.nv, n = 2 * M.nv, nu = M.nu, P = B;
  DeviceArray<float> unom, xnom, tnom, gains, du;
  if (unom.alloc(P * H * nu) || xnom.alloc(P * H * ds) || tnom.alloc(P * H) || gains.alloc(P * H * nu * n) ||
      du.alloc(P * H * nu))
    return fail(MJPC_B200_ERR_CUDA, "rollout_feedback_batched: out of device memory for the feedback policies");
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  h->d_unom = std::move(unom); h->d_xnom = std::move(xnom); h->d_tnom = std::move(tnom);
  h->d_gains = std::move(gains); h->d_du = std::move(du);
  h->fb_nprob = B;
  return 0;
}

// The rollout launch A, then the ranking of its candidates.  K > 0: A holds B x K x N trajectories of a model ensemble
// or an initial-state ensemble (stage_problems with R = K) and writes the member returns; ensemble_score_kernel scores
// the B x N candidates with the mean of the `worst` largest (worst < 1: the model ensemble's) into d_returns /
// d_failure, which are ranked.
int launch_rollout(mjpc_b200* h, const RolloutArgs& A_in, int K = 0, int worst = 0) {
  RolloutArgs A = A_in;
  const size_t smem = h->smem_bytes(A.P);
  CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
  // co-resident pair synchronisation: only when at most two candidates can ever be resident per SM and all are resident
  // at once (one wave); MJPC_B200_PAIR_SYNC=0 switches it off (profiling)
  {
    const char* ps = std::getenv("MJPC_B200_PAIR_SYNC");
    const bool on = !(ps && ps[0] == '0') && A.N > h->num_sms && A.N <= 2 * h->num_sms;
    A.pair_sync = on ? h->d_pair_sync.get() : nullptr;
    if (on) CUDA_TRY(cudaMemsetAsync(h->d_pair_sync, 0, (size_t)256 * 32 * sizeof(unsigned), h->stream));
  }
  // one candidate per CTA, whichever instance; the static ones share the generic one's arguments and shared-memory image
  const KernelSet* k;
  h->last_static = pick_kernels(h, &k);
  const bool plain = h->last_static == 2;
  launch_kernel(plain ? k->rollout_plain : k->rollout, A.N, plain ? 32 : k->rollout_threads, smem, h->stream, A);
  if (K) {
    const int B = A.nprob / K, n = B * A.nper;
    ensemble_score_kernel<<<(n + 7) / 8, 256, 0, h->stream>>>(A.returns, A.failure, B, K, A.nper,
                                                              worst > 0 ? worst : h->worst, h->d_returns, h->d_failure);
    rank_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_returns, A.nper, B, h->d_order);
  } else {
    rank_kernel<<<(A.N + 255) / 256, 256, 0, h->stream>>>(A.returns, A.nper, A.nprob, h->d_order);
  }
  CUDA_TRY(cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(cudaGetLastError());
  h->launches += K ? 3 : 2;
  h->lastN = K ? A.N / K : A.N; h->lastH = A.H;
  h->last_members = K; h->last_nper = A.nper;
  return 0;
}

RolloutArgs base_args(mjpc_b200* h, int N, int H) {
  RolloutArgs A;
  std::memset(&A, 0, sizeof(A));
  A.M = h->pack.M;
  A.pack = launch_pack(h); A.pack_stride = launch_stride(h); A.pack_index = h->d_variant_index;
  A.N = N; A.H = H;
  A.states = h->d_states; A.actions = h->d_actions; A.times = h->d_times; A.residual = h->d_residual;
  A.costs = h->d_costs; A.trace = h->d_trace; A.returns = h->d_returns; A.failure = h->d_failure;
  A.stats = h->d_stats;
  A.xfrc_std = h->xfrc_std; A.xfrc_rate = h->xfrc_rate; A.noise_seed = h->noise_seed;
  return A;
}

int read_back(mjpc_b200* h, int N, float* returns, uint8_t* failure, int* order) {
  float* hr = (float*)h->h_out.get();
  int* ho = (int*)(h->h_out + (size_t)N * 4);
  unsigned char* hf = h->h_out + (size_t)N * 8;
  CUDA_TRY(cudaMemcpyAsync(hr, h->d_returns, (size_t)N * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(ho, h->d_order, (size_t)N * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(hf, h->d_failure, (size_t)N, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  if (returns) std::memcpy(returns, hr, (size_t)N * 4);
  if (order) std::memcpy(order, ho, (size_t)N * 4);
  if (failure) std::memcpy(failure, hf, (size_t)N);
  return 0;
}

// ---- NCCL, bound at run time (dlopen): a process that already loaded an NCCL (PyTorch's) shares it by SONAME
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi& nccl_api() {
  static NcclApi api;
  if (api.lib) return api;
  api.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!api.lib) api.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!api.lib) return api;
#define BIND(field, name) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.lib, name))
  BIND(GetUniqueId, "ncclGetUniqueId"); BIND(CommInitRank, "ncclCommInitRank"); BIND(CommDestroy, "ncclCommDestroy");
  BIND(AllGather, "ncclAllGather"); BIND(Broadcast, "ncclBroadcast"); BIND(GetErrorString, "ncclGetErrorString");
#undef BIND
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Broadcast && api.GetErrorString;
  return api;
}
#define NCCL_TRY(expr)                                                                                     \
  do {                                                                                                     \
    ncclResult_t r_ = (expr);                                                                              \
    if (r_ != ncclSuccess)                                                                                 \
      return fail(MJPC_B200_ERR_CUDA, std::string(#expr) + ": " + nccl_api().GetErrorString(r_));          \
  } while (0)

// contiguous balanced candidate ranges (SURVEY.md 8e): the first N % G ranks own one candidate more
inline void shard_range(int N, int G, int r, int* lo, int* hi) {
  const int base = N / G, rem = N % G;
  *lo = r * base + std::min(r, rem);
  *hi = *lo + base + (r < rem ? 1 : 0);
}

// gathered [G][width][2] (return, failure flag) -> compact returns[N], failure[N] in global candidate order
__global__ void compact_gather_kernel(const float* __restrict__ gathered, int N, int G, int width, float* __restrict__ ret,
                                      unsigned char* __restrict__ failure) {
  const int base = N / G, rem = N % G;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    // owner of global candidate i under shard_range
    int r = i < rem * (base + 1) ? i / (base + 1) : rem + (base ? (i - rem * (base + 1)) / base : 0);
    const int lo = r * base + min(r, rem);
    const float* src = gathered + ((size_t)r * width + (i - lo)) * 2;
    ret[i] = src[0];
    failure[i] = src[1] != 0.f ? 1 : 0;
  }
}
__global__ void pack_slot_kernel(const float* __restrict__ ret, const unsigned char* __restrict__ failure, int n, int width,
                                 float* __restrict__ slot) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < width; i += gridDim.x * blockDim.x) {
    slot[2 * i] = i < n ? ret[i] : 3.0e38f;
    slot[2 * i + 1] = i < n ? (float)failure[i] : 1.f;
  }
}

}  // namespace

extern "C" {

const char* mjpc_b200_version(void) { return "mjpc_b200 0.1.0 (sm_90a)"; }
const char* mjpc_b200_last_error(void) { return g_last_error.c_str(); }

int mjpc_b200_create(const mjpc_model_blob* model, int max_candidates, int max_horizon, int device,
                     mjpc_b200_t** out) {
  if (!model || !model->data || !out || max_candidates < 1 || max_horizon < 1)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "create: bad argument");
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(MJPC_B200_ERR_CUDA, "no CUDA device: the engine has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "create: bad device ordinal");
  // the handle is built here and released to the caller only when complete; a refusal frees whatever it holds
  std::unique_ptr<mjpc_b200> h(new mjpc_b200);
  try {
    int maxcon = 32, maxefc = 96;
    h->pack = pack_model(model->data, model->nbytes, maxcon, maxefc);
  } catch (const std::exception& e) {
    return fail(MJPC_B200_ERR_BAD_BLOB, std::string("create: ") + e.what());
  }
  h->device = device;
  h->maxN = max_candidates; h->maxH = max_horizon;
  const DevModel& M = h->pack.M;
  {
    Blob b(model->data, model->nbytes);
    h->nuserdata = b.i("nuserdata");
    if (h->nuserdata != 0) return fail(MJPC_B200_ERR_UNSUPPORTED, "create: mjData::userdata (nuserdata > 0) is not supported");
    h->weight = b.reals("task_weight"); h->parameters = b.reals("task_parameters");
    h->task_state = b.reals("task_state"); h->risk = b.r("task_risk");
    for (int d : b.ints("task_dim_norm_residual")) h->max_term_dim = std::max(h->max_term_dim, d);
  }
  h->time_idx = time_like_state(M.residual_id);
  sensor_table(Blob(model->data, model->nbytes), &h->sensors, &h->sensor_why, &h->sensor_geoms);
  h->M0 = M; h->timestep0 = h->pack.timestep; h->f0 = h->pack.f;
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreate(&h->ev0));
  CUDA_TRY(cudaEventCreate(&h->ev1));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  h->num_sms = prop.multiProcessorCount;
  h->smem_optin = prop.sharedMemPerBlockOptin;
  const size_t smem_need = h->smem_bytes(h->maxP);
  if (smem_need > (size_t)prop.sharedMemPerBlockOptin)
    return fail(MJPC_B200_ERR_CAPACITY, "model does not fit in shared memory");
  // pack: floats then ints, one buffer (single TMA bulk copy per CTA)
  {
    std::vector<float>& f = h->pack.f;
    const size_t nf = f.size();
    f.resize(nf + h->pack.i.size());
    std::memcpy(f.data() + nf, h->pack.i.data(), h->pack.i.size() * 4);
    // not staged to shared memory: keyframe mocap positions, read from HBM by the tracking residual (Ctx::gkey)
    for (double x : h->pack.key_mpos) f.push_back((float)x);
    CUDA_TRY(h->d_pack.alloc(f.size()));
    CUDA_TRY(cudaMemcpy(h->d_pack, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
  }
  const size_t N = max_candidates, H = max_horizon, ds = M.nq + M.nv, n = 2 * M.nv, nu = M.nu, nr = M.num_residual;
  // launch inputs: up to max_candidates problems of one candidate each (stage_problems)
  const size_t in_floats = problem_floats(M, max_candidates, h->maxP, max_horizon) + N * h->maxP * nu;
  CUDA_TRY(h->d_in.alloc(in_floats));
  CUDA_TRY(h->d_unom.alloc(H * nu)); CUDA_TRY(h->d_xnom.alloc(H * ds)); CUDA_TRY(h->d_tnom.alloc(H));
  CUDA_TRY(h->d_gains.alloc(H * nu * n)); CUDA_TRY(h->d_du.alloc(H * nu)); CUDA_TRY(h->d_steps.alloc(N));
  CUDA_TRY(h->d_states.alloc(N * H * ds)); CUDA_TRY(h->d_actions.alloc(N * H * nu));
  CUDA_TRY(h->d_times.alloc(N * H)); CUDA_TRY(h->d_residual.alloc(N * H * nr));
  CUDA_TRY(h->d_costs.alloc(N * H)); CUDA_TRY(h->d_trace.alloc(N * H * 3 * (size_t)M.num_trace));
  CUDA_TRY(h->d_returns.alloc(N)); CUDA_TRY(h->d_failure.alloc(N)); CUDA_TRY(h->d_order.alloc(N)); CUDA_TRY(h->d_stats.alloc(12 * N));
  CUDA_TRY(h->d_pair_sync.alloc((size_t)256 * 32));
  {
    // the rows, then the rangefinders' geom lists (DevSensor::geom0)
    const size_t rows = h->sensors.size() * sizeof(DevSensor), list = h->sensor_geoms.size() * sizeof(int);
    CUDA_TRY(h->d_sensors.alloc(h->sensors.size() + (list + sizeof(DevSensor) - 1) / sizeof(DevSensor)));
    if (rows) CUDA_TRY(cudaMemcpy(h->d_sensors, h->sensors.data(), rows, cudaMemcpyHostToDevice));
    if (list)
      CUDA_TRY(cudaMemcpy(reinterpret_cast<char*>(h->d_sensors.get()) + rows, h->sensor_geoms.data(), list,
                          cudaMemcpyHostToDevice));
  }
  h->h_in_floats = in_floats + H * (nu + ds + 1 + nu * n + nu) + N + 64;
  CUDA_TRY(h->h_in.alloc(h->h_in_floats));
  h->h_out_bytes = N * 16 + 64;
  CUDA_TRY(h->h_out.alloc(h->h_out_bytes));
  const DevLayout L1 = make_layout(M, 1);
  const int* dof_parent = h->pack.i.data() + M.io[I_dof_parentid];
  if (spec_matches<SpecQuadruped>(M, L1, dof_parent)) h->kernels = &kQuadrupedKernels;
  else if (spec_matches<SpecHumanoidTrack>(M, L1, dof_parent)) h->kernels = &kHumanoidTrackKernels;
  // the dynamic shared-memory opt-in is per kernel and process-wide (raise_smem_limit only ever raises it: several
  // handles may coexist); a launch may fall back to the generic row (pick_kernels), so both rows get theirs
  const size_t smem_rollout = h->smem_bytes(h->maxP), smem_step = h->smem_bytes(1);
  for (const KernelSet* k : {h->kernels, &kGenericKernels}) {
    CUDA_TRY(raise_smem_limit(k->rollout, smem_rollout)); CUDA_TRY(raise_smem_limit(k->rollout_plain, smem_rollout));
    CUDA_TRY(raise_smem_limit(k->step, smem_step)); CUDA_TRY(raise_smem_limit(k->fd_center, smem_step));
    CUDA_TRY(raise_smem_limit(k->fd_column, smem_step)); CUDA_TRY(raise_smem_limit(k->plant, smem_step));
  }
  if (int rc = ilqg_init(h->ilqg, h->pack.M, (int)H)) return fail(rc, "ilqg buffer allocation failed");
  *out = h.release();
  return MJPC_B200_OK;
}

void mjpc_b200_destroy(mjpc_b200_t* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->comm && nccl_api().ok) nccl_api().CommDestroy(h->comm);
  delete h;
}

int mjpc_b200_get_info(const mjpc_b200_t* h, mjpc_b200_info* info) {
  if (!h || !info) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "get_info: null");
  const DevModel& M = h->pack.M;
  info->nq = M.nq; info->nv = M.nv; info->nu = M.nu; info->na = 0 /* na > 0 is rejected by create() */; info->nmocap = M.nmocap; info->nuserdata = h->nuserdata;
  info->dim_state = M.nq + M.nv; info->dim_dstate = 2 * M.nv;
  info->num_residual = M.num_residual; info->num_term = M.num_term; info->num_trace = M.num_trace;
  info->num_parameters = M.num_parameters; info->task_state_size = M.task_state_size;
  info->max_candidates = h->maxN; info->max_horizon = h->maxH; info->device = h->device;
  info->smem_bytes_per_warp = make_layout(M, 3).total * 4;
  return 0;
}

int mjpc_b200_set_task(mjpc_b200_t* h, const mjpc_task_desc* task) {
  if (!h || !task) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_task: null");
  CUDA_TRY(cudaSetDevice(h->device));
  if (task->weight) h->weight.assign(task->weight, task->weight + h->weight.size());
  if (task->parameters) h->parameters.assign(task->parameters, task->parameters + h->parameters.size());
  if (task->task_state) h->task_state.assign(task->task_state, task->task_state + h->task_state.size());
  h->risk = task->risk;
  return upload_task(h);
}

// Agent::PlanIteration's planning-model overrides (agent.cc:288-289): model_->opt.timestep = agent_timestep,
// model_->opt.integrator = agent_integrator.  The timestep is a live header option (no re-upload); only the Euler
// integrator (mjINT_EULER = 0) is implemented on the device - anything else is refused, never silently replaced.
int mjpc_b200_set_options(mjpc_b200_t* h, double timestep, int integrator) {
  if (!h || !(timestep > 0)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_options: bad argument");
  if (integrator != 0) return fail(MJPC_B200_ERR_UNSUPPORTED, "set_options: only the Euler integrator (0) is implemented");
  h->pack.timestep = timestep;
  h->pack.M.timestep = (float)timestep;
  return 0;
}

// Agent::PlanIteration's MakeDifferentiable (agent.cc:296-309, utilities.cc:60-75): while on, every joint's and geom's
// solimp[0] reads as 0 in the kernels (contact pairs take their solimp from the geoms here); off restores the model's own
// values (agent.cc:346-356).  Gradient-based planners (iLQG, iLQS, Gradient) plan with it on by default.
int mjpc_b200_set_differentiable(mjpc_b200_t* h, int on) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_differentiable: null");
  h->differentiable = on ? 1 : 0;
  h->pack.M.differentiable = on ? 1.f : 0.f;   // a header option: every launch copies the live header, no re-upload
  return 0;
}

// set_model_variants' and set_model_ensemble's blocks: each of the count blobs validated against the handle's model as
// created (variant_mismatch; an error names `call`, the `what` and its index), then laid out as one host image of
// count blocks of *stride floats.  Nothing is changed on a refusal.
static int model_blocks(mjpc_b200_t* h, const mjpc_model_blob* models, int count, const char* call, const char* what,
                        std::vector<float>* image, size_t* stride_out) {
  const DevModel& M = h->M0;
  size_t stride = 0;
  std::vector<ModelPack> packs(count);
  for (int v = 0; v < count; v++) {
    const std::string at = std::string(call) + ": " + what + " " + std::to_string(v) + ": ";
    if (!models[v].data) return fail(MJPC_B200_ERR_BAD_ARGUMENT, at + "NULL blob");
    std::vector<DevSensor> sensors;
    std::vector<std::string> why;
    std::vector<int> geoms;
    try {
      packs[v] = pack_model(models[v].data, models[v].nbytes, M.maxcon - 2 * M.ntendon, M.maxefc);
      Blob b(models[v].data, models[v].nbytes);
      if (b.i("nuserdata") != 0)
        return fail(MJPC_B200_ERR_UNSUPPORTED, at + "mjData::userdata (nuserdata > 0) is not supported");
      sensor_table(b, &sensors, &why, &geoms);
    } catch (const std::exception& e) {
      return fail(MJPC_B200_ERR_BAD_BLOB, at + e.what());
    }
    const std::string field = variant_mismatch(h, packs[v], sensors, why, geoms);
    if (!field.empty()) return fail(MJPC_B200_ERR_BAD_ARGUMENT, at + field + " differs from the handle's model");
    stride = std::max(stride, (size_t)(M.nf + M.ni) + packs[v].key_mpos.size() + 1);
  }
  stride = (stride + 31) & ~(size_t)31;   // 128-byte aligned blocks (the TMA copy needs 16)
  std::vector<float>& blocks = *image;
  blocks.assign((size_t)count * stride, 0.f);
  const size_t t0 = task_floats_begin(M), nt = task_floats_count(M);
  for (int v = 0; v < count; v++) {
    float* o = blocks.data() + (size_t)v * stride;
    const ModelPack& P = packs[v];
    std::copy(P.f.begin(), P.f.end(), o);
    std::copy(h->pack.f.begin() + t0, h->pack.f.begin() + t0 + nt, o + t0);   // the live task (set_task)
    std::memcpy(o + M.nf, P.i.data(), P.i.size() * 4);
    for (size_t k = 0; k < P.key_mpos.size(); k++) o[M.nf + M.ni + k] = (float)P.key_mpos[k];
    o[stride - 1] = P.M.meaninertia;
  }
  *stride_out = stride;
  return 0;
}

// device copies of a host block image and of a member / variant index
static cudaError_t upload_blocks(const std::vector<float>& blocks, const std::vector<int>& index, DeviceArray<float>* d,
                                 DeviceArray<int>* di) {
  cudaError_t e = d->alloc(blocks.size());
  if (e == cudaSuccess) e = di->alloc(index.size());
  if (e == cudaSuccess) e = cudaMemcpy(*d, blocks.data(), blocks.size() * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(*di, index.data(), index.size() * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) cudaGetLastError();
  return e;
}

// Per-problem model variants: validate every blob against the handle's model as created (variant_mismatch), then
// upload them into one allocation, variant v's block at d_variants + v * variant_stride:
//   [its nf floats, with the handle's live task floats][its ni ints][its keyframe table (Ctx::gkey)][pad][meaninertia]
// The blocks are what a handle created from the variant uploads as d_pack, so problem b of a launch computes what such
// a handle computes.  count = 0 (or NULL) clears them.  Nothing is changed on a refusal.
int mjpc_b200_set_model_variants(mjpc_b200_t* h, const mjpc_model_blob* models, int count) {
  if (!h || count < 0 || (count > 0 && !models)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_model_variants: bad argument");
  if (count > h->maxN)
    return fail(MJPC_B200_ERR_CAPACITY, "set_model_variants: more variants than max_candidates problems");
  if (count > 0)
    if (int rc = check_ensemble(h, "set_model_variants")) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  std::vector<float> blocks;
  size_t stride = 0;
  if (int rc = model_blocks(h, models, count, "set_model_variants", "variant", &blocks, &stride)) return rc;
  DeviceArray<float> d;
  DeviceArray<int> di;
  if (count) {
    std::vector<int> identity(h->maxN);
    for (int v = 0; v < h->maxN; v++) identity[v] = v < count ? v : 0;
    if (cudaError_t e = upload_blocks(blocks, identity, &d, &di))
      return fail(MJPC_B200_ERR_CUDA, std::string("set_model_variants: ") + cudaGetErrorString(e));
  }
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // launches in flight may still read the old blocks
  h->d_variants = std::move(d); h->d_variant_index = std::move(di);
  h->nvariants = count; h->nselected = count; h->variant_stride = (int)stride;
  h->resident_ok = false;
  return 0;
}

// The variant each problem of the following launches runs on: problem j on variant index[j] (NULL: the identity over
// all variants), and those launches hold exactly B problems.  Without variants set there is nothing to select.
int mjpc_b200_select_model_variants(mjpc_b200_t* h, const int* index, int B) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "select_model_variants: null");
  if (!h->nvariants) return 0;
  if (!index) B = h->nvariants;
  if (B < 1 || B > h->maxN) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "select_model_variants: bad B");
  std::vector<int> sel(B);
  for (int j = 0; j < B; j++) {
    sel[j] = index ? index[j] : j;
    if (sel[j] < 0 || sel[j] >= h->nvariants)
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "select_model_variants: variant index outside [0, count)");
  }
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(h->d_variant_index, sel.data(), (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // sel is pageable
  h->nselected = B;
  h->resident_ok = false;
  return 0;
}

// Grow the per-trajectory buffers (outputs, member returns, launch inputs and their pinned staging) to K x max_candidates
// trajectories, for the launches of a K-member ensemble; never shrinks.  On an allocation failure the handle keeps its
// buffers.
static int reserve_members(mjpc_b200_t* h, int K) {
  if (K <= h->traj_factor && h->d_member_returns) return 0;
  K = std::max(K, h->traj_factor);
  const DevModel& M = h->pack.M;
  const size_t N = (size_t)K * h->maxN, H = h->maxH, ds = M.nq + M.nv, nu = M.nu, nr = M.num_residual,
               ntr = 3 * (size_t)M.num_trace;
  const size_t in_floats = problem_floats(M, (int)N, h->maxP, h->maxH) + N * h->maxP * nu;
  DeviceArray<float> states, actions, residual, costs, trace, mret, din;
  DeviceArray<double> times;
  DeviceArray<long long> stats;
  DeviceArray<unsigned char> mfail;
  PinnedArray<float> hin;
  const bool grow_h_in = in_floats + 64 > h->h_in_floats;
  cudaError_t e = states.alloc(N * H * ds);
  if (e == cudaSuccess) e = actions.alloc(N * H * nu);
  if (e == cudaSuccess) e = times.alloc(N * H);
  if (e == cudaSuccess) e = residual.alloc(N * H * nr);
  if (e == cudaSuccess) e = costs.alloc(N * H);
  if (e == cudaSuccess) e = trace.alloc(N * H * ntr);
  if (e == cudaSuccess) e = stats.alloc(12 * N);
  if (e == cudaSuccess) e = mret.alloc(N);
  if (e == cudaSuccess) e = mfail.alloc(N);
  if (e == cudaSuccess) e = din.alloc(in_floats);
  if (e == cudaSuccess && grow_h_in) e = hin.alloc(in_floats + 64);
  if (e != cudaSuccess) return fail(MJPC_B200_ERR_CUDA, std::string("set_model_ensemble: ") + cudaGetErrorString(e));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // launches and copies in flight may still use the old buffers
  h->d_states = std::move(states); h->d_actions = std::move(actions); h->d_times = std::move(times);
  h->d_residual = std::move(residual); h->d_costs = std::move(costs); h->d_trace = std::move(trace);
  h->d_stats = std::move(stats); h->d_member_returns = std::move(mret); h->d_member_failure = std::move(mfail);
  h->d_in = std::move(din);
  if (grow_h_in) { h->h_in = std::move(hin); h->h_in_floats = in_floats + 64; }
  h->traj_factor = K;
  h->resident_ok = false;
  h->lastN = 0;   // the last launch's trajectories are gone
  return 0;
}

// A model ensemble: every spline launch rolls each candidate out on the K members and scores it (launch_rollout).  The
// members are validated and laid out as variants are (model_blocks); launch problem j runs on member j % K.
int mjpc_b200_set_model_ensemble(mjpc_b200_t* h, const mjpc_model_blob* models, int K, int worst) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_model_ensemble: null handle");
  if (K < 0 || K > 32) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_model_ensemble: K must be in [1, 32] (0 clears)");
  if (K == 0 || !models) {
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    h->d_members.reset(); h->d_member_index.reset();
    h->nmembers = 0; h->member_stride = 0; h->worst = 0;
    h->resident_ok = false;
    return 0;
  }
  if (worst < 1 || worst > K) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_model_ensemble: worst must be in [1, K]");
  if (h->nvariants)
    return fail(MJPC_B200_ERR_UNSUPPORTED,
                "set_model_ensemble: not available while model variants are set (set_model_variants)");
  CUDA_TRY(cudaSetDevice(h->device));
  std::vector<float> blocks;
  size_t stride = 0;
  if (int rc = model_blocks(h, models, K, "set_model_ensemble", "member", &blocks, &stride)) return rc;
  if (int rc = reserve_members(h, K)) return rc;
  std::vector<int> index((size_t)h->traj_factor * h->maxN);
  for (size_t j = 0; j < index.size(); j++) index[j] = (int)(j % K);
  DeviceArray<float> d;
  DeviceArray<int> di;
  if (cudaError_t e = upload_blocks(blocks, index, &d, &di))
    return fail(MJPC_B200_ERR_CUDA, std::string("set_model_ensemble: ") + cudaGetErrorString(e));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // launches in flight may still read the old blocks
  h->d_members = std::move(d); h->d_member_index = std::move(di);
  h->nmembers = K; h->member_stride = (int)stride; h->worst = worst;
  h->resident_ok = false;
  return 0;
}

// Validate and upload a spline launch of B problems x N candidates; it becomes the resident launch.  B = 1 is the
// single-problem call.  Nothing is changed on a refusal, so the handle stays usable.
static int upload_spline(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                         const double* weights, const double* parameters, const double* task_states, const float* knots,
                         const double* knot_times, int interp, int P, int N, int H) {
  const DevModel& M = h->pack.M;
  if (M.nmocap && !mocaps) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline: mocap required");
  if (B < 1 || N < 1 || H < 1 || P < 1 || interp < 0 || interp > 2) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline: bad sizes");
  if ((int64_t)B * N > h->maxN || H > h->maxH || P > h->maxP) return fail(MJPC_B200_ERR_CAPACITY, "rollout_spline: B*N/H/P above capacity");
  const int K = h->nmembers;
  if (K && (h->xfrc_std > 0.f || !h->noise_seeds.empty()))
    return fail(MJPC_B200_ERR_UNSUPPORTED, "rollout_spline: force noise (set_xfrc_noise) is not available while a "
                                           "model ensemble is set (set_model_ensemble)");
  CUDA_TRY(cudaSetDevice(h->device));
  RolloutArgs A = base_args(h, B * std::max(K, 1) * N, H);
  size_t end;
  if (int rc = stage_problems(h, B, states, times, mocaps, weights, parameters, task_states, knot_times, P, H, knots, N, &A,
                              &end, std::max(K, 1)))
    return rc;
  if (K) {   // launch problem b K + k: problem b on member k; the members' returns are scored by launch_rollout
    A.pack = h->d_members; A.pack_stride = h->member_stride; A.pack_index = h->d_member_index;
    A.returns = h->d_member_returns; A.failure = h->d_member_failure;
  }
  A.L = make_layout(h->pack.M, P);
  A.P = P; A.interp = interp; A.policy_kind = 0;
  h->resident = A;
  h->resident_members = K;
  h->resident_ok = true;
  return 0;
}

int mjpc_b200_upload_spline_inputs(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                                   const float* userdata, const float* knots, const double* knot_times, int interp,
                                   int P, int N, int H) {
  if (!h || !state || !knots || !knot_times) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline: null pointer");
  if (int rc = check_variants(h, -1, "rollout_spline")) return rc;
  // mjData::userdata: none of the implemented residuals reads it; a model that declares nuserdata > 0 is rejected at
  // create(), so a non-NULL pointer here can only be a caller error - refuse rather than silently ignore it
  if (userdata && h->nuserdata == 0) return fail(MJPC_B200_ERR_UNSUPPORTED, "rollout_spline: the model has nuserdata = 0, userdata must be NULL");
  return upload_spline(h, 1, state, &time, mocap, nullptr, nullptr, nullptr, knots, knot_times, interp, P, N, H);
}

int mjpc_b200_rollout_spline_batched(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                                     const double* weights, const double* parameters, const double* task_states,
                                     const float* knots, const double* knot_times, int interp, int P, int N, int H,
                                     float* returns, uint8_t* failure, int* order) {
  if (!h || !states || !times || !knots || !knot_times) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline_batched: null pointer");
  int rc = upload_spline(h, B, states, times, mocaps, weights, parameters, task_states, knots, knot_times, interp, P, N, H);
  if (rc) return rc;
  rc = launch_rollout(h, h->resident, h->resident_members);
  if (rc) return rc;
  return read_back(h, B * N, returns, failure, order);
}

// The buffers of a belief launch of B problems x K members: the per-trajectory buffers for K x max_candidates
// trajectories and the member returns (set_model_ensemble's reserve_members), and the launch's own tables, grown to B
// problems (never shrunk): covariances, the joint table (once), and the per-row variant index and per-problem status.
// On an allocation failure the handle keeps what it had.
static int reserve_belief(mjpc_b200_t* h, int B, int K) {
  const DevModel& M = h->pack.M;
  const size_t n = 2 * (size_t)M.nv;
  if (int rc = reserve_members(h, K)) return rc;
  if (!h->d_jnt) {
    std::vector<int> jnt(3 * (size_t)std::max(M.njnt, 1), 0);
    for (int j = 0; j < M.njnt; j++) {
      jnt[j] = h->pack.i[M.io[I_jnt_type] + j];
      jnt[M.njnt + j] = h->pack.i[M.io[I_jnt_qposadr] + j];
      jnt[2 * M.njnt + j] = h->pack.i[M.io[I_jnt_dofadr] + j];
    }
    DeviceArray<int> dj, db;
    cudaError_t e = dj.alloc(jnt.size());
    if (e == cudaSuccess) e = db.alloc(33 * (size_t)h->maxN);
    if (e == cudaSuccess) e = cudaMemcpy(dj, jnt.data(), jnt.size() * 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(MJPC_B200_ERR_CUDA, std::string("rollout_spline_belief_batched: ") + cudaGetErrorString(e));
    }
    h->d_jnt = std::move(dj); h->d_belief = std::move(db);
  }
  if (B > h->cov_problems) {
    DeviceArray<double> dc;
    if (cudaError_t e = dc.alloc((size_t)B * n * n))
      return fail(MJPC_B200_ERR_CUDA, std::string("rollout_spline_belief_batched: ") + cudaGetErrorString(e));
    CUDA_TRY(cudaStreamSynchronize(h->stream));   // a launch in flight may still read the old covariances
    h->d_cov = std::move(dc); h->cov_problems = B;
  }
  return 0;
}

// An initial-state ensemble launch: problem b is staged K times (stage_problems with R = K), state_sample_kernel
// overwrites rows b K + 1 .. b K + K - 1 with member states drawn from covariances[b], the rollout runs the B K N
// trajectories on the handle's instance (each row on its problem's variant, when variants are set), and
// ensemble_score_kernel scores them with `worst`.  Every refusal comes before anything is staged.
int mjpc_b200_rollout_spline_belief_batched(mjpc_b200_t* h, int B, int K, int worst, uint32_t seed, uint32_t iteration,
                                            const float* states, const double* covariances, const double* times,
                                            const float* mocaps, const double* weights, const double* parameters,
                                            const double* task_states, const float* knots, const double* knot_times,
                                            int interp, int P, int N, int H, float* returns, uint8_t* failure,
                                            int* order) {
  static const char* call = "rollout_spline_belief_batched";
  if (!h || !states || !covariances || !times || !knots || !knot_times)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": null pointer");
  const DevModel& M = h->pack.M;
  if (M.nmocap && !mocaps) return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": mocap required");
  if (K < 1 || K > 32) return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": K must be in [1, 32]");
  if (worst < 1 || worst > K) return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": worst must be in [1, K]");
  if (B < 1 || N < 1 || H < 1 || P < 1 || interp < 0 || interp > 2)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": bad sizes");
  if ((int64_t)B * N > h->maxN || H > h->maxH || P > h->maxP)
    return fail(MJPC_B200_ERR_CAPACITY, std::string(call) + ": B*N/H/P above capacity");
  if (h->nmembers)
    return fail(MJPC_B200_ERR_UNSUPPORTED, std::string(call) + ": not available while a model ensemble is set "
                                                               "(set_model_ensemble)");
  if (h->xfrc_std > 0.f || !h->noise_seeds.empty())
    return fail(MJPC_B200_ERR_UNSUPPORTED, std::string(call) + ": not available with force noise (set_xfrc_noise)");
  if (int rc = check_variants(h, B, call)) return rc;
  const size_t n = 2 * (size_t)M.nv, nn = n * n;
  for (int b = 0; b < B; b++)
    for (size_t e = 0; e < nn; e++)
      if (!std::isfinite(covariances[(size_t)b * nn + e]))
        return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": problem " + std::to_string(b) +
                                                    ": non-finite covariance entry " + std::to_string(e));
  const size_t smem = belief_smem((int)n, M.nq, M.nv);
  if (smem > h->smem_optin)
    return fail(MJPC_B200_ERR_CAPACITY, std::string(call) + ": the covariance does not fit in shared memory");
  CUDA_TRY(cudaSetDevice(h->device));
  if (int rc = reserve_belief(h, B, K)) return rc;
  RolloutArgs A = base_args(h, B * K * N, H);
  size_t end;
  if (int rc = stage_problems(h, B, states, times, mocaps, weights, parameters, task_states, knot_times, P, H, knots, N,
                              &A, &end, K))
    return rc;
  h->resident_ok = false;   // d_in now holds this launch, which is not a resident one
  CUDA_TRY(cudaMemcpyAsync(h->d_cov, covariances, (size_t)B * nn * 8, cudaMemcpyHostToDevice, h->stream));
  BeliefArgs S;
  S.B = B; S.K = K; S.n = (int)n; S.nq = M.nq; S.nv = M.nv; S.njnt = M.njnt;
  S.jnt = h->d_jnt; S.cov = h->d_cov; S.seed = seed; S.iteration = iteration;
  S.rows = const_cast<float*>(A.state);
  S.variant_index = h->nvariants ? h->d_variant_index.get() : nullptr;
  S.row_index = h->d_belief; S.status = h->d_belief + 32 * (size_t)h->maxN;
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute((const void*)state_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  state_sample_kernel<<<B, kBeliefThreads, smem, h->stream>>>(S);
  CUDA_TRY(cudaGetLastError());
  std::vector<int> status(B);
  CUDA_TRY(cudaMemcpyAsync(status.data(), S.status, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; b++)
    if (status[b])
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": problem " + std::to_string(b) +
                                                  ": the covariance is not positive semi-definite (a pivot below -tau, or a "
                                                  "pivot within tau of 0 with a coupling below it; "
                                                  "tau = 2 nv 2^-40 P_jj)");
  if (h->nvariants) A.pack_index = h->d_belief;
  A.returns = h->d_member_returns; A.failure = h->d_member_failure;
  A.L = make_layout(M, P);
  A.P = P; A.interp = interp; A.policy_kind = 0;
  if (int rc = launch_rollout(h, A, K, worst)) return rc;
  return read_back(h, B * N, returns, failure, order);
}

int mjpc_b200_host_state_member(const mjpc_model_blob* model, const double* state, const double* covariance,
                                uint32_t seed, uint32_t iteration, int problem, int member, double* out) {
  if (!model || !model->data || !state || !covariance || !out || problem < 0 || member < 0 || member > 31)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "host_state_member: bad argument");
  std::vector<int> type, qadr, dadr;
  int nq = 0, nv = 0;
  try {
    Blob b(model->data, model->nbytes);
    nq = b.i("nq"); nv = b.i("nv");
    type = b.ints("jnt_type"); qadr = b.ints("jnt_qposadr"); dadr = b.ints("jnt_dofadr");
  } catch (const std::exception& e) {
    return fail(MJPC_B200_ERR_BAD_BLOB, std::string("host_state_member: ") + e.what());
  }
  const int n = 2 * nv;
  std::copy(state, state + nq + nv, out);
  for (int e = 0; e < n * n; e++)
    if (!std::isfinite(covariance[e]))
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "host_state_member: non-finite covariance entry " + std::to_string(e));
  std::vector<double> L((size_t)n * n, 0.0), z(n), dx(n);
  for (int i = 0; i < n; i++)
    for (int c = 0; c <= i; c++) L[(size_t)i * n + c] = 0.5 * (covariance[i * n + c] + covariance[c * n + i]);
  std::vector<double> tau(n);
  for (int i = 0; i < n; i++) belief_tolerance(L.data(), n, i, tau.data());
  for (int j = 0; j < n; j++) {   // state_sample_kernel's order
    if (!belief_pivot(L.data(), n, j, tau.data()))
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "host_state_member: the covariance is not positive semi-definite");
    for (int i = j + 1; i < n; i++) belief_column(L.data(), n, j, i);
    for (int i = j + 1; i < n; i++)
      for (int c = j + 1; c <= i; c++) belief_update(L.data(), n, j, i, c);
  }
  if (member == 0) return 0;
  for (int e = 0; e < n; e++) z[e] = belief_normal(seed, iteration, problem, member, e);
  for (int i = 0; i < n; i++) dx[i] = belief_row(L.data(), z.data(), n, i);
  for (size_t j = 0; j < type.size(); j++) belief_joint(out + qadr[j], dx.data() + dadr[j], type[j]);
  for (int i = 0; i < nv; i++) out[nq + i] = belief_add(out[nq + i], dx[nv + i]);
  return 0;
}

int mjpc_b200_launch_resident(mjpc_b200_t* h) {
  if (!h || !h->resident_ok) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "launch_resident: no uploaded inputs");
  if (int rc = check_variants(h, h->resident.nprob, "launch_resident")) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  // the step table was built on the upload's clock; a set_options timestep since then needs a new upload
  if (h->resident.timestep != h->pack.timestep)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "launch_resident: the timestep changed since the upload");
  h->resident.M = h->pack.M;  // picks up set_task changes (risk)
  return launch_rollout(h, h->resident, h->resident_members);
}

int mjpc_b200_sync(mjpc_b200_t* h) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "sync: null");
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (h->lastN > 0 && cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  return 0;
}

int mjpc_b200_read_returns(mjpc_b200_t* h, float* returns, uint8_t* failure, int* order) {
  if (!h || h->lastN < 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "read_returns: nothing launched");
  CUDA_TRY(cudaSetDevice(h->device));
  return read_back(h, h->lastN, returns, failure, order);
}

int mjpc_b200_rollout_spline(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                             const float* userdata, const float* knots, const double* knot_times, int interp,
                             int P, int N, int H, float* returns, uint8_t* failure, int* order) {
  int rc = mjpc_b200_upload_spline_inputs(h, state, time, mocap, userdata, knots, knot_times, interp, P, N, H);
  if (rc) return rc;
  rc = launch_rollout(h, h->resident, h->resident_members);
  if (rc) return rc;
  return read_back(h, N, returns, failure, order);
}

// Feedback rollouts of B problems x K candidates in one launch; B = 1 is the single-problem call.  Every problem's
// nominal times and time-like task state are rebased to its own start time.  Nothing is changed on a refusal.
static int rollout_feedback_impl(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                                 const double* weights, const double* parameters, const double* task_states,
                                 const float* u_nom, const float* x_nom, const double* t_nom, const float* gains,
                                 const float* du, const float* step_sizes, int mode, int K, int H, float* returns,
                                 uint8_t* failure, int* order) {
  const DevModel& M = h->pack.M;
  if (M.nmocap && !mocaps) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_feedback: mocap required");
  if (B < 1 || K < 1 || H < 1 || mode < 0 || mode > 3) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_feedback: bad sizes");
  if ((int64_t)B * K > h->maxN || H > h->maxH) return fail(MJPC_B200_ERR_CAPACITY, "rollout_feedback: B*K/H above capacity");
  CUDA_TRY(cudaSetDevice(h->device));
  const size_t ds = M.nq + M.nv, n = 2 * M.nv, nu = M.nu, Hs = H, P = B;
  if (int rc = reserve_feedback(h, B)) return rc;
  if (int rc = reserve_h_in(h, problem_floats(M, B, 0, H) + P * Hs * (nu + ds + 1 + nu * n + nu) + P * K + 64)) return rc;
  RolloutArgs A = base_args(h, B * K, H);
  size_t o;
  if (int rc = stage_problems(h, B, states, times, mocaps, weights, parameters, task_states, t_nom, H, H, nullptr, K, &A, &o))
    return rc;
  auto put = [&](const float* src, size_t cnt) { size_t at = o; if (src) std::memcpy(h->h_in + o, src, cnt * 4); o += cnt; return at; };
  const size_t ou = put(u_nom, P * Hs * nu), ox = put(x_nom, P * Hs * ds);
  const size_t ot = o;
  for (int b = 0; b < B; b++)
    for (int i = 0; i < H; i++) h->h_in[o + (size_t)b * H + i] = (float)(t_nom[(size_t)b * H + i] - times[b]);
  o += P * Hs;
  const size_t og = put(gains, P * Hs * nu * n), od = put(du, P * Hs * nu), os = put(step_sizes, P * K);
  auto up = [&](float* dst, size_t at, size_t cnt) { return cudaMemcpyAsync(dst, h->h_in + at, cnt * 4, cudaMemcpyHostToDevice, h->stream); };
  CUDA_TRY(up(h->d_unom, ou, P * Hs * nu)); CUDA_TRY(up(h->d_xnom, ox, P * Hs * ds)); CUDA_TRY(up(h->d_tnom, ot, P * Hs));
  CUDA_TRY(up(h->d_gains, og, P * Hs * nu * n));
  if (du) CUDA_TRY(up(h->d_du, od, P * Hs * nu));
  CUDA_TRY(up(h->d_steps, os, P * K));
  A.L = make_layout(h->pack.M, 1);
  A.P = 1; A.policy_kind = 1;
  A.fb.u_nom = h->d_unom; A.fb.x_nom = h->d_xnom; A.fb.t_nom = h->d_tnom; A.fb.gains = h->d_gains;
  A.fb.du = du ? h->d_du.get() : nullptr; A.fb.iv = A.iv; A.fb.mode = mode; A.fb.H = H; A.fb.nper = K;
  A.step_sizes = h->d_steps;
  h->resident_ok = false;
  int rc = launch_rollout(h, A);
  if (rc) return rc;
  return read_back(h, B * K, returns, failure, order);
}

int mjpc_b200_rollout_feedback(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                               const float* userdata, const float* u_nom, const float* x_nom, const double* t_nom,
                               const float* gains, const float* du, const float* step_sizes, int mode, int K, int H,
                               float* returns, uint8_t* failure, int* order) {
  if (!h || !state || !u_nom || !x_nom || !t_nom || !gains || !step_sizes)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_feedback: null pointer");
  if (int rc = check_variants(h, -1, "rollout_feedback")) return rc;
  if (int rc = check_ensemble(h, "rollout_feedback")) return rc;
  if (userdata && h->nuserdata == 0) return fail(MJPC_B200_ERR_UNSUPPORTED, "rollout_feedback: the model has nuserdata = 0, userdata must be NULL");
  return rollout_feedback_impl(h, 1, state, &time, mocap, nullptr, nullptr, nullptr, u_nom, x_nom, t_nom, gains, du,
                               step_sizes, mode, K, H, returns, failure, order);
}

int mjpc_b200_rollout_feedback_batched(mjpc_b200_t* h, int B, const float* states, const double* times, const float* mocaps,
                                       const double* weights, const double* parameters, const double* task_states,
                                       const float* u_nom, const float* x_nom, const double* t_nom, const float* gains,
                                       const float* du, const float* step_sizes, int mode, int K, int H, float* returns,
                                       uint8_t* failure, int* order) {
  if (!h || !states || !times || !u_nom || !x_nom || !t_nom || !gains || !step_sizes)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_feedback_batched: null pointer");
  if (int rc = check_ensemble(h, "rollout_feedback_batched")) return rc;
  return rollout_feedback_impl(h, B, states, times, mocaps, weights, parameters, task_states, u_nom, x_nom, t_nom, gains,
                               du, step_sizes, mode, K, H, returns, failure, order);
}

void mjpc_b200_host_policy_intervals(const double* nodes, int count, double time0, double timestep, int H, double* times,
                                     int* upper, float* frac) {
  std::vector<PolicyInterval> iv(std::max(H, 0));
  build_policy_intervals(nodes, count, time0, timestep, H, iv.data());
  for (int t = 0; t < H; t++) { times[t] = iv[t].time; upper[t] = iv[t].upper; frac[t] = iv[t].frac; }
}

// trajectories [first, first + count) of the last launch into rows [row, row + count) of the host arrays
static int fetch_impl(mjpc_b200_t* h, int first, int count, float* states, float* actions, double* times,
                      float* residual, float* costs, float* trace, int row = 0) {
  const DevModel& M = h->pack.M;
  const size_t H = h->lastH, ds = M.nq + M.nv, nu = M.nu, nr = M.num_residual, ntr = 3 * M.num_trace;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  auto get = [&](void* dst, const void* src, size_t per, size_t elt) {
    return dst ? cudaMemcpy((char*)dst + (size_t)row * per * elt, (const char*)src + (size_t)first * per * elt,
                            (size_t)count * per * elt, cudaMemcpyDeviceToHost)
               : cudaSuccess;
  };
  CUDA_TRY(get(states, h->d_states, H * ds, 4)); CUDA_TRY(get(actions, h->d_actions, H * nu, 4));
  CUDA_TRY(get(times, h->d_times, H, 8)); CUDA_TRY(get(residual, h->d_residual, H * nr, 4));
  CUDA_TRY(get(costs, h->d_costs, H, 4)); CUDA_TRY(get(trace, h->d_trace, H * ntr, 4));
  return 0;
}

// the launched trajectory of candidate c (flat b N + i) of the last launch as member k rolled it out
static int member_trajectory(const mjpc_b200_t* h, int c, int k) {
  if (!h->last_members) return c;
  const int b = c / h->last_nper, i = c - b * h->last_nper;
  return (b * h->last_members + k) * h->last_nper + i;
}

int mjpc_b200_fetch_trajectory(mjpc_b200_t* h, int candidate, float* states, float* actions, double* times,
                               float* residual, float* costs, float* trace) {
  if (!h || h->lastN < 1 || candidate < 0 || candidate >= h->lastN)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_trajectory: bad candidate");
  return fetch_impl(h, member_trajectory(h, candidate, 0), 1, states, actions, times, residual, costs, trace);
}

int mjpc_b200_fetch_trajectory_member(mjpc_b200_t* h, int candidate, int member, float* states, float* actions,
                                      double* times, float* residual, float* costs, float* trace) {
  if (!h || h->lastN < 1 || candidate < 0 || candidate >= h->lastN)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_trajectory_member: bad candidate");
  if (member < 0 || member >= std::max(h->last_members, 1))
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_trajectory_member: member " + std::to_string(member) +
                                                " outside the last launch's " + std::to_string(std::max(h->last_members, 1)));
  return fetch_impl(h, member_trajectory(h, candidate, member), 1, states, actions, times, residual, costs, trace);
}

int mjpc_b200_fetch_all(mjpc_b200_t* h, float* states, float* actions, double* times, float* residual, float* costs,
                        float* trace) {
  if (!h || h->lastN < 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_all: nothing to fetch");
  if (!h->last_members) return fetch_impl(h, 0, h->lastN, states, actions, times, residual, costs, trace);
  for (int b = 0; b < h->lastN / h->last_nper; b++)   // member 0 of each problem's candidates
    if (int rc = fetch_impl(h, member_trajectory(h, b * h->last_nper, 0), h->last_nper, states, actions, times, residual,
                            costs, trace, b * h->last_nper))
      return rc;
  return 0;
}

int mjpc_b200_fetch_ensemble(mjpc_b200_t* h, float* member_returns, uint8_t* member_failure) {
  if (!h || h->lastN < 1 || !h->last_members)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_ensemble: the last launch was not a model-ensemble launch");
  const size_t n = (size_t)h->lastN * h->last_members;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (member_returns) CUDA_TRY(cudaMemcpy(member_returns, h->d_member_returns, n * 4, cudaMemcpyDeviceToHost));
  if (member_failure) CUDA_TRY(cudaMemcpy(member_failure, h->d_member_failure, n, cudaMemcpyDeviceToHost));
  return 0;
}

void mjpc_b200_host_ensemble_score(const float* member_returns, const uint8_t* member_failure, int K, int worst,
                                   float* score, uint8_t* failure) {
  if (K < 1 || K > 32 || worst < 1 || worst > K) return;
  const float* r = member_returns;
  bool failed = false;
  int at[32];
  for (int k = 0; k < K; k++) {
    failed |= member_failure[k] != 0;
    int rank = 0;   // descending, ties to the lower member, NaN first (ensemble_score_kernel)
    for (int j = 0; j < K; j++)
      rank += (r[j] > r[k]) || (r[j] == r[k] && j < k) || (r[j] != r[j] && (r[k] == r[k] || j < k));
    at[rank] = k;
  }
  double sum = 0.0;
  for (int p = 0; p < worst; p++) sum += (double)r[at[p]];
  *score = failed ? 1.0e6f : (float)(sum / (double)worst);
  *failure = failed ? 1 : 0;
}

// Test hooks: rank_kernel and ensemble_score_kernel on the caller's data, launched as launch_rollout launches them, on
// the handle's stream and in scratch of their own (the last launch's buffers are untouched).
int mjpc_b200_debug_rank(mjpc_b200_t* h, const float* returns, int nseg, int N, int* order) {
  if (!h || !returns || !order || nseg < 1 || N < 1 || (long long)nseg * N > INT_MAX / 2)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "debug_rank: bad argument");
  const size_t n = (size_t)nseg * N;
  CUDA_TRY(cudaSetDevice(h->device));
  DeviceArray<float> d_ret;
  DeviceArray<int> d_order;
  CUDA_TRY(d_ret.alloc(n)); CUDA_TRY(d_order.alloc(n));
  CUDA_TRY(cudaMemcpyAsync(d_ret, returns, n * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemsetAsync(d_order, 0xFF, n * 4, h->stream));   // -1: a slot the kernel does not write stays visible
  rank_kernel<<<(int)((n + 255) / 256), 256, 0, h->stream>>>(d_ret, N, nseg, d_order);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(order, d_order, n * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int mjpc_b200_debug_ensemble_score(mjpc_b200_t* h, const float* member_returns, const uint8_t* member_failure, int B,
                                   int K, int N, int worst, float* returns, uint8_t* failure) {
  if (!h || !member_returns || !member_failure || !returns || !failure || B < 1 || N < 1 || K < 1 || K > 32 ||
      worst < 1 || worst > K || (long long)B * K * N > INT_MAX / 32)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "debug_ensemble_score: bad argument");
  const size_t n = (size_t)B * N, nm = n * K;
  CUDA_TRY(cudaSetDevice(h->device));
  DeviceArray<float> d_mr, d_ret;
  DeviceArray<unsigned char> d_mf, d_fail;
  CUDA_TRY(d_mr.alloc(nm)); CUDA_TRY(d_mf.alloc(nm)); CUDA_TRY(d_ret.alloc(n)); CUDA_TRY(d_fail.alloc(n));
  CUDA_TRY(cudaMemcpyAsync(d_mr, member_returns, nm * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync(d_mf, member_failure, nm, cudaMemcpyHostToDevice, h->stream));
  ensemble_score_kernel<<<(int)((n + 7) / 8), 256, 0, h->stream>>>(d_mr, d_mf, B, K, N, worst, d_ret, d_fail);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(returns, d_ret, n * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(failure, d_fail, n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

// grow step_impl's device scratch and pinned staging to `words` floats each (never shrinks); on failure the old ones stay
int reserve_step(mjpc_b200_t* h, size_t words) {
  if (words <= h->step_words) return 0;
  DeviceArray<float> d;
  PinnedArray<float> p;
  CUDA_TRY(d.alloc(words));
  if (p.alloc(words)) return fail(MJPC_B200_ERR_CUDA, "step: out of pinned host memory");
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  h->d_step = std::move(d); h->h_step = std::move(p); h->step_words = words;
  return 0;
}

// B single steps (see step_batch_kernel) on instance `fn`.  times are absolute; the task state is rebased to time0
// (device time = times[b] - time0).  Outputs may be NULL; qM [B][nv nv], efc_force [B][maxefc] and contact
// [B][maxcon][8] are the optional ones, their rows past each problem's counts read as zeros.  sensordata [B][dim]
// (NULL: not evaluated) receives sensors [s0, s0 + ns) of the handle's table, dim = their total dimension.  e0 / e1,
// when given, time the kernel.  Inputs go up in one copy from the handle's pinned staging, outputs come back in one.
static int step_impl(mjpc_b200_t* h, const void* fn, int B, const float* qpos, const float* qvel, const float* ctrl,
                     const float* warmstart, const float* mocap, double time0, const double* times, float* qacc,
                     float* next_qpos, float* next_qvel, float* residual, float* cost, int* counts, float* qM,
                     float* efc_force, float* contact, cudaEvent_t e0, cudaEvent_t e1, int s0 = 0, int ns = 0,
                     float* sensordata = nullptr) {
  const DevModel& M = h->pack.M;
  CUDA_TRY(cudaSetDevice(h->device));
  const size_t Bs = B, nq = M.nq, nv = M.nv, nu = M.nu, nr = std::max(M.num_residual, 1), nm = 7 * (size_t)M.nmocap,
               nts = (size_t)M.task_state_size;
  const int adr0 = ns ? h->sensors[s0].adr : 0;
  const size_t nsd = ns ? (size_t)(h->sensors[s0 + ns - 1].adr - adr0 + sensor_dim(h->sensors[s0 + ns - 1].type)) : 0;
  size_t words = 0;
  auto take = [&](size_t n) { const size_t at = words; words += n; return at; };
  const size_t o_qpos = take(Bs * nq), o_qvel = take(Bs * nv), o_ctrl = take(Bs * nu), o_warm = take(Bs * nv),
               o_time = take(Bs), o_mocap = take(nm), o_ts = take(nts), in_words = words, o_qacc = take(Bs * nv),
               o_nq = take(Bs * nq), o_nv = take(Bs * nv), o_res = take(Bs * nr), o_cost = take(Bs),
               o_counts = take(4 * Bs), o_qM = take(qM ? Bs * nv * nv : 0), o_efc = take(efc_force ? Bs * M.maxefc : 0),
               o_con = take(contact ? Bs * M.maxcon * 8 : 0), o_sens = take(sensordata ? Bs * nsd : 0);
  if (int rc = reserve_step(h, words)) return rc;
  float *d = h->d_step, *p = h->h_step;
  std::memcpy(p + o_qpos, qpos, Bs * nq * 4); std::memcpy(p + o_qvel, qvel, Bs * nv * 4);
  std::memcpy(p + o_ctrl, ctrl, Bs * nu * 4);
  if (warmstart) std::memcpy(p + o_warm, warmstart, Bs * nv * 4);
  for (int i = 0; i < B; i++) p[o_time + i] = (float)(times[i] - time0);
  if (nm) std::memcpy(p + o_mocap, mocap, nm * 4);
  rebase_task_state(h, nullptr, time0, p + o_ts);
  // every transfer on the engine stream, ordered with the kernel
  CUDA_TRY(cudaMemsetAsync(d + in_words, 0, (words - in_words) * 4, h->stream));
  CUDA_TRY(cudaMemcpyAsync(d, p, in_words * 4, cudaMemcpyHostToDevice, h->stream));
  StepBatchArgs A;
  std::memset(&A, 0, sizeof(A));
  A.M = h->pack.M; A.L = make_layout(h->pack.M, 1); A.pack = h->d_pack;
  A.qpos = d + o_qpos; A.qvel = d + o_qvel; A.ctrl = d + o_ctrl; A.warmstart = warmstart ? d + o_warm : nullptr;
  A.mocap = d + o_mocap; A.task_state = nts ? d + o_ts : nullptr; A.time = d + o_time; A.B = B;
  A.qacc = d + o_qacc; A.next_qpos = d + o_nq; A.next_qvel = d + o_nv; A.residual = d + o_res; A.cost = d + o_cost;
  A.counts = (int*)(d + o_counts);
  A.qM = qM ? d + o_qM : nullptr; A.efc_force = efc_force ? d + o_efc : nullptr; A.contact = contact ? d + o_con : nullptr;
  if (sensordata) {
    A.sensors = h->d_sensors + s0; A.nsensor = ns; A.sensor_adr0 = adr0; A.sensor_dim = (int)nsd;
    A.sensordata = d + o_sens;
  }
  if (e0) CUDA_TRY(cudaEventRecord(e0, h->stream));
  launch_kernel(fn, B, 32, h->smem_bytes(1), h->stream, A);
  if (e1) CUDA_TRY(cudaEventRecord(e1, h->stream));
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  CUDA_TRY(cudaMemcpyAsync(p + in_words, d + in_words, (words - in_words) * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (e0 && cudaEventElapsedTime(&h->last_ms, e0, e1) != cudaSuccess) cudaGetLastError();
  auto get = [&](void* dst, size_t at, size_t bytes) { if (dst) std::memcpy(dst, p + at, bytes); };
  get(qacc, o_qacc, Bs * nv * 4); get(next_qpos, o_nq, Bs * nq * 4);
  get(next_qvel, o_nv, Bs * nv * 4); get(residual, o_res, Bs * M.num_residual * 4);
  get(cost, o_cost, Bs * 4); get(counts, o_counts, Bs * 16);
  get(qM, o_qM, Bs * nv * nv * 4); get(efc_force, o_efc, Bs * M.maxefc * 4);
  get(contact, o_con, Bs * M.maxcon * 8 * 4); get(sensordata, o_sens, Bs * nsd * 4);
  return 0;
}

// One step of the generic instance at device time (float)time, with the task state as set_task left it: step_impl
// with B = 1 and time0 = 0.  Not timed: last_kernel_ms and last_kernel_static keep describing the last planning launch.
int mjpc_b200_step_debug(mjpc_b200_t* h, const float* qpos, const float* qvel, const float* ctrl,
                         const float* mocap, double time, const float* warmstart, float* qacc, float* residual,
                         float* next_qpos, float* next_qvel, float* qM, float* efc_force, int* counts) {
  if (!h || !qpos || !qvel || !ctrl) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_debug: null");
  if (int rc = check_variants(h, -1, "step_debug")) return rc;
  if (int rc = check_ensemble(h, "step_debug")) return rc;
  h->dbg_ncon = -1;
  h->dbg_contact.resize((size_t)h->pack.M.maxcon * 8);
  if (efc_force) std::fill_n(efc_force, 256, 0.f);   // the caller's efc_force holds 256 floats, the first maxefc are rows
  int cnt[4];
  if (int rc = step_impl(h, kGenericKernels.step, 1, qpos, qvel, ctrl, warmstart, mocap, 0.0, &time, qacc, next_qpos,
                         next_qvel, residual, nullptr, cnt, qM, efc_force, h->dbg_contact.data(), nullptr, nullptr))
    return rc;
  if (counts) std::memcpy(counts, cnt, 16);
  h->dbg_ncon = cnt[0];
  return 0;
}

int mjpc_b200_step_debug_contacts(mjpc_b200_t* h, int capacity, float* contact, int* ncon) {
  if (!h || capacity < 0 || (capacity > 0 && !contact) || !ncon)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_debug_contacts: bad argument");
  if (int rc = check_variants(h, -1, "step_debug_contacts")) return rc;
  if (int rc = check_ensemble(h, "step_debug_contacts")) return rc;
  if (h->dbg_ncon < 0) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_debug_contacts: no step_debug call to report");
  *ncon = h->dbg_ncon;
  const int n = std::min(h->dbg_ncon, capacity);
  if (n > 0) std::memcpy(contact, h->dbg_contact.data(), (size_t)n * 8 * 4);
  return 0;
}

// ---- multi-GPU: one planning problem, candidates sharded over the ranks of an NCCL communicator (SURVEY.md 8e)
int mjpc_b200_comm_unique_id(void* out, size_t nbytes) {
  if (!out || nbytes < sizeof(ncclUniqueId)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "comm_unique_id: need 128 bytes");
  NcclApi& api = nccl_api();
  if (!api.ok) return fail(MJPC_B200_ERR_UNSUPPORTED, "libnccl.so.2 not found");
  ncclUniqueId id;
  NCCL_TRY(api.GetUniqueId(&id));
  std::memcpy(out, &id, sizeof(id));
  return 0;
}

int mjpc_b200_comm_init(mjpc_b200_t* h, int nranks, int rank, const void* unique_id, size_t nbytes) {
  if (!h || nranks < 1 || rank < 0 || rank >= nranks || !unique_id || nbytes < sizeof(ncclUniqueId))
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "comm_init: bad argument");
  if (h->comm) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "comm_init: communicator already initialised");
  NcclApi& api = nccl_api();
  if (!api.ok) return fail(MJPC_B200_ERR_UNSUPPORTED, "libnccl.so.2 not found");
  CUDA_TRY(cudaSetDevice(h->device));
  // the exchange buffers first, then the communicator, then everything is stored at once: a refusal leaves no
  // communicator on the handle, so the call can be repeated
  const DevModel& M = h->pack.M;
  const size_t width = h->maxN, total = (size_t)nranks * h->maxN,
               bcast_floats = (size_t)h->maxH * (M.nq + M.nv + M.nu + M.num_residual + 1 + 3 * M.num_trace + 2) + 16;
  DeviceArray<float> slot, gather, returns_all, bcast;
  DeviceArray<unsigned char> failure_all;
  DeviceArray<int> order_all;
  CUDA_TRY(slot.alloc(2 * width)); CUDA_TRY(gather.alloc(2 * width * nranks));
  CUDA_TRY(returns_all.alloc(total)); CUDA_TRY(failure_all.alloc(total)); CUDA_TRY(order_all.alloc(total));
  CUDA_TRY(bcast.alloc(bcast_floats));
  ncclUniqueId id;
  std::memcpy(&id, unique_id, sizeof(id));
  ncclComm_t comm = nullptr;
  NCCL_TRY(api.CommInitRank(&comm, nranks, id, rank));
  h->comm = comm; h->nranks = nranks; h->rank = rank;
  h->maxTotal = (int)total; h->bcast_floats = bcast_floats;
  h->d_slot = std::move(slot); h->d_gather = std::move(gather); h->d_returns_all = std::move(returns_all);
  h->d_failure_all = std::move(failure_all); h->d_order_all = std::move(order_all); h->d_bcast = std::move(bcast);
  return 0;
}

int mjpc_b200_comm_info(const mjpc_b200_t* h, int* nranks, int* rank) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "comm_info: null");
  if (nranks) *nranks = h->nranks;
  if (rank) *rank = h->rank;
  return 0;
}

// SamplingPlanner::Rollouts for ONE planning problem on all ranks: every rank passes the same N candidates (inputs are
// replicated: a few KB), rolls out its contiguous shard, then the per-candidate returns and failure flags are exchanged
// with ONE ncclAllGather enqueued on the engine stream behind the rollout kernel (no host hop), compacted to global
// candidate order and ranked on the device.  returns / failure / order describe all N candidates, identical on every rank.
int mjpc_b200_rollout_spline_sharded(mjpc_b200_t* h, const float* state, double time, const float* mocap,
                                     const float* userdata, const float* knots, const double* knot_times, int interp,
                                     int P, int N, int H, float* returns, uint8_t* failure, int* order) {
  if (!h || !knots) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline_sharded: null");
  if (int rc = check_variants(h, -1, "rollout_spline_sharded")) return rc;
  if (int rc = check_ensemble(h, "rollout_spline_sharded")) return rc;
  if (!h->noise_seeds.empty())
    return fail(MJPC_B200_ERR_UNSUPPORTED, "rollout_spline_sharded: per-problem noise keys (set_xfrc_noise_batched)");
  if (h->nranks > 1 && !h->comm) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "rollout_spline_sharded: comm_init first");
  if (h->nranks == 1) {
    int rc = mjpc_b200_rollout_spline(h, state, time, mocap, userdata, knots, knot_times, interp, P, N, H, returns, failure, order);
    if (rc == 0) { h->totalN = N; h->shard_lo = 0; h->shard_hi = N; }
    return rc;
  }
  if (N < h->nranks || N > h->maxTotal) return fail(MJPC_B200_ERR_CAPACITY, "rollout_spline_sharded: N outside [nranks, nranks * max_candidates]");
  const DevModel& M = h->pack.M;
  int lo, hi;
  shard_range(N, h->nranks, h->rank, &lo, &hi);
  const int n = hi - lo, width = N / h->nranks + (N % h->nranks ? 1 : 0);
  if (n > h->maxN) return fail(MJPC_B200_ERR_CAPACITY, "rollout_spline_sharded: shard above max_candidates");
  int rc = mjpc_b200_upload_spline_inputs(h, state, time, mocap, userdata, knots + (size_t)lo * P * M.nu, knot_times, interp, P, n, H);
  if (rc) return rc;
  h->resident.cand0 = lo;
  rc = launch_rollout(h, h->resident);
  if (rc) return rc;
  NcclApi& api = nccl_api();
  pack_slot_kernel<<<(width + 255) / 256, 256, 0, h->stream>>>(h->d_returns, h->d_failure, n, width, h->d_slot);
  NCCL_TRY(api.AllGather(h->d_slot, h->d_gather, 2 * (size_t)width, ncclFloat, h->comm, h->stream));
  compact_gather_kernel<<<(N + 255) / 256, 256, 0, h->stream>>>(h->d_gather, N, h->nranks, width, h->d_returns_all, h->d_failure_all);
  rank_kernel<<<(N + 255) / 256, 256, 0, h->stream>>>(h->d_returns_all, N, 1, h->d_order_all);
  CUDA_TRY(cudaEventRecord(h->ev1, h->stream));   // the timed span now covers rollout + exchange + ranking
  CUDA_TRY(cudaGetLastError());
  h->launches += 3;
  h->totalN = N; h->shard_lo = lo; h->shard_hi = hi;
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  // N may exceed max_candidates, which sizes the pinned h_out: pageable copies straight into the caller's arrays
  if (returns) CUDA_TRY(cudaMemcpy(returns, h->d_returns_all, (size_t)N * 4, cudaMemcpyDeviceToHost));
  if (failure) CUDA_TRY(cudaMemcpy(failure, h->d_failure_all, (size_t)N, cudaMemcpyDeviceToHost));
  if (order) CUDA_TRY(cudaMemcpy(order, h->d_order_all, (size_t)N * 4, cudaMemcpyDeviceToHost));
  return 0;
}

// Trajectory of GLOBAL candidate `candidate` of the last sharded rollout on every rank: the owner packs it into one
// buffer, ncclBroadcast on the engine stream, every rank unpacks (BestTrajectory must be available wherever the policy
// is installed).  Any output pointer may be NULL.
int mjpc_b200_fetch_trajectory_sharded(mjpc_b200_t* h, int candidate, float* states, float* actions, double* times,
                                       float* residual, float* costs, float* trace) {
  if (!h || h->totalN < 1 || candidate < 0 || candidate >= h->totalN)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_trajectory_sharded: bad candidate");
  if (h->nranks == 1) return mjpc_b200_fetch_trajectory(h, candidate, states, actions, times, residual, costs, trace);
  const DevModel& M = h->pack.M;
  const size_t H = h->lastH, ds = M.nq + M.nv, nu = M.nu, nr = M.num_residual, ntr = 3 * M.num_trace;
  CUDA_TRY(cudaSetDevice(h->device));
  int owner = 0, lo = 0, hi = 0;
  for (owner = 0; owner < h->nranks; owner++) { shard_range(h->totalN, h->nranks, owner, &lo, &hi); if (candidate < hi) break; }
  float* b = h->d_bcast;
  const size_t o_s = 0, o_a = o_s + H * ds, o_r = o_a + H * nu, o_c = o_r + H * nr, o_tr = o_c + H, o_t = (o_tr + H * ntr + 1) & ~(size_t)1,
               total = o_t + 2 * H;
  if (total > h->bcast_floats) return fail(MJPC_B200_ERR_CAPACITY, "fetch_trajectory_sharded: horizon above capacity");
  if (owner == h->rank) {
    const size_t i = candidate - lo;
    auto cp = [&](size_t off, const void* src, size_t bytes) { return cudaMemcpyAsync(b + off, src, bytes, cudaMemcpyDeviceToDevice, h->stream); };
    CUDA_TRY(cp(o_s, h->d_states + i * H * ds, H * ds * 4)); CUDA_TRY(cp(o_a, h->d_actions + i * H * nu, H * nu * 4));
    CUDA_TRY(cp(o_r, h->d_residual + i * H * nr, H * nr * 4)); CUDA_TRY(cp(o_c, h->d_costs + i * H, H * 4));
    if (ntr) CUDA_TRY(cp(o_tr, h->d_trace + i * H * ntr, H * ntr * 4));
    CUDA_TRY(cp(o_t, h->d_times + i * H, H * 8));
  }
  NCCL_TRY(nccl_api().Broadcast(b, b, total, ncclFloat, owner, h->comm, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  auto get = [&](void* dst, size_t off, size_t bytes) { return dst ? cudaMemcpy(dst, b + off, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; };
  CUDA_TRY(get(states, o_s, H * ds * 4)); CUDA_TRY(get(actions, o_a, H * nu * 4)); CUDA_TRY(get(residual, o_r, H * nr * 4));
  CUDA_TRY(get(costs, o_c, H * 4)); CUDA_TRY(get(trace, o_tr, H * ntr * 4)); CUDA_TRY(get(times, o_t, H * 8));
  return 0;
}

// Batched single-step parity hook (step_impl) on the instance a rollout of this handle runs
int mjpc_b200_step_batch(mjpc_b200_t* h, int B, const float* qpos, const float* qvel, const float* ctrl,
                         const float* warmstart, const float* mocap, double time0, const double* times, float* qacc,
                         float* next_qpos, float* next_qvel, float* residual, float* cost, int* counts) {
  if (!h || B < 1 || !qpos || !qvel || !ctrl || !times) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_batch: bad argument");
  if (int rc = check_variants(h, -1, "step_batch")) return rc;
  if (int rc = check_ensemble(h, "step_batch")) return rc;
  if (h->pack.M.nmocap && !mocap) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_batch: mocap required");
  const KernelSet* k;
  const int kind = pick_kernels(h, &k);
  if (int rc = step_impl(h, k->step, B, qpos, qvel, ctrl, warmstart, mocap, time0, times, qacc, next_qpos, next_qvel,
                         residual, cost, counts, nullptr, nullptr, nullptr, h->ev0, h->ev1))
    return rc;
  h->last_static = kind ? 1 : 0;
  return 0;
}

// The sigma-point step of a state estimator (Unscented::EvaluateSigmaPoints, unscented.cc:353-394): B states, one
// ctrl, mocap and time, each advanced by one step_batch step with the measurement sensors of its pre-step state.
int mjpc_b200_step_sensors(mjpc_b200_t* h, int B, const float* states, const float* ctrl, const float* warmstart,
                           const float* mocap, double time, int sensor_start, int nsensor, float* next_states,
                           float* sensordata, float* qacc, int* counts) {
  if (!h || B < 1 || !states || (!ctrl && h->pack.M.nu) || !next_states || !sensordata)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_sensors: bad argument");
  if (int rc = check_variants(h, -1, "step_sensors")) return rc;
  if (int rc = check_ensemble(h, "step_sensors")) return rc;
  const DevModel& M = h->pack.M;
  if (M.nmocap && !mocap) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_sensors: mocap required");
  const int nsens = (int)h->sensors.size();
  if (sensor_start < 0 || nsensor < 1 || sensor_start > nsens - nsensor)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "step_sensors: sensor range [" + std::to_string(sensor_start) + ", " +
                                                std::to_string((long long)sensor_start + nsensor) + ") outside the model's " +
                                                std::to_string(nsens) + " sensors");
  for (int i = sensor_start; i < sensor_start + nsensor; i++)
    if (!h->sensor_why[i].empty())
      return fail(MJPC_B200_ERR_UNSUPPORTED, "step_sensors: sensor " + std::to_string(i) + ": " + h->sensor_why[i]);
  if (B > h->maxN) return fail(MJPC_B200_ERR_CAPACITY, "step_sensors: B > max_candidates");
  const KernelSet* k;
  const int kind = pick_kernels(h, &k);
  const size_t nq = M.nq, nv = M.nv, nu = M.nu, ds = nq + nv;
  std::vector<float> q(B * nq), v(B * nv), u(B * nu), nq_out(B * nq), nv_out(B * nv);
  std::vector<double> t(B, time);
  for (int b = 0; b < B; b++) {
    std::memcpy(&q[b * nq], states + b * ds, nq * 4); std::memcpy(&v[b * nv], states + b * ds + nq, nv * 4);
    std::memcpy(&u[b * nu], ctrl, nu * 4);
  }
  if (int rc = step_impl(h, k->step, B, q.data(), v.data(), u.data(), warmstart, mocap, time, t.data(), qacc,
                         nq_out.data(), nv_out.data(), nullptr, nullptr, counts, nullptr, nullptr, nullptr, h->ev0,
                         h->ev1, sensor_start, nsensor, sensordata))
    return rc;
  for (int b = 0; b < B; b++) {
    std::memcpy(next_states + b * ds, &nq_out[b * nq], nq * 4); std::memcpy(next_states + b * ds + nq, &nv_out[b * nv], nv * 4);
  }
  h->last_static = kind ? 1 : 0;
  return 0;
}

// ---- closed-loop plants (plant_bank.h, plant_step_kernel in rollout_kernels.cuh)

int mjpc_b200_plant_init(mjpc_b200_t* h, int num_plants, int sensor_start, int nsensor) {
  if (!h || num_plants < 1 || nsensor < 0) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_init: bad argument");
  if (int rc = check_ensemble(h, "plant_init")) return rc;
  if (num_plants > h->maxN) return fail(MJPC_B200_ERR_CAPACITY, "plant_init: num_plants > max_candidates");
  const int nsens = (int)h->sensors.size();
  if (nsensor && (sensor_start < 0 || sensor_start > nsens - nsensor))
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_init: sensor range [" + std::to_string(sensor_start) + ", " +
                                                std::to_string((long long)sensor_start + nsensor) + ") outside the model's " +
                                                std::to_string(nsens) + " sensors");
  for (int i = sensor_start; i < sensor_start + nsensor; i++)
    if (!h->sensor_why[i].empty())
      return fail(MJPC_B200_ERR_UNSUPPORTED, "plant_init: sensor " + std::to_string(i) + ": " + h->sensor_why[i]);
  CUDA_TRY(cudaSetDevice(h->device));
  const DevModel& M = h->pack.M;
  std::unique_ptr<PlantBank> k(new PlantBank);
  PlantArgs& a = k->a;
  std::memset(&a, 0, sizeof(a));
  a.B = num_plants;
  if (nsensor) {
    const DevSensor& last = h->sensors[sensor_start + nsensor - 1];
    a.sensor_adr0 = h->sensors[sensor_start].adr;
    k->nsd = last.adr - a.sensor_adr0 + sensor_dim(last.type);
    a.sensors = h->d_sensors + sensor_start; a.nsensor = nsensor; a.sensor_dim = k->nsd;
  }
  const size_t B = num_plants, nq = M.nq, nv = M.nv, nu = M.nu, nm = 7 * (size_t)M.nmocap, nts = M.task_state_size,
               nw = M.num_term, np = M.num_parameters, nsd = k->nsd;
  size_t bytes = 0;
  auto take = [&](size_t n) { const size_t at = bytes; bytes += (n + 255) & ~(size_t)255; return at; };
  const size_t nx = 6 * (size_t)M.nbody;
  const size_t o_qpos = take(B * nq * 4), o_qvel = take(B * nv * 4), o_warm = take(B * nv * 4), o_time = take(B * 8),
               o_sum = take(B * 8), o_steps = take(B * 4), o_warn = take(B * 4), o_status = take(B * 4),
               o_dist = take(B * sizeof(PlantDisturbance)), o_cnoise = take(B * nu * 4), o_xnoise = take(B * nx * 4),
               o_held = take(B * nx * 4), o_next = take(B * (nu + nx) * 4), o_sstd = take(B * nsd * 4);
  // the upload and the outputs, each one contiguous block laid out as its pinned mirror
  size_t in = 0, out = 0;
  auto in_take = [&](size_t n) { const size_t at = in; in += (n + 15) & ~(size_t)15; return at; };
  auto out_take = [&](size_t n) { const size_t at = out; out += (n + 15) & ~(size_t)15; return at; };
  k->o_ctrl = in_take(B * nu * 4); k->o_mocap = in_take(B * nm * 4); k->o_ts = in_take(B * nts * 4);
  k->o_weight = in_take(B * nw * 4); k->o_par = in_take(B * np * 4);
  k->o_time = out_take(B * 8); k->o_state = out_take(B * (nq + nv) * 4); k->o_cost = out_take(B * 4);
  k->o_status = out_take(B * 4); k->o_sens = out_take(B * nsd * 4); k->o_ctrl_out = out_take(B * nu * 4);
  k->in_bytes = in; k->out_bytes = out;
  const size_t o_in = take(in), o_out = take(out);
  auto fail_k = [&](cudaError_t e) {
    return fail(MJPC_B200_ERR_CUDA, std::string("plant_init: ") + cudaGetErrorString(e));
  };
  if (cudaError_t e = k->d_mem.alloc(bytes)) return fail_k(e);
  if (cudaError_t e = cudaMemset(k->d_mem, 0, bytes)) return fail_k(e);
  if (cudaError_t e = k->h_stage.alloc(in + out)) return fail_k(e);
  std::memset(k->h_stage, 0, in + out);
  unsigned char* base = k->d_mem;
  a.qpos = (float*)(base + o_qpos); a.qvel = (float*)(base + o_qvel); a.warm = (float*)(base + o_warm);
  a.time = (double*)(base + o_time); a.cost_sum = (double*)(base + o_sum);
  a.steps = (int*)(base + o_steps); a.warnings = (int*)(base + o_warn); a.status = (int*)(base + o_status);
  a.dist = (const PlantDisturbance*)(base + o_dist); a.ctrl_noise = (float*)(base + o_cnoise);
  a.xfrc_noise = (float*)(base + o_xnoise); a.xfrc_held = (const float*)(base + o_held); a.noise_next = (float*)(base + o_next);
  a.sensor_std = (const float*)(base + o_sstd);
  k->d_in = base + o_in; k->d_out = base + o_out;
  a.ctrl = (const float*)(k->d_in + k->o_ctrl); a.mocap = (const float*)(k->d_in + k->o_mocap);
  a.task_state = nts ? (const float*)(k->d_in + k->o_ts) : nullptr;
  a.weight = nw ? (const float*)(k->d_in + k->o_weight) : nullptr;
  a.parameters = np ? (const float*)(k->d_in + k->o_par) : nullptr;
  a.time_out = (double*)(k->d_out + k->o_time); a.state_out = (float*)(k->d_out + k->o_state);
  a.cost_out = (float*)(k->d_out + k->o_cost); a.status_out = (int*)(k->d_out + k->o_status);
  a.sensordata = nsd ? (float*)(k->d_out + k->o_sens) : nullptr;
  a.ctrl_out = (float*)(k->d_out + k->o_ctrl_out);
  std::vector<int> idle(B, PLANT_IDLE);
  if (cudaError_t e = cudaMemcpy(a.status, idle.data(), B * 4, cudaMemcpyHostToDevice)) return fail_k(e);
  // every plant starts with the handle's task (set_task), no mocap and no disturbance (the zeroed allocation);
  // plant_reset starts its episode
  k->mocap.assign(B * nm, 0.f);
  k->dist.assign(B, PlantDisturbance{});
  k->time.assign(B, 0.0);
  for (size_t b = 0; b < B; b++) {
    k->weight.insert(k->weight.end(), h->weight.begin(), h->weight.end());
    k->parameters.insert(k->parameters.end(), h->parameters.begin(), h->parameters.end());
    k->task_state.insert(k->task_state.end(), h->task_state.begin(), h->task_state.end());
  }
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // a step in flight may still use the old bank
  h->plants = std::move(k);
  return 0;
}

// the bank and one of its plants, or a refusal naming the call
static int plant_check(mjpc_b200_t* h, int plant, const char* call) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": null handle");
  if (!h->plants) return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": no plants (plant_init)");
  if (int rc = check_ensemble(h, call)) return rc;
  if (plant < 0 || plant >= h->plants->a.B)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, std::string(call) + ": plant " + std::to_string(plant) + " outside [0, " +
                                                std::to_string(h->plants->a.B) + ")");
  return 0;
}

// one plant's device fields from (write = 1) or to (write = 0) the host; NULL pointers are skipped
static int plant_fields(mjpc_b200_t* h, int b, int write, void* qpos, void* qvel, void* warm, void* time, void* cost_sum,
                        void* steps, void* warnings, void* status) {
  const PlantArgs& a = h->plants->a;
  const size_t nq = h->pack.M.nq, nv = h->pack.M.nv;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  const struct { void* host; void* dev; size_t n; } f[] = {
      {qpos, a.qpos + b * nq, nq * 4}, {qvel, a.qvel + b * nv, nv * 4}, {warm, a.warm + b * nv, nv * 4},
      {time, a.time + b, 8}, {cost_sum, a.cost_sum + b, 8}, {steps, a.steps + b, 4}, {warnings, a.warnings + b, 4},
      {status, a.status + b, 4}};
  for (const auto& x : f)
    if (x.host && x.n)
      CUDA_TRY(write ? cudaMemcpy(x.dev, x.host, x.n, cudaMemcpyHostToDevice) : cudaMemcpy(x.host, x.dev, x.n, cudaMemcpyDeviceToHost));
  return 0;
}

// zero plant b's OU states: with the step count at 0 its episode replays its seed's noise (app.cc:428-431)
static int plant_zero_noise(mjpc_b200_t* h, int b) {
  const PlantArgs& a = h->plants->a;
  const size_t nu = h->pack.M.nu, nx = 6 * (size_t)h->pack.M.nbody;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (nu) CUDA_TRY(cudaMemset(a.ctrl_noise + b * nu, 0, nu * 4));
  CUDA_TRY(cudaMemset(a.xfrc_noise + b * nx, 0, nx * 4));
  return 0;
}

int mjpc_b200_plant_reset(mjpc_b200_t* h, int plant, const float* qpos, const float* qvel, double time, const float* mocap) {
  if (int rc = plant_check(h, plant, "plant_reset")) return rc;
  const DevModel& M = h->pack.M;
  if (!qpos || !qvel || (M.nmocap && !mocap)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_reset: bad argument");
  std::vector<float> warm(M.nv, 0.f);
  double zero = 0.0;
  int izero = 0, running = PLANT_RUNNING;
  if (int rc = plant_fields(h, plant, 1, (void*)qpos, (void*)qvel, warm.data(), &time, &zero, &izero, &izero, &running))
    return rc;
  if (int rc = plant_zero_noise(h, plant)) return rc;
  PlantBank& k = *h->plants;
  const size_t nm = 7 * (size_t)M.nmocap;
  if (nm) std::copy(mocap, mocap + nm, k.mocap.begin() + plant * nm);
  k.time[plant] = time;
  return 0;
}

int mjpc_b200_plant_set(mjpc_b200_t* h, int plant, const float* qpos, const float* qvel, const float* mocap) {
  if (int rc = plant_check(h, plant, "plant_set")) return rc;
  if (int rc = plant_fields(h, plant, 1, (void*)qpos, (void*)qvel, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr))
    return rc;
  const size_t nm = 7 * (size_t)h->pack.M.nmocap;
  if (mocap && nm) std::copy(mocap, mocap + nm, h->plants->mocap.begin() + plant * nm);
  return 0;
}

int mjpc_b200_plant_set_task(mjpc_b200_t* h, int plant, const double* weight, const double* parameters,
                             const double* task_state) {
  if (int rc = plant_check(h, plant, "plant_set_task")) return rc;
  const DevModel& M = h->pack.M;
  PlantBank& k = *h->plants;
  const size_t nw = M.num_term, np = M.num_parameters, nts = M.task_state_size;
  if (weight) std::copy(weight, weight + nw, k.weight.begin() + plant * nw);
  if (parameters) std::copy(parameters, parameters + np, k.parameters.begin() + plant * np);
  if (task_state) std::copy(task_state, task_state + nts, k.task_state.begin() + plant * nts);
  return 0;
}

// One step of every plant: ONE upload from the pinned staging (ctrl, mocap, the task rows with the task state rebased
// to each plant's time), ONE plant_step_kernel launch on the handle's instance, ONE download of the outputs.
int mjpc_b200_plant_step(mjpc_b200_t* h, const float* ctrl, float* state_out, double* time_out, float* cost_out,
                         float* sensordata_out, int* status_out) {
  if (!h) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_step: null handle");
  if (!h->plants) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_step: no plants (plant_init)");
  const DevModel& M = h->pack.M;
  if (!ctrl && M.nu) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_step: ctrl required");
  PlantBank& k = *h->plants;
  PlantArgs a = k.a;
  if (int rc = check_variants(h, a.B, "plant step")) return rc;
  if (int rc = check_ensemble(h, "plant_step")) return rc;
  const size_t B = a.B, nu = M.nu, nm = 7 * (size_t)M.nmocap, nts = M.task_state_size, nw = M.num_term,
               np = M.num_parameters, ds = M.nq + M.nv;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // the staging may still feed an earlier copy
  unsigned char* in = k.h_stage;
  if (nu) std::memcpy(in + k.o_ctrl, ctrl, B * nu * 4);
  if (nm) std::memcpy(in + k.o_mocap, k.mocap.data(), B * nm * 4);
  for (size_t b = 0; b < B; b++) {
    rebase_task_state(h, k.task_state.data() + b * nts, k.time[b], (float*)(in + k.o_ts) + b * nts);
    for (size_t i = 0; i < nw; i++) ((float*)(in + k.o_weight))[b * nw + i] = (float)k.weight[b * nw + i];
    for (size_t i = 0; i < np; i++) ((float*)(in + k.o_par))[b * np + i] = (float)k.parameters[b * np + i];
  }
  CUDA_TRY(cudaMemcpyAsync(k.d_in, in, k.in_bytes, cudaMemcpyHostToDevice, h->stream));
  const KernelSet* ks;
  const int kind = pick_kernels(h, &ks);
  a.M = M; a.L = make_layout(M, 1);
  a.pack = launch_pack(h); a.pack_stride = launch_stride(h); a.pack_index = h->d_variant_index;
  a.timestep = h->pack.timestep;
  CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
  launch_kernel(ks->plant, a.B, 32, h->smem_bytes(1), h->stream, a);
  CUDA_TRY(cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  unsigned char* out = k.h_stage + k.in_bytes;
  CUDA_TRY(cudaMemcpyAsync(out, k.d_out, k.out_bytes, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  std::memcpy(k.time.data(), out + k.o_time, B * 8);
  if (time_out) std::memcpy(time_out, out + k.o_time, B * 8);
  if (state_out) std::memcpy(state_out, out + k.o_state, B * ds * 4);
  if (cost_out) std::memcpy(cost_out, out + k.o_cost, B * 4);
  if (status_out) std::memcpy(status_out, out + k.o_status, B * 4);
  if (sensordata_out && k.nsd) std::memcpy(sensordata_out, out + k.o_sens, B * k.nsd * 4);
  h->last_static = kind ? 1 : 0;
  return 0;
}

static bool finite_f(double x) { return std::isfinite(x) && std::isfinite((float)x); }

int mjpc_b200_plant_set_disturbance(mjpc_b200_t* h, int plant, double ctrl_std, double ctrl_rate, double xfrc_std,
                                    double xfrc_rate, uint32_t seed) {
  if (int rc = plant_check(h, plant, "plant_set_disturbance")) return rc;
  for (const auto& [std_, rate] : {std::pair<double, double>{ctrl_std, ctrl_rate}, {xfrc_std, xfrc_rate}}) {
    if (!finite_f(std_) || std_ < 0)
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_set_disturbance: a std must be finite and >= 0");
    if (std_ > 0 && (!finite_f(rate) || !((float)rate > 0)))
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_set_disturbance: a rate must be finite and > 0 where its std is > 0");
  }
  PlantBank& k = *h->plants;
  PlantDisturbance d = k.dist[plant];
  d.ctrl_std = (float)ctrl_std; d.ctrl_rate = (float)ctrl_rate; d.xfrc_std = (float)xfrc_std; d.xfrc_rate = (float)xfrc_rate;
  d.seed = seed;
  if (int rc = plant_zero_noise(h, plant)) return rc;
  CUDA_TRY(cudaMemcpy((PlantDisturbance*)k.a.dist + plant, &d, sizeof(d), cudaMemcpyHostToDevice));
  k.dist[plant] = d;
  return 0;
}

int mjpc_b200_plant_set_xfrc(mjpc_b200_t* h, int plant, const float* xfrc) {
  if (int rc = plant_check(h, plant, "plant_set_xfrc")) return rc;
  const size_t nx = 6 * (size_t)h->pack.M.nbody;
  std::vector<float> w(nx, 0.f);
  if (xfrc) w.assign(xfrc, xfrc + nx);
  int held = 0;
  for (float x : w) {
    if (!std::isfinite(x)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_set_xfrc: non-finite wrench");
    held |= x != 0.f;
  }
  PlantBank& k = *h->plants;
  PlantDisturbance d = k.dist[plant];
  d.held = held;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy((float*)k.a.xfrc_held + plant * nx, w.data(), nx * 4, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy((PlantDisturbance*)k.a.dist + plant, &d, sizeof(d), cudaMemcpyHostToDevice));
  k.dist[plant] = d;
  return 0;
}

// Measurement noise: the std row of plant `plant` in the bank, and its sens flag on when any entry is > 0, so that a
// plant without sensor noise steps exactly as before
int mjpc_b200_plant_set_sensor_noise(mjpc_b200_t* h, int plant, const float* std_) {
  if (int rc = plant_check(h, plant, "plant_set_sensor_noise")) return rc;
  PlantBank& k = *h->plants;
  const size_t nsd = k.nsd;
  std::vector<float> w(nsd, 0.f);
  if (std_) w.assign(std_, std_ + nsd);
  int on = 0;
  for (size_t e = 0; e < nsd; e++) {
    if (!std::isfinite(w[e]) || w[e] < 0.f)
      return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_set_sensor_noise: std[" + std::to_string(e) +
                                                  "] must be finite and >= 0");
    on |= w[e] > 0.f;
  }
  PlantDisturbance d = k.dist[plant];
  d.sens = on;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (nsd) CUDA_TRY(cudaMemcpy((float*)k.a.sensor_std + plant * nsd, w.data(), nsd * 4, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy((PlantDisturbance*)k.a.dist + plant, &d, sizeof(d), cudaMemcpyHostToDevice));
  k.dist[plant] = d;
  return 0;
}

int mjpc_b200_plant_get_disturbance(mjpc_b200_t* h, int plant, float* ctrl_noise, float* xfrc_noise) {
  if (int rc = plant_check(h, plant, "plant_get_disturbance")) return rc;
  const PlantArgs& a = h->plants->a;
  const size_t nu = h->pack.M.nu, nx = 6 * (size_t)h->pack.M.nbody;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (ctrl_noise && nu) CUDA_TRY(cudaMemcpy(ctrl_noise, a.ctrl_noise + plant * nu, nu * 4, cudaMemcpyDeviceToHost));
  if (xfrc_noise) CUDA_TRY(cudaMemcpy(xfrc_noise, a.xfrc_noise + plant * nx, nx * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int mjpc_b200_plant_last_ctrl(mjpc_b200_t* h, float* ctrl_out) {
  if (!h || !ctrl_out) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_last_ctrl: bad argument");
  if (!h->plants) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "plant_last_ctrl: no plants (plant_init)");
  if (int rc = check_ensemble(h, "plant_last_ctrl")) return rc;
  const PlantBank& k = *h->plants;
  // the last step's outputs, in the pinned staging since its download (zeros before the first step)
  std::memcpy(ctrl_out, k.h_stage + k.in_bytes + k.o_ctrl_out, (size_t)k.a.B * h->pack.M.nu * 4);
  return 0;
}

int mjpc_b200_plant_get(mjpc_b200_t* h, int plant, float* state, float* warmstart, double* time, double* cost_sum,
                        int* steps, int* warnings, int* status) {
  if (int rc = plant_check(h, plant, "plant_get")) return rc;
  const size_t nq = h->pack.M.nq;
  return plant_fields(h, plant, 0, state, state ? state + nq : nullptr, warmstart, time, cost_sum, steps, warnings, status);
}

int mjpc_b200_fetch_stats(mjpc_b200_t* h, int64_t* stats) {
  if (!h || !stats || h->lastN < 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "fetch_stats: nothing to fetch");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  const size_t rows = (size_t)h->lastN * std::max(h->last_members, 1);   // every launched trajectory
  CUDA_TRY(cudaMemcpy(stats, h->d_stats, rows * 12 * sizeof(long long), cudaMemcpyDeviceToHost));
  return 0;
}

// NoisyRollout (mjpc/trajectory.cc:100-210) for the following rollouts of this handle: Ornstein-Uhlenbeck
// xfrc_applied noise with stationary std `xfrc_std` [N, N m] and correlation time `xfrc_rate` [s]; 0 switches it off.
int mjpc_b200_set_xfrc_noise(mjpc_b200_t* h, double xfrc_std, double xfrc_rate, uint32_t seed) {
  if (!h || xfrc_std < 0 || !(xfrc_rate > 0)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_xfrc_noise: bad argument");
  h->xfrc_std = (float)xfrc_std; h->xfrc_rate = (float)xfrc_rate; h->noise_seed = seed;
  h->noise_seeds.clear();
  h->resident_ok = false;
  return MJPC_B200_OK;
}

// ... with one key per problem for the following launches of exactly B problems: problem b draws as a launch of it
// alone after set_xfrc_noise(seeds[b]) does
int mjpc_b200_set_xfrc_noise_batched(mjpc_b200_t* h, double xfrc_std, double xfrc_rate, int B, const uint32_t* seeds) {
  if (!h || xfrc_std < 0 || !(xfrc_rate > 0) || B < 1 || !seeds)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "set_xfrc_noise_batched: bad argument");
  h->xfrc_std = (float)xfrc_std; h->xfrc_rate = (float)xfrc_rate;
  h->noise_seeds.assign(seeds, seeds + B);
  h->resident_ok = false;
  return MJPC_B200_OK;
}

int64_t mjpc_b200_launch_count(const mjpc_b200_t* h) { return h ? h->launches : 0; }
float mjpc_b200_last_kernel_ms(const mjpc_b200_t* h) { return h ? h->last_ms : 0.f; }
int mjpc_b200_last_kernel_static(const mjpc_b200_t* h) { return h ? h->last_static : 0; }

// Header + state-layout words and the dof tree of a model, as the static kernel tables (spec_*.h) store them.  Host only.
int mjpc_b200_spec_words(const mjpc_model_blob* model, int* out, int capacity) {
  if (!model || !model->data || !out) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "spec_words: null");
  try {
    ModelPack P = pack_model(model->data, model->nbytes, 32, 96);
    const DevLayout L = make_layout(P.M, 1);
    const int nm = (int)(sizeof(DevModel) / 4), nl = (int)D_COUNT, nv = P.M.nv;
    if (capacity < 2 + nm + nl + nv) return fail(MJPC_B200_ERR_CAPACITY, "spec_words: buffer too small");
    out[0] = nm; out[1] = nl;
    std::memcpy(out + 2, &P.M, sizeof(DevModel));
    for (int i = 0; i < nl; i++) out[2 + nm + i] = L.off[i];
    std::memcpy(out + 2 + nm + nl, P.i.data() + P.M.io[I_dof_parentid], 4 * (size_t)nv);   // the dof tree
    return 2 + nm + nl + nv;
  } catch (const std::exception& e) {
    return fail(MJPC_B200_ERR_BAD_BLOB, std::string("spec_words: ") + e.what());
  }
}
void* mjpc_b200_stream(mjpc_b200_t* h) { return h ? (void*)h->stream : nullptr; }
float* mjpc_b200_device_returns(mjpc_b200_t* h) { return h ? h->d_returns.get() : nullptr; }

// ---- iLQG entry points (kernels in ilqg_kernels.cuh).  Each single-problem call is the B = 1 case of its batched
// twin: one staging path and one launch path per sweep.

// B rows of a double task array converted to float, as upload_task converts the handle's; empty for NULL
static std::vector<float> to_float(const double* v, size_t count) {
  return v ? std::vector<float>(v, v + count) : std::vector<float>();
}

// the derivative sweep's per-problem task states ts [B][task_state_size] and relative times trel [B][H]
static void derivative_times(mjpc_b200_t* h, int B, const double* t, const double* task_states, int H,
                             std::vector<float>* ts_out, std::vector<float>* trel_out) {
  const DevModel& M = h->pack.M;
  const size_t nts = M.task_state_size;
  std::vector<float>& ts = *ts_out;
  std::vector<float>& trel = *trel_out;
  ts.resize((size_t)B * nts); trel.resize((size_t)B * H);
  // derivative sweeps use absolute-time task state rebased to each problem's own t[0].  A time on a rollout's clock
  // (t[0] plus i timesteps in double: what rollouts record) is evaluated at that rollout step's fp32 relative time,
  // the sum of i fp32 timesteps the residuals of the rollout read, so that the Jacobians belong to the trajectory's own
  // residuals; any other time at its rounded offset from t[0].
  const float h32 = M.timestep;
  for (int b = 0; b < B; b++) {
    const double t0 = t[(size_t)b * H];
    rebase_task_state(h, task_states ? task_states + b * nts : nullptr, t0, ts.data() + b * nts);
    double clock = t0;
    float clock32 = 0.f;
    for (int i = 0; i < H; i++) {
      const double ti = t[(size_t)b * H + i];
      trel[(size_t)b * H + i] = ti == clock ? clock32 : (float)(ti - t0);
      clock += h->pack.timestep; clock32 += h32;
    }
  }
}

static int model_derivatives_impl(mjpc_b200_t* h, int B, const float* x, const float* u, const double* t,
                                  const float* mocaps, const double* weights, const double* parameters,
                                  const double* task_states, int H, int skip, float tol, int mode, float* A, float* B_,
                                  float* C, float* D) {
  const DevModel& M = h->pack.M;
  CUDA_TRY(cudaSetDevice(h->device));
  std::vector<float> ts, trel;
  derivative_times(h, B, t, task_states, H, &ts, &trel);
  const std::vector<float> w = to_float(weights, (size_t)B * M.num_term), p = to_float(parameters, (size_t)B * M.num_parameters);
  const size_t smem = h->smem_bytes(1);
  if (ilqg_reserve(h->ilqg, M, B, h->stream)) return fail(MJPC_B200_ERR_CUDA, "model_derivatives: out of device memory");
  const KernelSet* k;
  pick_kernels(h, &k);
  int launches = 0;
  int rc = ilqg_model_derivatives(h->ilqg, M, launch_pack(h), launch_stride(h), h->d_variant_index,
                                  h->stream, k->fd_center, k->fd_column, B, x, u, trel.data(), mocaps, ts.data(),
                                  weights ? w.data() : nullptr, parameters ? p.data() : nullptr, H, tol, A, B_, C, D,
                                  smem, &launches, h->ev0, h->ev1, skip, mode);
  h->launches += launches;
  if (rc == 0 && cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  if (rc) return fail(rc, "model_derivatives: CUDA failure");
  return 0;
}

int mjpc_b200_model_derivatives(mjpc_b200_t* h, const float* x, const float* u, const double* t, const float* mocap,
                                int H, int skip, float tol, int mode, float* A, float* B, float* C, float* D) {
  if (!h || !x || !u || !t || !A || !B || !C || !D) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives: null");
  if (int rc = check_variants(h, -1, "model_derivatives")) return rc;
  if (int rc = check_ensemble(h, "model_derivatives")) return rc;
  if (H < 1 || H > h->maxH || !(tol > 0)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives: bad H or tol");
  if (skip < 0 || mode < 0 || mode > 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives: bad skip or mode");
  if (h->pack.M.nmocap && !mocap) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives: mocap required");
  return model_derivatives_impl(h, 1, x, u, t, mocap, nullptr, nullptr, nullptr, H, skip, tol, mode, A, B, C, D);
}

int mjpc_b200_model_derivatives_batched(mjpc_b200_t* h, int B, const float* x, const float* u, const double* t,
                                        const float* mocaps, const double* weights, const double* parameters,
                                        const double* task_states, int H, int skip, float tol, int mode, float* A,
                                        float* B_, float* C, float* D) {
  if (!h || !x || !u || !t || !A || !B_ || !C || !D) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives_batched: null");
  if (B < 1 || H < 1 || !(tol > 0)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives_batched: bad B, H or tol");
  if (H > h->maxH) return fail(MJPC_B200_ERR_CAPACITY, "model_derivatives_batched: H above max_horizon");
  if (skip < 0 || mode < 0 || mode > 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives_batched: bad skip or mode");
  if (h->pack.M.nmocap && !mocaps) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "model_derivatives_batched: mocap required");
  if (int rc = check_variants(h, B, "model_derivatives_batched")) return rc;
  if (int rc = check_ensemble(h, "model_derivatives_batched")) return rc;
  return model_derivatives_impl(h, B, x, u, t, mocaps, weights, parameters, task_states, H, skip, tol, mode, A, B_, C, D);
}

static int cost_derivatives_impl(mjpc_b200_t* h, int B, const double* weights, const float* residual, const float* C,
                                 const float* D, int H, float* cx, float* cu, float* cxx, float* cuu, float* cxu) {
  const DevModel& M = h->pack.M;
  CUDA_TRY(cudaSetDevice(h->device));
  if (cost_derivatives_smem(M, h->max_term_dim) > h->smem_optin)
    return fail(MJPC_B200_ERR_CAPACITY, "cost_derivatives: the widest cost term does not fit in shared memory");
  const std::vector<float> w = to_float(weights, (size_t)B * M.num_term);
  if (ilqg_reserve(h->ilqg, M, B, h->stream)) return fail(MJPC_B200_ERR_CUDA, "cost_derivatives: out of device memory");
  int launches = 0;
  int rc = ilqg_cost_derivatives(h->ilqg, M, h->d_pack, h->stream, B, weights ? w.data() : nullptr, residual, C, D, H,
                                 cx, cu, cxx, cuu, cxu, h->max_term_dim, &launches, h->ev0, h->ev1);
  h->launches += launches;
  if (rc == 0 && cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  if (rc) return fail(rc, "cost_derivatives: CUDA failure");
  return 0;
}

int mjpc_b200_cost_derivatives(mjpc_b200_t* h, const float* residual, const float* C, const float* D, int H,
                               float* cx, float* cu, float* cxx, float* cuu, float* cxu) {
  if (!h || !residual || !C || !D || !cx || !cu || !cxx || !cuu || !cxu)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "cost_derivatives: null");
  if (int rc = check_variants(h, -1, "cost_derivatives")) return rc;
  if (H < 1 || H > h->maxH) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "cost_derivatives: bad H");
  return cost_derivatives_impl(h, 1, nullptr, residual, C, D, H, cx, cu, cxx, cuu, cxu);
}

int mjpc_b200_cost_derivatives_batched(mjpc_b200_t* h, int B, const double* weights, const float* residual, const float* C,
                                       const float* D, int H, float* cx, float* cu, float* cxx, float* cuu, float* cxu) {
  if (!h || !residual || !C || !D || !cx || !cu || !cxx || !cuu || !cxu)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "cost_derivatives_batched: null");
  if (B < 1 || H < 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "cost_derivatives_batched: bad B or H");
  if (H > h->maxH) return fail(MJPC_B200_ERR_CAPACITY, "cost_derivatives_batched: H above max_horizon");
  return cost_derivatives_impl(h, B, weights, residual, C, D, H, cx, cu, cxx, cuu, cxu);
}

int mjpc_b200_gradient_batched(mjpc_b200_t* h, int B, const float* x, const float* u, const double* t,
                               const float* mocaps, const double* weights, const double* parameters,
                               const double* task_states, const float* residual, int H, int skip, float tol, int mode,
                               double* k, double* dV0) {
  if (!h || !x || !u || !t || !residual || !k || !dV0) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "gradient_batched: null");
  if (B < 1 || H < 2 || !(tol > 0)) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "gradient_batched: bad B, H or tol");
  if (H > h->maxH) return fail(MJPC_B200_ERR_CAPACITY, "gradient_batched: H above max_horizon");
  if (skip < 0 || mode < 0 || mode > 1) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "gradient_batched: bad skip or mode");
  if (h->pack.M.nmocap && !mocaps) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "gradient_batched: mocap required");
  if (int rc = check_variants(h, B, "gradient_batched")) return rc;
  if (int rc = check_ensemble(h, "gradient_batched")) return rc;
  const DevModel& M = h->pack.M;
  CUDA_TRY(cudaSetDevice(h->device));
  if (cost_derivatives_smem(M, h->max_term_dim) > h->smem_optin)
    return fail(MJPC_B200_ERR_CAPACITY, "gradient_batched: the widest cost term does not fit in shared memory");
  std::vector<float> ts, trel;
  derivative_times(h, B, t, task_states, H, &ts, &trel);
  const std::vector<float> w = to_float(weights, (size_t)B * M.num_term), p = to_float(parameters, (size_t)B * M.num_parameters);
  if (ilqg_reserve(h->ilqg, M, B, h->stream)) return fail(MJPC_B200_ERR_CUDA, "gradient_batched: out of device memory");
  const KernelSet* ks;
  pick_kernels(h, &ks);
  // the two derivative sweeps exactly as their batched entry points stage them, except that A, B, C, D and the cost
  // derivatives stay on the device; one span from the first kernel to the sweep's end
  int launches = 0;
  int rc = ilqg_model_derivatives(h->ilqg, M, launch_pack(h), launch_stride(h), h->d_variant_index,
                                  h->stream, ks->fd_center, ks->fd_column, B, x, u, trel.data(),
                                  mocaps, ts.data(), weights ? w.data() : nullptr, parameters ? p.data() : nullptr, H,
                                  tol, nullptr, nullptr, nullptr, nullptr, h->smem_bytes(1), &launches, h->ev0,
                                  nullptr, skip, mode);
  if (rc == 0)
    rc = ilqg_cost_derivatives(h->ilqg, M, h->d_pack, h->stream, B, weights ? w.data() : nullptr, residual, nullptr,
                               nullptr, H, nullptr, nullptr, nullptr, nullptr, nullptr, h->max_term_dim, &launches,
                               nullptr, nullptr, true);
  if (rc == 0) rc = ilqg_gradient_sweep(h->ilqg, h->stream, B, H, k, dV0, &launches, h->ev1);
  h->launches += launches;
  if (rc == 0 && cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  if (rc) return fail(rc, "gradient_batched: CUDA failure");
  return 0;
}

static int backward_pass_impl(mjpc_b200_t* h, int B, const float* A, const float* B_, const float* cx, const float* cu,
                              const float* cxx, const float* cxu, const float* cuu, const float* actions, int H,
                              const float* mu, int reg_type, int limits, float* K, float* du, float* dV, float* Vx,
                              float* Vxx, int* status_out) {
  CUDA_TRY(cudaSetDevice(h->device));
  if (ilqg_reserve(h->ilqg, h->pack.M, B, h->stream)) return fail(MJPC_B200_ERR_CUDA, "backward_pass: out of device memory");
  int launches = 0;
  int rc = ilqg_backward_pass(h->ilqg, h->pack.M, h->d_pack, h->stream, B, A, B_, cx, cu, cxx, cxu, cuu, actions, H, mu,
                              reg_type, limits, K, du, dV, Vx, Vxx, status_out, &launches, h->ev0, h->ev1);
  h->launches += launches;
  if (rc == 0 && cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1) != cudaSuccess) cudaGetLastError();
  if (rc) return fail(rc, "backward_pass: CUDA failure");
  return 0;
}

int mjpc_b200_backward_pass(mjpc_b200_t* h, const float* A, const float* B, const float* cx, const float* cu,
                            const float* cxx, const float* cxu, const float* cuu, const float* actions, int H,
                            float mu, int reg_type, int limits, float* K, float* du, float* dV, float* Vx, float* Vxx,
                            int* status_out) {
  if (!h || !A || !B || !cx || !cu || !cxx || !cxu || !cuu || !actions || !K || !du || !dV || !status_out)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "backward_pass: null");
  if (int rc = check_variants(h, -1, "backward_pass")) return rc;
  if (H < 2 || H > h->maxH) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "backward_pass: bad H");
  return backward_pass_impl(h, 1, A, B, cx, cu, cxx, cxu, cuu, actions, H, &mu, reg_type, limits, K, du, dV, Vx, Vxx,
                            status_out);
}

int mjpc_b200_backward_pass_batched(mjpc_b200_t* h, int B, const float* A, const float* B_, const float* cx,
                                    const float* cu, const float* cxx, const float* cxu, const float* cuu,
                                    const float* actions, int H, const float* mu, int reg_type, int limits, float* K,
                                    float* du, float* dV, float* Vx, float* Vxx, int* status) {
  if (!h || !A || !B_ || !cx || !cu || !cxx || !cxu || !cuu || !actions || !mu || !K || !du || !dV || !status)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "backward_pass_batched: null");
  if (B < 1 || H < 2) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "backward_pass_batched: bad B or H");
  if (H > h->maxH) return fail(MJPC_B200_ERR_CAPACITY, "backward_pass_batched: H above max_horizon");
  return backward_pass_impl(h, B, A, B_, cx, cu, cxx, cxu, cuu, actions, H, mu, reg_type, limits, K, du, dV, Vx, Vxx, status);
}

}  // extern "C"

// ---- the state estimators' filter bank (filter_bank.h, kernels in estimator_kernels.cuh)
namespace mjpc_b200_bank {

int Init(mjpc_b200_t* h, const Desc& d) {
  if (!h || (d.kind != kFilterKalman && d.kind != kFilterUnscented) || d.num_filters < 1 || d.rows < 1 || d.njnt < 0)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank: bad argument");
  const DevModel& M = h->pack.M;
  const int nsens = (int)h->sensors.size();
  if (d.sensor_start < 0 || d.nsensor < 1 || d.sensor_start > nsens - d.nsensor)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank: sensor range outside the model's sensors");
  for (int i = d.sensor_start; i < d.sensor_start + d.nsensor; i++)
    if (!h->sensor_why[i].empty())
      return fail(MJPC_B200_ERR_UNSUPPORTED, "filter bank: sensor " + std::to_string(i) + ": " + h->sensor_why[i]);
  if ((int64_t)d.num_filters * d.rows > h->maxN) return fail(MJPC_B200_ERR_CAPACITY, "filter bank: rows above max_candidates");
  CUDA_TRY(cudaSetDevice(h->device));
  std::unique_ptr<FilterBank> k(new FilterBank);
  FilterBankArgs& a = k->a;
  std::memset(&a, 0, sizeof(a));
  a.nq = M.nq; a.nv = M.nv; a.nu = M.nu; a.nmocap = M.nmocap; a.njnt = d.njnt;
  a.kind = d.kind; a.B = d.num_filters; a.rows = d.rows;
  a.timestep = d.timestep; a.sigma_step = d.sigma_step; a.weight_mean0 = d.weight_mean0;
  a.weight_covariance0 = d.weight_covariance0; a.weight_sigma = d.weight_sigma; a.epsilon = d.epsilon;
  a.centered = d.centered;
  k->s0 = d.sensor_start; k->nsens = d.nsensor;
  k->adr0 = h->sensors[d.sensor_start].adr;
  const DevSensor& last = h->sensors[d.sensor_start + d.nsensor - 1];
  k->nsd = last.adr - k->adr0 + sensor_dim(last.type);
  a.ny = k->nsd;
  const size_t B = a.B, R = (size_t)a.B * a.rows, nq = a.nq, nv = a.nv, nx = nq + nv, ns = 2 * nv, ny = a.ny,
               nu = a.nu, nm = 7 * (size_t)a.nmocap, nr = std::max(M.num_residual, 1), nts = M.task_state_size;
  const size_t scratch = filter_scratch_layout(a);
  // carve one allocation, every piece 256-byte aligned
  size_t bytes = 0;
  auto take = [&](size_t n) { const size_t at = bytes; bytes += (n + 255) & ~(size_t)255; return at; };
  const size_t o_jnt = take(3 * (size_t)d.njnt * 4), o_state = take(B * nx * 8), o_P = take(B * ns * ns * 8),
               o_time = take(B * 8), o_np = take(B * ns * 8), o_ns = take(B * ny * 8), o_warm = take(B * nv * 4),
               o_warn = take(B * 4), o_status = take(B * 4);
  k->in_bytes = B * ny * 8 + B * nu * 4 + B * nm * 4;
  const size_t o_in = take(k->in_bytes), o_qpos = take(R * nq * 4), o_qvel = take(R * nv * 4),
               o_rctrl = take(R * nu * 4), o_rwarm = take(R * nv * 4), o_rmocap = take(R * nm * 4),
               o_rtime = take(R * 4), o_task = take(nts * 4), o_qacc = take(R * nv * 4), o_nq = take(R * nq * 4),
               o_nv = take(R * nv * 4), o_res = take(R * nr * 4), o_cost = take(R * 4), o_counts = take(4 * R * 4),
               o_sens = take(R * ny * 4), o_scratch = take(B * scratch * 8);
  auto fail_k = [&](cudaError_t e) {
    return fail(MJPC_B200_ERR_CUDA, std::string("filter bank: ") + cudaGetErrorString(e));
  };
  if (cudaError_t e = k->d_mem.alloc(bytes)) return fail_k(e);
  if (cudaError_t e = cudaMemset(k->d_mem, 0, bytes)) return fail_k(e);
  if (cudaError_t e = k->h_stage.alloc(k->in_bytes + B * 4)) return fail_k(e);
  unsigned char* base = k->d_mem;
  auto at = [&](size_t o) { return (void*)(base + o); };
  a.jnt = (const int*)at(o_jnt);
  a.state = (double*)at(o_state); a.P = (double*)at(o_P); a.time = (double*)at(o_time);
  a.noise_process = (double*)at(o_np); a.noise_sensor = (double*)at(o_ns); a.warm = (float*)at(o_warm);
  a.warnings = (int*)at(o_warn); a.status = (int*)at(o_status);
  k->d_in = (unsigned char*)at(o_in);
  a.sensor = (const double*)k->d_in; a.ctrl = (const float*)(k->d_in + B * ny * 8);
  a.mocap = (const float*)(k->d_in + B * ny * 8 + B * nu * 4);
  a.qpos = (float*)at(o_qpos); a.qvel = (float*)at(o_qvel); a.rctrl = (float*)at(o_rctrl); a.rwarm = (float*)at(o_rwarm);
  a.rmocap = (float*)at(o_rmocap); k->d_rtime = (float*)at(o_rtime); k->d_task = (float*)at(o_task);
  a.qacc = (const float*)at(o_qacc); a.next_qpos = (const float*)at(o_nq); a.next_qvel = (const float*)at(o_nv);
  k->d_res = (float*)at(o_res); k->d_cost = (float*)at(o_cost); a.counts = (const int*)at(o_counts);
  a.sensordata = (const float*)at(o_sens); a.scratch = (double*)at(o_scratch);
  // the joints, and the task state at time 0: every row steps at device time 0 (the residual, which reads them, does
  // not feed the filters)
  std::vector<int> jnt(3 * (size_t)d.njnt);
  for (int j = 0; j < d.njnt; j++) {
    jnt[j] = d.jnt_type[j]; jnt[d.njnt + j] = d.jnt_qposadr[j]; jnt[2 * d.njnt + j] = d.jnt_dofadr[j];
  }
  std::vector<float> ts(nts);
  rebase_task_state(h, nullptr, 0.0, ts.data());
  if (cudaError_t e = cudaMemcpy((void*)a.jnt, jnt.data(), jnt.size() * 4, cudaMemcpyHostToDevice)) return fail_k(e);
  if (nts)
    if (cudaError_t e = cudaMemcpy(k->d_task, ts.data(), nts * 4, cudaMemcpyHostToDevice)) return fail_k(e);
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // an update in flight may still use the old bank
  h->bank = std::move(k);
  return 0;
}

int Access(mjpc_b200_t* h, int b, int field, void* data, int write) {
  if (!h || !h->bank || !data || b < 0 || b >= h->bank->a.B) return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank: bad access");
  const FilterBankArgs& a = h->bank->a;
  const size_t nx = a.nq + a.nv, ns = 2 * a.nv;
  void* p;
  size_t n;
  switch (field) {
    case STATE: p = a.state + b * nx; n = nx * 8; break;
    case COVARIANCE: p = a.P + b * ns * ns; n = ns * ns * 8; break;
    case TIME: p = a.time + b; n = 8; break;
    case NOISE_PROCESS: p = a.noise_process + b * ns; n = ns * 8; break;
    case NOISE_SENSOR: p = a.noise_sensor + (size_t)b * a.ny; n = (size_t)a.ny * 8; break;
    case WARMSTART: p = a.warm + b * (size_t)a.nv; n = (size_t)a.nv * 4; break;
    case WARNINGS: p = a.warnings + b; n = 4; break;
    default: return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank: bad field");
  }
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(write ? cudaMemcpy(p, data, n, cudaMemcpyHostToDevice) : cudaMemcpy(data, p, n, cudaMemcpyDeviceToHost));
  return 0;
}

// the step launch of every filter's rows, as step_impl launches one (inputs and outputs already on the device)
static int step_rows(mjpc_b200_t* h, const KernelSet* ks) {
  FilterBank& k = *h->bank;
  const FilterBankArgs& a = k.a;
  StepBatchArgs A;
  std::memset(&A, 0, sizeof(A));
  A.M = h->pack.M; A.L = make_layout(h->pack.M, 1);
  A.pack = launch_pack(h); A.pack_stride = launch_stride(h); A.pack_rows = a.rows; A.pack_index = h->d_variant_index;
  A.qpos = a.qpos; A.qvel = a.qvel; A.ctrl = a.rctrl; A.warmstart = a.rwarm;
  A.mocap = a.rmocap; A.mocap_stride = 7 * a.nmocap;
  A.task_state = h->pack.M.task_state_size ? k.d_task : nullptr; A.time = k.d_rtime; A.B = a.B * a.rows;
  A.qacc = (float*)a.qacc; A.next_qpos = (float*)a.next_qpos; A.next_qvel = (float*)a.next_qvel;
  A.residual = k.d_res; A.cost = k.d_cost; A.counts = (int*)a.counts;
  A.sensors = h->d_sensors + k.s0; A.nsensor = k.nsens; A.sensor_adr0 = k.adr0; A.sensor_dim = k.nsd;
  A.sensordata = (float*)a.sensordata;
  launch_kernel(ks->step, A.B, 32, h->smem_bytes(1), h->stream, A);
  h->launches += 1;
  return 0;
}

// the update inputs into the bank: sensor [B][ny], ctrl [B][nu], mocap [B][7 nmocap]; a NULL one keeps what the last
// staging left
static int stage_inputs(mjpc_b200_t* h, const float* ctrl, const double* sensor, const float* mocap) {
  FilterBank& k = *h->bank;
  const FilterBankArgs& a = k.a;
  const size_t B = a.B, ny = a.ny, nu = a.nu, nm = 7 * (size_t)a.nmocap;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));   // the staging may still feed an earlier copy
  if (sensor) std::memcpy(k.h_stage, sensor, B * ny * 8);
  if (nu && ctrl) std::memcpy(k.h_stage + B * ny * 8, ctrl, B * nu * 4);
  if (nm && mocap) std::memcpy(k.h_stage + B * ny * 8 + B * nu * 4, mocap, B * nm * 4);
  CUDA_TRY(cudaMemcpyAsync(k.d_in, k.h_stage, k.in_bytes, cudaMemcpyHostToDevice, h->stream));
  return 0;
}

// The kernels of one phase (0 Unscented, 1 Kalman measurement, 2 Kalman prediction) on every filter: the step rows
// before the step launch, and the update after it
static void run_filter_kernel(mjpc_b200_t* h, int phase, const void* fn) {
  FilterBankArgs a = h->bank->a;
  a.phase = phase;
  void* args[] = {&a};
  cudaLaunchKernel(fn, dim3(a.B), dim3(kFilterThreads), args, 0, h->stream);
  h->launches += 1;
}
static void launch_phase_rows(mjpc_b200_t* h, int phase) { run_filter_kernel(h, phase, (const void*)estimator_rows_kernel); }
static void launch_phase_update(mjpc_b200_t* h, int phase) {
  run_filter_kernel(h, phase, phase == 0 ? (const void*)unscented_update_kernel
                              : phase == 1 ? (const void*)kalman_measurement_kernel : (const void*)kalman_prediction_kernel);
}

// the statuses [B] of the last kernels, after the stream's work
static int read_status(mjpc_b200_t* h, int* status) {
  FilterBank& k = *h->bank;
  CUDA_TRY(cudaGetLastError());
  int* st = (int*)(k.h_stage + k.in_bytes);
  CUDA_TRY(cudaMemcpyAsync(st, k.a.status, k.a.B * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::copy(st, st + k.a.B, status);
  return 0;
}

int Update(mjpc_b200_t* h, const float* ctrl, const double* sensor, const float* mocap, int phases, int* status) {
  if (!h || !h->bank || phases < MEASUREMENT || phases > MEASUREMENT_AND_PREDICTION || (!ctrl && h->pack.M.nu) ||
      (!sensor && (h->bank->a.kind == kFilterUnscented || (phases & MEASUREMENT))) || (!mocap && h->pack.M.nmocap) ||
      !status)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank update: bad argument");
  const FilterBankArgs& a = h->bank->a;
  if (int rc = check_variants(h, a.B, "filter bank update")) return rc;
  if (int rc = check_ensemble(h, "filter bank update")) return rc;
  if (int rc = stage_inputs(h, ctrl, sensor, mocap)) return rc;
  const KernelSet* ks;
  const int kind = pick_kernels(h, &ks);
  auto run = [&](int phase) {
    launch_phase_rows(h, phase);
    step_rows(h, ks);
    launch_phase_update(h, phase);
  };
  if (a.kind == kFilterUnscented) {
    run(0);
  } else {
    if (phases & MEASUREMENT) {
      run(1);
    } else {   // the prediction skips a failed filter: clear the statuses an earlier update left
      CUDA_TRY(cudaMemsetAsync(a.status, 0, a.B * 4, h->stream));
    }
    if (phases & PREDICTION) run(2);
  }
  if (int rc = read_status(h, status)) return rc;
  h->last_static = kind ? 1 : 0;
  return 0;
}

// whether the bank's kind runs `phase`
static bool bank_phase(const mjpc_b200_t* h, int phase) {
  return h && h->bank && (h->bank->a.kind == kFilterUnscented ? phase == 0 : phase == 1 || phase == 2);
}

int DebugRows(mjpc_b200_t* h, int phase, const float* ctrl, const float* mocap, float* qpos, float* qvel, float* warm,
              int* status) {
  if (!bank_phase(h, phase) || (!ctrl && h->pack.M.nu) || (!mocap && h->pack.M.nmocap) || !qpos || !qvel || !warm ||
      !status)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank debug_rows: bad argument");
  const FilterBankArgs& a = h->bank->a;
  const size_t R = (size_t)a.B * a.rows;
  if (int rc = stage_inputs(h, ctrl, nullptr, mocap)) return rc;
  launch_phase_rows(h, phase);
  CUDA_TRY(cudaMemcpyAsync(qpos, a.qpos, R * a.nq * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(qvel, a.qvel, R * a.nv * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(warm, a.rwarm, R * a.nv * 4, cudaMemcpyDeviceToHost, h->stream));
  return read_status(h, status);
}

int DebugFinish(mjpc_b200_t* h, int phase, const double* sensor, const float* next_qpos, const float* next_qvel,
                const float* qacc, const float* sensordata, const int* counts, int* status) {
  if (!bank_phase(h, phase) || (!sensor && phase < 2) || !next_qpos || !next_qvel || !qacc || !sensordata || !counts ||
      !status)
    return fail(MJPC_B200_ERR_BAD_ARGUMENT, "filter bank debug_finish: bad argument");
  const FilterBankArgs& a = h->bank->a;
  const size_t R = (size_t)a.B * a.rows;
  if (int rc = stage_inputs(h, nullptr, sensor, nullptr)) return rc;
  CUDA_TRY(cudaMemsetAsync(a.status, 0, a.B * 4, h->stream));
  CUDA_TRY(cudaMemcpyAsync((void*)a.next_qpos, next_qpos, R * a.nq * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync((void*)a.next_qvel, next_qvel, R * a.nv * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync((void*)a.qacc, qacc, R * a.nv * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync((void*)a.sensordata, sensordata, R * a.ny * 4, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync((void*)a.counts, counts, R * 4 * 4, cudaMemcpyHostToDevice, h->stream));
  launch_phase_update(h, phase);
  return read_status(h, status);
}

}  // namespace mjpc_b200_bank
