// dev_model.h - packed, read-only model/task constants as the kernels see them, and the host-side packer
// that builds them from the model blob (mujoco_mpc_b200/blob.py).
//
// HBM layout: ONE contiguous float array + ONE contiguous int array per model ("model pack"), staged into
// shared memory once per CTA with a 1-D TMA bulk copy (cp.async.bulk, csrc/rollout_kernels.cu).  The
// DevModel header (sizes + offsets into the two arrays) travels as a __grid_constant__ kernel parameter.
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace mjpc_dev {

// ---- float arrays copied verbatim from the blob (converted double -> float)
#define MJPC_F_ARRAYS(X)                                                                                         \
  X(body_pos) X(body_quat) X(body_ipos) X(body_iquat) X(body_mass) X(body_inertia) X(body_subtreemass)           \
  X(body_invweight0) X(jnt_pos) X(jnt_axis) X(jnt_range) X(jnt_stiffness) X(jnt_margin) X(jnt_solref)            \
  X(jnt_solimp) X(qpos0) X(qpos_spring) X(dof_damping) X(dof_armature) X(dof_frictionloss) X(dof_solref)         \
  X(dof_solimp) X(dof_invweight0) X(geom_size) X(geom_pos) X(geom_quat) X(geom_friction) X(geom_solmix)          \
  X(geom_solref) X(geom_solimp) X(geom_margin) X(geom_gap) X(geom_rbound) X(site_pos) X(site_quat)               \
  X(actuator_gear) X(actuator_gainprm) X(actuator_biasprm) X(actuator_ctrlrange) X(actuator_forcerange)          \
  X(key_qpos) X(task_weight) X(task_norm_parameter) X(task_parameters) X(task_state) X(wrap_coef) X(tendon_range)     \
  X(tendon_margin) X(tendon_solref) X(tendon_solimp) X(tendon_invweight0)
// ---- int arrays copied verbatim from the blob
#define MJPC_I_ARRAYS(X)                                                                                         \
  X(body_parentid) X(body_rootid) X(body_jntnum) X(body_jntadr) X(body_dofnum) X(body_dofadr) X(body_mocapid)    \
  X(jnt_type) X(jnt_qposadr) X(jnt_dofadr) X(jnt_bodyid) X(jnt_limited) X(dof_bodyid) X(dof_jntid)               \
  X(dof_parentid) X(geom_type) X(geom_bodyid) X(geom_condim) X(geom_priority) X(site_bodyid) X(actuator_trnid) X(actuator_trntype)  \
  X(actuator_biastype) X(actuator_ctrllimited) X(actuator_forcelimited) X(pair_geom1) X(pair_geom2)              \
  X(ray_geoms) X(task_dim_norm_residual) X(task_norm) X(task_num_norm_parameter) X(task_trace_objtype)           \
  X(task_trace_objid) X(task_ids) X(tendon_adr) X(tendon_num) X(tendon_limited) X(wrap_dof) X(wrap_qposadr)
// ---- int arrays derived on the host for warp-parallel traversal
//   level_adr/level_body : bodies grouped by tree depth (lanes work on one level at a time)
//   body_subtreeend      : DFS order => subtree of b is the contiguous range [b, body_subtreeend[b])
//   body_lastdof         : last dof of the nearest ancestor-or-self that has dofs (-1 if none)
//   body_dofmask_lo/hi   : bitmask of the dofs on the chain from the root to the body
//   mpair_i/mpair_j      : (dof, ancestor-or-self dof) pairs = the structurally non-zero entries of M
//   floss_dof            : dofs with frictionloss > 0;  limit_jnt: limited slide/hinge joints
//   hpair_i/hpair_j      : structurally non-zero lower-triangle entries of the Newton Hessian M + J^T D J:
//                          the M pattern plus (chain(b1) u chain(b2))^2 for every dynamic-dynamic geom pair
//   floss_row            : constraint row of each dof's friction-loss constraint (-1 if none)
//   chain_adr/num/dof    : dofs on the chain root -> body, in root-to-leaf order (compact contact Jacobians)
#define MJPC_I_DERIVED(X)                                                                                        \
  X(level_adr) X(level_body) X(body_subtreeend) X(body_lastdof) X(body_dofmask_lo) X(body_dofmask_hi)            \
  X(mpair_i) X(mpair_j) X(floss_dof) X(limit_jnt) X(hpair_i) X(hpair_j) X(floss_row) X(chain_adr) X(chain_num) X(chain_dof)

enum FloatArrayId {
#define X(n) F_##n,
  MJPC_F_ARRAYS(X)
#undef X
      F_COUNT
};
enum IntArrayId {
#define X(n) I_##n,
  MJPC_I_ARRAYS(X) MJPC_I_DERIVED(X)
#undef X
      I_COUNT
};

enum { GEOM_PLANE = 0, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX };
enum { JNT_FREE = 0, JNT_BALL, JNT_SLIDE, JNT_HINGE };
enum { OBJ_BODY = 0, OBJ_XBODY, OBJ_GEOM, OBJ_SITE };
enum { CONE_PYRAMIDAL = 0, CONE_ELLIPTIC = 1 };
enum { RESIDUAL_PARTICLE = 0, RESIDUAL_PARTICLE_COPY = 1, RESIDUAL_CARTPOLE = 2, RESIDUAL_QUADRUPED_FLAT = 3,
       RESIDUAL_HUMANOID_STAND = 4, RESIDUAL_HUMANOID_TRACK = 5, RESIDUAL_SHADOW_REORIENT = 6,
       RESIDUAL_NONE = 7 /* no cost terms: k_residual writes nothing */ };

// integer fields of the header (sizes, option flags, task dimensions, pack sizes).  A statically specialised
// kernel (spec_*.h) turns every one of them, and the offset tables below, into compile-time constants.
#define MJPC_M_INTS(X)                                                                                           \
  X(nq) X(nv) X(nu) X(nbody) X(njnt) X(ngeom) X(nsite) X(nmocap) X(nkey) X(npair) X(nray) X(nlevel) X(nmpair)    \
  X(ntendon)                                                                                                     \
  X(nfloss) X(nlimit) X(nhpair) X(cone) X(iterations) X(ls_iterations) X(disable_contact) X(disable_eulerdamp)  \
  X(disable_frictionloss) X(disable_limit) X(disable_refsafe) X(disable_warmstart) X(maxcon) X(maxefc)           \
  X(residual_id) X(num_residual) X(num_term) X(num_trace) X(num_parameters) X(task_state_size) X(any_damping)    \
  X(nf) X(ni)

struct DevModel {
#define X(n) int n;
  MJPC_M_INTS(X)       // nf, ni: total floats / ints in the pack
#undef X
  float timestep, impratio, tolerance, ls_tolerance, meaninertia, risk;   // always read from the live header
  float differentiable;   // != 0: MakeDifferentiable (utilities.cc:60-75) - solimp[0] of joints and geoms reads as 0
  float gravity[3];
  int fo[F_COUNT];     // offsets (floats)
  int io[I_COUNT];     // offsets (ints)
};

// ---- host side ------------------------------------------------------------------------------------------
struct Blob {
  const uint8_t* p;
  size_t n;
  int nent;
  Blob(const void* data, size_t nbytes) : p((const uint8_t*)data), n(nbytes), nent(0) {
    if (!data || nbytes < 16 || std::memcmp(p, "MJPCB200", 8) != 0) throw std::runtime_error("bad model blob magic");
    std::memcpy(&nent, p + 12, 4);
    if ((size_t)16 + 56 * (size_t)nent > nbytes) throw std::runtime_error("truncated model blob");
  }
  bool find(const char* name, int* dt, int* cnt, int64_t* off) const {
    for (int i = 0; i < nent; i++) {
      const uint8_t* e = p + 16 + 56 * (size_t)i;
      if (std::strncmp((const char*)e, name, 40) == 0) {
        std::memcpy(dt, e + 40, 4); std::memcpy(cnt, e + 44, 4); std::memcpy(off, e + 48, 8);
        if ((size_t)*off + (size_t)*cnt * (*dt ? 8 : 4) > n) throw std::runtime_error("blob entry out of range");
        return true;
      }
    }
    return false;
  }
  std::vector<int> ints(const char* name) const {
    int dt, c; int64_t off;
    if (!find(name, &dt, &c, &off) || dt != 0) throw std::runtime_error(std::string("blob: missing int array ") + name);
    std::vector<int> v(c);
    if (c) std::memcpy(v.data(), p + off, 4 * (size_t)c);
    return v;
  }
  std::vector<double> reals(const char* name) const {
    int dt, c; int64_t off;
    if (!find(name, &dt, &c, &off) || dt != 1) throw std::runtime_error(std::string("blob: missing real array ") + name);
    std::vector<double> v(c);
    if (c) std::memcpy(v.data(), p + off, 8 * (size_t)c);
    return v;
  }
  int i(const char* name) const { return ints(name).at(0); }
  double r(const char* name) const { return reals(name).at(0); }
};

struct ModelPack {
  DevModel M;
  std::vector<float> f;
  std::vector<int> i;
  std::vector<double> key_mpos, key_mquat, qpos0;
  double timestep = 0;   // opt.timestep in double: the rollout clock of the policy step table (M.timestep is its fp32)
};

inline ModelPack pack_model(const void* data, size_t nbytes, int maxcon, int maxefc) {
  Blob b(data, nbytes);
  ModelPack P;
  DevModel& M = P.M;
  std::memset(&M, 0, sizeof(M));
  M.nq = b.i("nq"); M.nv = b.i("nv"); M.nu = b.i("nu"); M.nbody = b.i("nbody"); M.njnt = b.i("njnt");
  M.ngeom = b.i("ngeom"); M.nsite = b.i("nsite"); M.nmocap = b.i("nmocap"); M.nkey = b.i("nkey");
  M.npair = b.i("npair"); M.ntendon = b.i("ntendon");
  if (b.i("na") != 0) throw std::runtime_error("actuator activations (na > 0) are not supported");
  M.cone = b.i("opt_cone"); M.iterations = b.i("opt_iterations"); M.ls_iterations = b.i("opt_ls_iterations");
  if (b.i("opt_integrator") != 0) throw std::runtime_error("only the Euler integrator is implemented");
  M.disable_contact = b.i("opt_disable_contact"); M.disable_eulerdamp = b.i("opt_disable_eulerdamp");
  M.disable_frictionloss = b.i("opt_disable_frictionloss"); M.disable_limit = b.i("opt_disable_limit");
  M.disable_refsafe = b.i("opt_disable_refsafe"); M.disable_warmstart = b.i("opt_disable_warmstart");
  // contact slots: maxcon geometric contacts, then two per fixed tendon for its limit pseudo-contacts (k_collision)
  M.maxcon = maxcon + 2 * M.ntendon; M.maxefc = maxefc;
  M.residual_id = b.i("task_residual_id"); M.num_residual = b.i("task_num_residual");
  M.num_term = b.i("task_num_term"); M.num_trace = b.i("task_num_trace");
  P.timestep = b.r("opt_timestep");
  M.timestep = (float)P.timestep; M.impratio = (float)b.r("opt_impratio");
  M.tolerance = (float)b.r("opt_tolerance"); M.ls_tolerance = (float)b.r("opt_ls_tolerance");
  M.meaninertia = (float)b.r("stat_meaninertia"); M.risk = (float)b.r("task_risk");
  auto g = b.reals("opt_gravity");
  for (int k = 0; k < 3; k++) M.gravity[k] = (float)g[k];
  // verbatim arrays
  // keyframe tables of mocap tasks (thousands of frames) do not fit the shared-memory pack: they stay in HBM
  // (engine.cu appends key_mpos behind the staged pack); residuals that index key_qpos need nkey small
#define X(n) { auto v = b.reals(#n); if (std::string(#n) == "key_qpos" && v.size() > 1024) v.clear();               \
               M.fo[F_##n] = (int)P.f.size(); for (double x : v) P.f.push_back((float)x);                          \
               while (P.f.size() % 4) P.f.push_back(0.f); }
  MJPC_F_ARRAYS(X)
#undef X
#define X(n) { auto v = b.ints(#n); M.io[I_##n] = (int)P.i.size(); P.i.insert(P.i.end(), v.begin(), v.end()); }
  MJPC_I_ARRAYS(X)
#undef X
  M.num_parameters = (int)b.reals("task_parameters").size();
  M.task_state_size = (int)b.reals("task_state").size();
  M.nray = (int)b.ints("ray_geoms").size();
  P.key_mpos = b.reals("key_mpos"); P.key_mquat = b.reals("key_mquat"); P.qpos0 = b.reals("qpos0");
  // derived traversal tables
  auto parent = b.ints("body_parentid"), depth = b.ints("body_depth"), dofnum = b.ints("body_dofnum"),
       dofadr = b.ints("body_dofadr"), dofpar = b.ints("dof_parentid"), jtype = b.ints("jnt_type"),
       jlim = b.ints("jnt_limited");
  auto floss = b.reals("dof_frictionloss"), damping = b.reals("dof_damping");
  int nb = M.nbody, nv = M.nv;
  if (nv > 64) throw std::runtime_error("nv > 64 not supported (dof chain masks are 64-bit)");
  int maxdepth = 0;
  for (int x : depth) maxdepth = std::max(maxdepth, x);
  std::vector<int> level_adr, level_body;
  for (int l = 1; l <= maxdepth; l++) {
    level_adr.push_back((int)level_body.size());
    for (int bb = 1; bb < nb; bb++) if (depth[bb] == l) level_body.push_back(bb);
  }
  level_adr.push_back((int)level_body.size());
  M.nlevel = maxdepth;
  std::vector<int> subend(nb), lastdof(nb, -1), mlo(nb, 0), mhi(nb, 0);
  for (int bb = 0; bb < nb; bb++) {
    int e = bb + 1;
    while (e < nb && depth[e] > depth[bb]) e++;   // DFS order: descendants follow contiguously
    subend[bb] = e;
  }
  for (int bb = 1; bb < nb; bb++) {
    lastdof[bb] = dofnum[bb] > 0 ? dofadr[bb] + dofnum[bb] - 1 : lastdof[parent[bb]];
    uint64_t mask = 0;
    for (int d = lastdof[bb]; d >= 0; d = dofpar[d]) mask |= (uint64_t)1 << d;
    mlo[bb] = (int)(uint32_t)(mask & 0xffffffffu); mhi[bb] = (int)(uint32_t)(mask >> 32);
  }
  std::vector<int> mpi, mpj, fl, lj;
  for (int d = 0; d < nv; d++)
    for (int a = d; a >= 0; a = dofpar[a]) { mpi.push_back(d); mpj.push_back(a); }
  if (!M.disable_frictionloss)
    for (int d = 0; d < nv; d++) if (floss[d] > 0) fl.push_back(d);
  if (!M.disable_limit)
    for (int j = 0; j < M.njnt; j++) if (jlim[j] && (jtype[j] == JNT_SLIDE || jtype[j] == JNT_HINGE)) lj.push_back(j);
  M.nmpair = (int)mpi.size(); M.nfloss = (int)fl.size(); M.nlimit = (int)lj.size();
  M.any_damping = 0;
  for (double x : damping) if (x > 0) M.any_damping = 1;
  auto put = [&](int id, const std::vector<int>& v) { M.io[id] = (int)P.i.size(); P.i.insert(P.i.end(), v.begin(), v.end()); };
  put(I_level_adr, level_adr); put(I_level_body, level_body); put(I_body_subtreeend, subend);
  put(I_body_lastdof, lastdof); put(I_body_dofmask_lo, mlo); put(I_body_dofmask_hi, mhi);
  put(I_mpair_i, mpi); put(I_mpair_j, mpj); put(I_floss_dof, fl); put(I_limit_jnt, lj);
  {
    // Hessian pattern: M's pattern, widened by contacts that couple two different kinematic chains
    std::vector<uint8_t> pat((size_t)nv * nv, 0);
    for (size_t k = 0; k < mpi.size(); k++) pat[(size_t)mpi[k] * nv + mpj[k]] = 1;
    auto g1 = b.ints("pair_geom1"), g2 = b.ints("pair_geom2"), gb = b.ints("geom_bodyid");
    auto chain = [&](int bb) { uint64_t m = ((uint64_t)(uint32_t)mhi[bb] << 32) | (uint32_t)mlo[bb]; return m; };
    for (size_t k = 0; k < g1.size(); k++) {
      const uint64_t m1 = chain(gb[g1[k]]), m2 = chain(gb[g2[k]]);
      if (!m1 || !m2) continue;
      const uint64_t mm = m1 | m2;
      for (int r = 0; r < nv; r++) if ((mm >> r) & 1) for (int c2 = 0; c2 <= r; c2++) if ((mm >> c2) & 1) pat[(size_t)r * nv + c2] = 1;
    }
    {
      // fixed tendons couple the dofs they wrap (limit rows)
      auto tadr = b.ints("tendon_adr"), tnum = b.ints("tendon_num"), wdof = b.ints("wrap_dof");
      for (size_t t = 0; t < tadr.size(); t++) {
        if (tnum[t] > 16) throw std::runtime_error("a tendon wraps more than 16 dofs (compact Jacobian width)");
        for (int a = tadr[t]; a < tadr[t] + tnum[t]; a++)
          for (int c2 = tadr[t]; c2 < tadr[t] + tnum[t]; c2++) {
            const int r = std::max(wdof[a], wdof[c2]), q = std::min(wdof[a], wdof[c2]);
            pat[(size_t)r * nv + q] = 1;
          }
      }
    }
    std::vector<int> hi_, hj_, frow(nv, -1);
    for (int r = 0; r < nv; r++) for (int c2 = 0; c2 <= r; c2++) if (pat[(size_t)r * nv + c2]) { hi_.push_back(r); hj_.push_back(c2); }
    for (size_t k = 0; k < fl.size(); k++) frow[fl[k]] = (int)k;
    M.nhpair = (int)hi_.size();
    put(I_hpair_i, hi_); put(I_hpair_j, hj_); put(I_floss_row, frow);
    // dof chains per body, and the widest chain union any candidate pair can produce (compact Jacobian width)
    std::vector<int> cadr(nb, 0), cnum(nb, 0), cdofs;
    for (int bb = 0; bb < nb; bb++) {
      std::vector<int> ch;
      for (int d = lastdof[bb]; d >= 0; d = dofpar[d]) ch.push_back(d);
      cadr[bb] = (int)cdofs.size(); cnum[bb] = (int)ch.size();
      cdofs.insert(cdofs.end(), ch.rbegin(), ch.rend());
    }
    int widest = 0;
    for (size_t k = 0; k < g1.size(); k++) {
      const uint64_t c1 = chain(gb[g1[k]]), c2m = chain(gb[g2[k]]);
      const uint64_t mm = (c1 && c2m) ? (c1 ^ c2m) : (c1 | c2m);   // two moving bodies: common ancestor dofs cancel
      int cnt = 0;
      for (int r = 0; r < nv; r++) cnt += (int)((mm >> r) & 1);
      widest = std::max(widest, cnt);
    }
    if (widest > 16) throw std::runtime_error("a contact pair couples more than 16 dofs (compact Jacobian width)");
    put(I_chain_adr, cadr); put(I_chain_num, cnum); put(I_chain_dof, cdofs);
  }
  while (P.i.size() % 4) P.i.push_back(0);
  while (P.f.size() % 4) P.f.push_back(0.f);
  M.nf = (int)P.f.size(); M.ni = (int)P.i.size();
  return P;
}

}  // namespace mjpc_dev
