// dev_physics.cuh - warp-cooperative forward dynamics: the device restatement of what MJPC reaches through
// mj_step / mj_forward (mjpc/trajectory.cc:158,198).  Same pipeline and constants as the CPU oracle
// (oracle/physics.h) but laid out for 32 lanes: lanes split bodies of one tree level, dofs, candidate geom
// pairs, constraint rows and matrix entries; reductions use warp shuffles; every phase ends in __syncwarp().
#pragma once
#include "dev_data.cuh"

namespace mjpc_dev {



// ------------------------------------------------------------------------------------------ position stage
template <class SP>
__device__ __noinline__ void k_kinematics(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  float *xpos = DF(xpos), *xquat = DF(xquat), *xmat = DF(xmat), *xipos = DF(xipos), *ximat = DF(ximat);
  float *xanchor = DF(xanchor), *xaxis = DF(xaxis);
  const float* qpos = DF(qpos);
  if (lane < 3) { xpos[lane] = 0; xipos[lane] = 0; }
  if (lane < 4) xquat[lane] = lane == 0 ? 1.f : 0.f;
  if (lane < 9) { float v = (lane % 4 == 0) ? 1.f : 0.f; xmat[lane] = v; ximat[lane] = v; }
  __syncwarp();
  const int *level_adr = MI(level_adr), *level_body = MI(level_body), *parentid = MI(body_parentid),
            *mocapid = MI(body_mocapid), *jntadr = MI(body_jntadr), *jntnum = MI(body_jntnum),
            *jtype = MI(jnt_type), *jqadr = MI(jnt_qposadr);
  const float *bpos = MF(body_pos), *bquat = MF(body_quat), *bipos = MF(body_ipos), *biquat = MF(body_iquat),
              *jpos = MF(jnt_pos), *jaxis = MF(jnt_axis), *qpos0 = MF(qpos0);
  for (int l = 0; l < M.nlevel; l++) {
    const int a = level_adr[l], e = level_adr[l + 1];
    for (int k = a + lane; k < e; k += 32) {
      const int b = level_body[k];
      const int p = parentid[b];
      float pos[3], quat[4];
      if (mocapid[b] >= 0) {
        const int mk = mocapid[b];
        for (int q = 0; q < 3; q++) pos[q] = DF(mocap_pos)[3 * mk + q];
        for (int q = 0; q < 4; q++) quat[q] = DF(mocap_quat)[4 * mk + q];
        quat_normalize(quat);
      } else {
        rot_vec(pos, xmat + 9 * p, bpos + 3 * b);
        for (int q = 0; q < 3; q++) pos[q] += xpos[3 * p + q];
        quat_mul(quat, xquat + 4 * p, bquat + 4 * b);
      }
      for (int j = jntadr[b]; j < jntadr[b] + jntnum[b]; j++) {
        const int qa = jqadr[j];
        const int t = jtype[j];
        if (t == JNT_FREE) {
          for (int q = 0; q < 3; q++) pos[q] = qpos[qa + q];
          for (int q = 0; q < 4; q++) quat[q] = qpos[qa + 3 + q];
          quat_normalize(quat);
          for (int q = 0; q < 3; q++) { xanchor[3 * j + q] = pos[q]; xaxis[3 * j + q] = (q == 2) ? 1.f : 0.f; }
          continue;
        }
        float R[9], anchor[3], axis[3];
        quat2mat(R, quat);
        rot_vec(anchor, R, jpos + 3 * j);
        for (int q = 0; q < 3; q++) anchor[q] += pos[q];
        rot_vec(axis, R, jaxis + 3 * j);
        for (int q = 0; q < 3; q++) { xanchor[3 * j + q] = anchor[q]; xaxis[3 * j + q] = axis[q]; }
        if (t == JNT_SLIDE) {
          const float qq = qpos[qa] - qpos0[qa];
          for (int q = 0; q < 3; q++) pos[q] += axis[q] * qq;
        } else {
          float ql[4], qn[4], off[3];
          if (t == JNT_HINGE) {
            axis_angle_quat(ql, jaxis + 3 * j, qpos[qa] - qpos0[qa]);
          } else {
            for (int q = 0; q < 4; q++) ql[q] = qpos[qa + q];
            quat_normalize(ql);
          }
          quat_mul(qn, quat, ql);
          for (int q = 0; q < 4; q++) quat[q] = qn[q];
          quat2mat(R, quat);
          rot_vec(off, R, jpos + 3 * j);
          for (int q = 0; q < 3; q++) pos[q] = anchor[q] - off[q];
        }
      }
      quat_normalize(quat);
      for (int q = 0; q < 3; q++) xpos[3 * b + q] = pos[q];
      for (int q = 0; q < 4; q++) xquat[4 * b + q] = quat[q];
      float R[9], ip[3], iq[4];
      quat2mat(R, quat);
      for (int q = 0; q < 9; q++) xmat[9 * b + q] = R[q];
      rot_vec(ip, R, bipos + 3 * b);
      for (int q = 0; q < 3; q++) xipos[3 * b + q] = pos[q] + ip[q];
      quat_mul(iq, quat, biquat + 4 * b);
      quat2mat(R, iq);
      for (int q = 0; q < 9; q++) ximat[9 * b + q] = R[q];
    }
    __syncwarp();
  }
  const int* gbody = MI(geom_bodyid);
  const float *gpos = MF(geom_pos), *gquat = MF(geom_quat);
  float *gxpos = DF(geom_xpos), *gxmat = DF(geom_xmat);
  for (int g = lane; g < M.ngeom; g += 32) {
    const int b = gbody[g];
    float p[3], q[4], R[9];
    rot_vec(p, xmat + 9 * b, gpos + 3 * g);
    for (int k = 0; k < 3; k++) gxpos[3 * g + k] = xpos[3 * b + k] + p[k];
    quat_mul(q, xquat + 4 * b, gquat + 4 * g);
    quat2mat(R, q);
    for (int k = 0; k < 9; k++) gxmat[9 * g + k] = R[k];
  }
  const int* sbody = MI(site_bodyid);
  const float* spos = MF(site_pos);
  float* sxpos = DF(site_xpos);
  for (int s = lane; s < M.nsite; s += 32) {
    const int b = sbody[s];
    float p[3];
    rot_vec(p, xmat + 9 * b, spos + 3 * s);
    for (int k = 0; k < 3; k++) sxpos[3 * s + k] = xpos[3 * b + k] + p[k];
  }
  __syncwarp();
}

template <class SP>
__device__ __noinline__ void k_com_pos(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  const int *subend = MI(body_subtreeend), *rootid = MI(body_rootid);
  const float *mass = MF(body_mass), *submass = MF(body_subtreemass), *inertia = MF(body_inertia);
  float *scom = DF(subtree_com), *xipos = DF(xipos), *ximat = DF(ximat), *cinert = DF(cinert);
  // DFS body order: the subtree of b is the contiguous id range [b, subend[b])
  for (int b = lane; b < M.nbody; b += 32) {
    float s[3] = {0, 0, 0};
    if (submass[b] < kMinVal) {
      for (int k = 0; k < 3; k++) s[k] = xipos[3 * b + k];
    } else {
      MJPC_ROLL
      for (int q = subend[b] - 1; q >= b; q--)
        for (int k = 0; k < 3; k++) s[k] += mass[q] * xipos[3 * q + k];
      for (int k = 0; k < 3; k++) s[k] /= submass[b];
    }
    for (int k = 0; k < 3; k++) scom[3 * b + k] = s[k];
  }
  __syncwarp();
  for (int b = 1 + lane; b < M.nbody; b += 32) {
    const float* R = ximat + 9 * b;
    const float* I = inertia + 3 * b;
    const float m = mass[b];
    float o[3];
    for (int k = 0; k < 3; k++) o[k] = xipos[3 * b + k] - scom[3 * rootid[b] + k];
    float W[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        W[3 * i + j] = R[3 * i] * I[0] * R[3 * j] + R[3 * i + 1] * I[1] * R[3 * j + 1] + R[3 * i + 2] * I[2] * R[3 * j + 2];
    const float oo = dot3(o, o);
    float* ci = cinert + 10 * b;
    ci[0] = W[0] + m * (oo - o[0] * o[0]); ci[1] = W[4] + m * (oo - o[1] * o[1]); ci[2] = W[8] + m * (oo - o[2] * o[2]);
    ci[3] = W[1] - m * o[0] * o[1]; ci[4] = W[2] - m * o[0] * o[2]; ci[5] = W[5] - m * o[1] * o[2];
    ci[6] = m * o[0]; ci[7] = m * o[1]; ci[8] = m * o[2]; ci[9] = m;
  }
  const int *jbody = MI(jnt_bodyid), *jdof = MI(jnt_dofadr), *jtype = MI(jnt_type);
  float *cdof = DF(cdof), *xanchor = DF(xanchor), *xaxis = DF(xaxis), *xmat = DF(xmat);
  for (int j = lane; j < M.njnt; j += 32) {
    const int b = jbody[j];
    int da = jdof[j];
    float off[3];
    for (int k = 0; k < 3; k++) off[k] = scom[3 * rootid[b] + k] - xanchor[3 * j + k];
    const float* ax = xaxis + 3 * j;
    const int t = jtype[j];
    if (t == JNT_FREE) {
      for (int k = 0; k < 3; k++) {
        float* cd = cdof + 6 * (da + k);
        for (int q = 0; q < 6; q++) cd[q] = 0;
        cd[3 + k] = 1;
      }
      da += 3;
    }
    if (t == JNT_FREE || t == JNT_BALL) {
      for (int k = 0; k < 3; k++) {
        float* cd = cdof + 6 * (da + k);
        float col[3] = {xmat[9 * b + k], xmat[9 * b + 3 + k], xmat[9 * b + 6 + k]};
        for (int q = 0; q < 3; q++) cd[q] = col[q];
        cross3(cd + 3, col, off);
      }
    } else if (t == JNT_SLIDE) {
      float* cd = cdof + 6 * da;
      for (int q = 0; q < 3; q++) { cd[q] = 0; cd[3 + q] = ax[q]; }
    } else {
      float* cd = cdof + 6 * da;
      for (int q = 0; q < 3; q++) cd[q] = ax[q];
      cross3(cd + 3, ax, off);
    }
  }
  __syncwarp();
}

// SPD solve A x = b (x may alias b) of qM, qM + h diag(damping) or the Newton Hessian.  Static specs factor along the
// dof tree when the matrix has the tree's pattern (`tree_pattern`; qM and the Euler matrix always do) and leave A
// unchanged; otherwise the dense factor overwrites A.
template <class SP>
__device__ __forceinline__ void spd_solve(Ctx& c, float* A, float* inv, float* x, const float* b, bool tree_pattern) {
  if constexpr (SP::kTreeFactor) {
    if (tree_pattern) { warp_tree_factor_solve<typename SP::Tree>(A, x, b, c.lane); return; }
  }
  warp_chol_factor_solve<SP::kNV>(A, inv, x, b, SP::model(c).nv, c.lane);
}

// composite rigid body inertia -> dense joint-space inertia qM (and qLD, the copy the dense factor overwrites)
template <class SP>
__device__ __noinline__ void k_crb(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const int* subend = MI(body_subtreeend);
  float *cinert = DF(cinert), *crb = DF(crb), *cdof = DF(cdof), *dofbuf = DF(dofbuf), *qM = DF(qM), *qLD = DF(qLD);
  for (int b = 1 + lane; b < M.nbody; b += 32) {
    float s[10];
    for (int k = 0; k < 10; k++) s[k] = 0;
    MJPC_ROLL
    for (int q = subend[b] - 1; q >= b; q--)
      for (int k = 0; k < 10; k++) s[k] += cinert[10 * q + k];
    for (int k = 0; k < 10; k++) crb[10 * b + k] = s[k];
  }
  __syncwarp();
  const int* dbody = MI(dof_bodyid);
  for (int i = lane; i < nv; i += 32) mul_inert_vec(dofbuf + 6 * i, crb + 10 * dbody[i], cdof + 6 * i);
  __syncwarp();
  const int *mpi = MI(mpair_i), *mpj = MI(mpair_j);
  const float* arm = MF(dof_armature);
  for (int k = lane; k < M.nmpair; k += 32) {
    const int i = mpi[k], j = mpj[k];
    float s = 0;
    for (int q = 0; q < 6; q++) s += cdof[6 * j + q] * dofbuf[6 * i + q];
    if (i == j) s += arm[i];
    qM[i * nv + j] = s; qM[j * nv + i] = s;
  }
  __syncwarp();
  // entries of qM outside the (dof, ancestor) pattern stay zero (zeroed once per rollout); the dense factor
  // fills in, so the whole matrix is re-copied before every factorisation (the tree factor reads qM itself)
  if constexpr (!SP::kTreeFactor) {
    for (int w = lane; w < nv * nv; w += 32) qLD[w] = qM[w];
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------ collision
struct RawContact { float dist, pos[3], normal[3]; };

__device__ __forceinline__ int collide_plane_sphere(RawContact* out, const float* pp, const float* pm,
                                                    const float* sp, float r) {
  float n[3] = {pm[2], pm[5], pm[8]};
  float diff[3] = {sp[0] - pp[0], sp[1] - pp[1], sp[2] - pp[2]};
  float dist = dot3(diff, n) - r;
  out->dist = dist;
  for (int k = 0; k < 3; k++) { out->normal[k] = n[k]; out->pos[k] = sp[k] - n[k] * (r + dist * 0.5f); }
  return 1;
}
__device__ __forceinline__ int collide_plane_capsule(RawContact* out, const float* pp, const float* pm,
                                                     const float* cp, const float* cm, const float* size) {
  float axis[3] = {cm[2], cm[5], cm[8]};
  int n = 0;
  for (int s = -1; s <= 1; s += 2) {
    float e[3];
    for (int k = 0; k < 3; k++) e[k] = cp[k] + (float)s * size[1] * axis[k];
    n += collide_plane_sphere(out + n, pp, pm, e, size[0]);
  }
  return n;
}
__device__ __forceinline__ int collide_plane_box(RawContact* out, const float* pp, const float* pm, const float* bp,
                                                 const float* bm, const float* size, float margin) {
  float nrm[3] = {pm[2], pm[5], pm[8]};
  int n = 0;
  for (int k = 0; k < 8 && n < 4; k++) {
    float loc[3] = {(k & 1 ? size[0] : -size[0]), (k & 2 ? size[1] : -size[1]), (k & 4 ? size[2] : -size[2])};
    float w[3], corner[3], diff[3];
    rot_vec(w, bm, loc);
    for (int q = 0; q < 3; q++) { corner[q] = bp[q] + w[q]; diff[q] = corner[q] - pp[q]; }
    float dist = dot3(diff, nrm);
    if (dist > margin) continue;
    out[n].dist = dist;
    for (int q = 0; q < 3; q++) { out[n].normal[q] = nrm[q]; out[n].pos[q] = corner[q] - nrm[q] * dist * 0.5f; }
    n++;
  }
  return n;
}
__device__ __forceinline__ int collide_plane_cylinder(RawContact* out, const float* pp, const float* pm,
                                                      const float* cp, const float* cm, const float* size,
                                                      float margin) {
  float nrm[3] = {pm[2], pm[5], pm[8]};
  float axis[3] = {cm[2], cm[5], cm[8]};
  const float r = size[0], h = size[1];
  float prj = dot3(axis, nrm);
  if (prj > 0) { for (int k = 0; k < 3; k++) axis[k] = -axis[k]; prj = -prj; }
  float vec[3];
  for (int k = 0; k < 3; k++) vec[k] = -nrm[k] + axis[k] * prj;
  // vec has length sin(tilt); its fp32 rounding residual along the axis would, scaled to r, lift the rim points off
  // the rim plane near an upright axis (oracle/physics.h collide_plane_cylinder, reduced precision): project it out
  const float va = dot3(vec, axis);
  for (int k = 0; k < 3; k++) vec[k] -= axis[k] * va;
  float len = norm3(vec);
  if (len < 1e-6f) { vec[0] = cm[0]; vec[1] = cm[3]; vec[2] = cm[6]; len = 1; }
  for (int k = 0; k < 3; k++) vec[k] *= r / len;
  float side[3];
  cross3(side, vec, axis);
  float diff[3] = {cp[0] - pp[0], cp[1] - pp[1], cp[2] - pp[2]};
  const float dist0 = dot3(diff, nrm);
  int n = 0;
  for (int k = 0; k < 4; k++) {
    float cand[3];
    for (int q = 0; q < 3; q++) {
      if (k == 0) cand[q] = axis[q] * h + vec[q];
      else if (k == 1) cand[q] = -axis[q] * h + vec[q];
      else if (k == 2) cand[q] = axis[q] * h - vec[q] * 0.5f + side[q] * 0.8660254037844386f;
      else cand[q] = axis[q] * h - vec[q] * 0.5f - side[q] * 0.8660254037844386f;
    }
    float dist = dist0 + dot3(cand, nrm);
    if (dist > margin) continue;
    out[n].dist = dist;
    for (int q = 0; q < 3; q++) { out[n].normal[q] = nrm[q]; out[n].pos[q] = cp[q] + cand[q] - nrm[q] * dist * 0.5f; }
    n++;
  }
  return n;
}
__device__ __forceinline__ int collide_sphere_sphere(RawContact* out, const float* p1, float r1, const float* p2,
                                                     float r2) {
  float dv[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  float len = norm3(dv);
  float n[3] = {1, 0, 0};
  if (len >= kMinVal) { n[0] = dv[0] / len; n[1] = dv[1] / len; n[2] = dv[2] / len; }
  float dist = len - r1 - r2;
  out->dist = dist;
  for (int k = 0; k < 3; k++) { out->normal[k] = n[k]; out->pos[k] = p1[k] + n[k] * (r1 + dist * 0.5f); }
  return 1;
}
__device__ __forceinline__ int collide_sphere_capsule(RawContact* out, const float* sp, float sr, const float* cp,
                                                      const float* cm, const float* csize) {
  float axis[3] = {cm[2], cm[5], cm[8]};
  float dv[3] = {sp[0] - cp[0], sp[1] - cp[1], sp[2] - cp[2]};
  float x = fmaxf(-csize[1], fminf(csize[1], dot3(dv, axis)));
  float q[3] = {cp[0] + axis[0] * x, cp[1] + axis[1] * x, cp[2] + axis[2] * x};
  return collide_sphere_sphere(out, sp, sr, q, csize[0]);
}
__device__ __forceinline__ int collide_sphere_box(RawContact* out, const float* sp, float sr, const float* bp,
                                                  const float* bm, const float* bs) {
  float dv[3] = {sp[0] - bp[0], sp[1] - bp[1], sp[2] - bp[2]};
  float loc[3], cl[3];
  rot_vec_T(loc, bm, dv);
  bool inside = true;
  for (int k = 0; k < 3; k++) {
    cl[k] = fmaxf(-bs[k], fminf(bs[k], loc[k]));
    if (cl[k] != loc[k]) inside = false;
  }
  float nl[3], dist, pl[3];
  if (!inside) {
    float dd[3] = {cl[0] - loc[0], cl[1] - loc[1], cl[2] - loc[2]};
    float len = norm3(dd);
    for (int k = 0; k < 3; k++) nl[k] = dd[k] / len;
    dist = len - sr;
    for (int k = 0; k < 3; k++) pl[k] = cl[k] - nl[k] * dist * 0.5f;
  } else {
    int kk = 0;
    float best = bs[0] - fabsf(loc[0]);
    for (int k = 1; k < 3; k++) { float g = bs[k] - fabsf(loc[k]); if (g < best) { best = g; kk = k; } }
    float sgn = loc[kk] >= 0 ? 1.f : -1.f;
    nl[0] = nl[1] = nl[2] = 0;
    dist = -best - sr;
    for (int k = 0; k < 3; k++) pl[k] = loc[k];
    for (int k = 0; k < 3; k++)
      if (k == kk) { nl[k] = -sgn; pl[k] = 0.5f * (sgn * bs[k] + loc[k] - sgn * sr); }
  }
  float nw[3], pw[3];
  rot_vec(nw, bm, nl);
  rot_vec(pw, bm, pl);
  out->dist = dist;
  for (int k = 0; k < 3; k++) { out->normal[k] = nw[k]; out->pos[k] = bp[k] + pw[k]; }
  return 1;
}

// [EXT] mjc_CapsuleCapsule restated (same algorithm as oracle/physics.h collide_capsule_capsule): nearest points of the
// two axis segments, then a sphere test there; (nearly) parallel axes test the segment ends and may return two contacts
__device__ __forceinline__ int collide_capsule_capsule(RawContact* out, const float* p1, const float* m1, const float* s1,
                                                        const float* p2, const float* m2, const float* s2, float margin) {
  const float a1[3] = {m1[2], m1[5], m1[8]}, a2[3] = {m2[2], m2[5], m2[8]};
  const float dif[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
  const float ma = dot3(a1, a1), mb = -dot3(a1, a2), mc = dot3(a2, a2), u = -dot3(a1, dif), v = dot3(a2, dif);
  const float det = ma * mc - mb * mb;
  const float r1 = s1[0], l1 = s1[1], r2 = s2[0], l2 = s2[1];
  auto sphere = [&](RawContact* o, float x1, float x2) {
    float v1[3], v2[3];
    for (int k = 0; k < 3; k++) { v1[k] = p1[k] + a1[k] * x1; v2[k] = p2[k] + a2[k] * x2; }
    collide_sphere_sphere(o, v1, r1, v2, r2);
    return o->dist <= margin ? 1 : 0;
  };
  // parallel test scaled to fp32's resolution (oracle/physics.h capsules_parallel): for exactly parallel unit axes
  // the rounding residual of det is ~1e-7, so an absolute mjMINVAL would send them to the nearest-point solve, which
  // divides rounding noise by rounding noise and returns one contact at an arbitrary end
  if (fabsf(det) >= kCapsuleParallel * ma * mc) {
    float x1 = (mc * u - mb * v) / det, x2 = (ma * v - mb * u) / det;
    if (x1 > l1) { x1 = l1; x2 = (v - mb * l1) / mc; }
    else if (x1 < -l1) { x1 = -l1; x2 = (v + mb * l1) / mc; }
    if (x2 > l2) { x2 = l2; x1 = fmaxf(-l1, fminf(l1, (u - mb * l2) / ma)); }
    else if (x2 < -l2) { x2 = -l2; x1 = fmaxf(-l1, fminf(l1, (u + mb * l2) / ma)); }
    return sphere(out, x1, x2);
  }
  int n = sphere(out, l1, fmaxf(-l2, fminf(l2, (v - mb * l1) / mc)));
  n += sphere(out + n, -l1, fmaxf(-l2, fminf(l2, (v + mb * l1) / mc)));
  if (n >= 2) return n;
  n += sphere(out + n, fmaxf(-l1, fminf(l1, (u - mb * l2) / ma)), l2);
  if (n >= 2) return n;
  n += sphere(out + n, fmaxf(-l1, fminf(l1, (u + mb * l2) / ma)), -l2);
  return n;
}

template <class SP>
__device__ __noinline__ void k_collision(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  c.ncon = 0;
  c.npseudo = 0;
  const int *pg1 = MI(pair_geom1), *pg2 = MI(pair_geom2), *gtype = MI(geom_type), *gprio = MI(geom_priority),
            *gcondim = MI(geom_condim);
  const float *gmargin = MF(geom_margin), *ggap = MF(geom_gap), *gsize = MF(geom_size), *grbound = MF(geom_rbound),
              *gfric = MF(geom_friction), *gsolmix = MF(geom_solmix), *gsolref = MF(geom_solref),
              *gsolimp = MF(geom_solimp);
  const float *gxpos = DF(geom_xpos), *gxmat = DF(geom_xmat);
  int ncon = 0;
  const int npair = M.disable_contact ? 0 : M.npair;
  const int maxgeom = M.maxcon - 2 * M.ntendon;    // geometric contact budget; the last slots hold tendon limits
  // Two stages (with every pair MuJoCo's filters keep - 395 on the A1 - the narrow phase must not run 13 divergent rounds):
  // (1) bounding test of 32 pairs per round, survivors appended IN PAIR ORDER to a queue in shared memory (ballot +
  // prefix count); (2) whenever 32 survivors are pending (and once at the end) one narrow-phase round, one pair per lane.
  int* queue = reinterpret_cast<int*>(DF(efc_blk));   // 64 ints of the block scratch (free until the constraint phases)
  int nq = 0, nextpair = 0;
  while (nextpair < npair || nq > 0) {
    while (nq < 32 && nextpair < npair) {
      const int p = nextpair + lane;
      bool pass = false;
      if (p < npair) {
        const int g1 = pg1[p], g2 = pg2[p];
        const float margin = fmaxf(gmargin[g1], gmargin[g2]);
        const float *p1 = gxpos + 3 * g1, *p2 = gxpos + 3 * g2;
        const float dv[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
        if (gtype[g1] == GEOM_PLANE) {
          const float* m1 = gxmat + 9 * g1;
          const float n[3] = {m1[2], m1[5], m1[8]};
          pass = !(dot3(dv, n) > grbound[g2] + margin);
        } else {
          const float bound = grbound[g1] + grbound[g2] + margin;
          pass = !(dot3(dv, dv) > bound * bound);
        }
      }
      const unsigned mask = __ballot_sync(kFull, pass);
      if (pass) queue[nq + __popc(mask & ((1u << lane) - 1u))] = p;
      nq += __popc(mask);
      nextpair += 32;
      __syncwarp();
    }
    if (nq == 0) break;                               // nothing pending and no pairs left (warp-uniform)
    const int nb = min(nq, 32);
    const int p = queue[min(lane, nb - 1)];
    RawContact raw[4];
    int cnt = 0, g1 = 0, g2 = 0;
    float margin = 0, gap = 0;
    if (lane < nb) {
      g1 = pg1[p]; g2 = pg2[p];
      const int t1 = gtype[g1], t2 = gtype[g2];
      margin = fmaxf(gmargin[g1], gmargin[g2]);
      gap = fmaxf(ggap[g1], ggap[g2]);
      const float *p1 = gxpos + 3 * g1, *p2 = gxpos + 3 * g2, *m1 = gxmat + 9 * g1, *m2 = gxmat + 9 * g2;
      const float *s1 = gsize + 3 * g1, *s2 = gsize + 3 * g2;
      int n = 0;
      {
        if (t1 == GEOM_PLANE && t2 == GEOM_SPHERE) n = collide_plane_sphere(raw, p1, m1, p2, s2[0]);
        else if (t1 == GEOM_PLANE && t2 == GEOM_CAPSULE) n = collide_plane_capsule(raw, p1, m1, p2, m2, s2);
        else if (t1 == GEOM_PLANE && t2 == GEOM_BOX) n = collide_plane_box(raw, p1, m1, p2, m2, s2, margin);
        else if (t1 == GEOM_PLANE && t2 == GEOM_CYLINDER) n = collide_plane_cylinder(raw, p1, m1, p2, m2, s2, margin);
        else if (t1 == GEOM_SPHERE && t2 == GEOM_SPHERE) n = collide_sphere_sphere(raw, p1, s1[0], p2, s2[0]);
        else if (t1 == GEOM_SPHERE && t2 == GEOM_CAPSULE) n = collide_sphere_capsule(raw, p1, s1[0], p2, m2, s2);
        else if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) n = collide_sphere_box(raw, p1, s1[0], p2, m2, s2);
        else if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) n = collide_capsule_capsule(raw, p1, m1, s1, p2, m2, s2, margin);
      }
      MJPC_ROLL
      for (int k = 0; k < n; k++)
        if (raw[k].dist < margin) { if (cnt != k) raw[cnt] = raw[k]; cnt++; }
    }
    const int incl = warp_incl_scan(cnt, lane);
    const int total = __shfl_sync(kFull, incl, 31);
    const int excl = incl - cnt;
    MJPC_ROLL
    for (int k = 0; k < cnt; k++) {
      const int idx = ncon + excl + k;
      if (idx >= maxgeom) break;  // capacity (warning raised below)
      DF(con_dist)[idx] = raw[k].dist;
      float fr[9];
      for (int q = 0; q < 3; q++) { DF(con_pos)[3 * idx + q] = raw[k].pos[q]; fr[q] = raw[k].normal[q]; }
      make_frame(fr);
      for (int q = 0; q < 9; q++) DF(con_frame)[9 * idx + q] = fr[q];
      DF(con_margin)[idx] = margin - gap;
      DI(con_g1)[idx] = g1; DI(con_g2)[idx] = g2;
      float f3[3], solref[2], solimp[5];
      int dim;
      if (gprio[g1] != gprio[g2]) {
        const int gp = gprio[g1] > gprio[g2] ? g1 : g2;
        dim = gcondim[gp];
        for (int q = 0; q < 2; q++) solref[q] = gsolref[2 * gp + q];
        for (int q = 0; q < 5; q++) solimp[q] = gsolimp[5 * gp + q];
        for (int q = 0; q < 3; q++) f3[q] = gfric[3 * gp + q];
      } else {
        dim = max(gcondim[g1], gcondim[g2]);
        const float w1 = gsolmix[g1], w2 = gsolmix[g2];
        float mix;
        if (w1 >= kMinVal && w2 >= kMinVal) mix = w1 / (w1 + w2);
        else if (w1 < kMinVal && w2 < kMinVal) mix = 0.5f;
        else mix = w1 < kMinVal ? 0.f : 1.f;
        const float *r1 = gsolref + 2 * g1, *r2 = gsolref + 2 * g2;
        if (r1[0] > 0 && r2[0] > 0) { for (int q = 0; q < 2; q++) solref[q] = mix * r1[q] + (1 - mix) * r2[q]; }
        else { for (int q = 0; q < 2; q++) solref[q] = fminf(r1[q], r2[q]); }
        for (int q = 0; q < 5; q++) solimp[q] = mix * gsolimp[5 * g1 + q] + (1 - mix) * gsolimp[5 * g2 + q];
        for (int q = 0; q < 3; q++) f3[q] = fmaxf(gfric[3 * g1 + q], gfric[3 * g2 + q]);
      }
      for (int q = 0; q < 3; q++) f3[q] = fmaxf(f3[q], kMinMu);
      float* cf = DF(con_friction) + 5 * idx;
      cf[0] = cf[1] = f3[0]; cf[2] = f3[1]; cf[3] = cf[4] = f3[2];
      for (int q = 0; q < 2; q++) DF(con_solref)[2 * idx + q] = solref[q];
      for (int q = 0; q < 5; q++) DF(con_solimp)[5 * idx + q] = solimp[q];
      DI(con_dim)[idx] = dim;
      DF(con_mu)[idx] = 0;
      DI(con_adr)[idx] = -1;
    }
    // contact buffer full: MuJoCo raises mjWARN_CONTACTFULL and Trajectory::Rollout turns any warning into failure
    // (trajectory.cc:169-173, utilities.cc:804-816) - never a silently truncated contact set in the ranking
    if (ncon + total > maxgeom) c.warn = 1;
    ncon = min(ncon + total, maxgeom);
    __syncwarp();
    const int rest = nq - nb;                       // <= 31 survivors of the last bounding round stay pending
    const int moved = queue[min(nb + lane, 63)];
    __syncwarp();
    if (lane < rest) queue[lane] = moved;
    nq = rest;
    __syncwarp();
  }
  // Active limits of fixed tendons ride along as frictionless pseudo-contacts (dim 1) appended after the geometric
  // contacts: they need exactly what a contact row needs - a short dof list, a compact Jacobian row, dist, margin,
  // solref/solimp - and every later phase then treats them uniformly.  con_g1 = -(tendon+1) marks them, con_mu
  // carries the side (+-1).  (Row order therefore differs from the oracle's: tendon limits come after contacts.)
  // Each fixed tendon has two slots of its own after the geometric budget (pack_model), so, as in MuJoCo, where
  // tendon limits are constraint rows and take no contact slot, they never count against maxcon.
  int npseudo = 0;
  if (!M.disable_limit && M.ntendon > 0 && lane == 0) {
    const int *tadr = MI(tendon_adr), *tnum = MI(tendon_num), *tlim = MI(tendon_limited), *wq = MI(wrap_qposadr);
    const float *wc = MF(wrap_coef), *trange = MF(tendon_range), *tmargin = MF(tendon_margin);
    const float* qpos = DF(qpos);
    for (int t = 0; t < M.ntendon; t++) {
      if (!tlim[t]) continue;
      float len = 0.f;
      for (int w = tadr[t]; w < tadr[t] + tnum[t]; w++) len += wc[w] * qpos[wq[w]];
      for (int side = -1; side <= 1; side += 2) {
        const float dd = side * (trange[2 * t + (side + 1) / 2] - len);
        if (dd < tmargin[t]) {
          const int idx = ncon + npseudo;
          DF(con_dist)[idx] = dd; DF(con_margin)[idx] = tmargin[t];
          DI(con_g1)[idx] = -(t + 1); DI(con_g2)[idx] = -(t + 1);
          for (int q = 0; q < 2; q++) DF(con_solref)[2 * idx + q] = MF(tendon_solref)[2 * t + q];
          for (int q = 0; q < 5; q++) DF(con_solimp)[5 * idx + q] = MF(tendon_solimp)[5 * t + q];
          for (int q = 0; q < 5; q++) DF(con_friction)[5 * idx + q] = 0.f;
          DI(con_dim)[idx] = 1;
          DF(con_mu)[idx] = (float)side;
          DI(con_adr)[idx] = -1;
          npseudo++;
        }
      }
    }
  }
  npseudo = __shfl_sync(kFull, npseudo, 0);
  __syncwarp();
  c.npseudo = npseudo;
  c.ncon = ncon + npseudo;
}

// ------------------------------------------------------------------------------------------ constraints
__device__ __forceinline__ float get_impedance(const float* solimp, float pos, float margin, bool zero_dmin = false) {
  const float dmin = fminf(kMaxImp, fmaxf(kMinImp, zero_dmin ? 0.f : solimp[0]));
  const float dmax = fminf(kMaxImp, fmaxf(kMinImp, solimp[1]));
  const float width = fmaxf(0.f, solimp[2]);
  const float mid = fminf(kMaxImp, fmaxf(kMinImp, solimp[3]));
  const float power = fmaxf(1.f, solimp[4]);
  if (dmin == dmax || width <= kMinVal) return 0.5f * (dmin + dmax);
  float x = (pos - margin) / width;
  if (x < 0) x = -x;
  if (x >= 1) return dmax;
  if (x == 0) return dmin;
  float y;
  if (power == 1) y = x;
  else if (x <= mid) y = powf(x, power) / powf(mid, power - 1);
  else y = 1 - powf(1 - x, power) / powf(1 - mid, power - 1);
  return dmin + y * (dmax - dmin);
}

constexpr int kL = 16;  // width of a compact constraint-Jacobian row (dofs of the chains a contact couples)
// Small data-dependent trip counts (contact dimension <= 6, chain width <= kL) are written as fixed-bound,
// fully unrolled, predicated loops: straight-line code with no taken branches, which is what a single
// resident warp per scheduler needs (every loop back-edge is an exposed fetch bubble).
#define FOR_DIM(j, start, dim) _Pragma("unroll") for (int j = (start); j < 6; j++) if (j < (dim))
// the rows of one contact: dim <= 6 for an elliptic cone, 2 (condim - 1) <= 10 for a pyramidal one
#define FOR_ROWS(j, nrow) _Pragma("unroll") for (int j = 0; j < 10; j++) if (j < (nrow))
#define FOR_KL(l, nd) _Pragma("unroll") for (int l = 0; l < kL; l++) if (l < (nd))

// J row (compact) dot a dof-indexed vector: friction-loss / limit rows touch one dof, contact rows their chain
template <class SP>
__device__ __forceinline__ float row_dot(Ctx& c, int row, int nsimple, const float* v) {
  if (row < nsimple) return DF(efc_sgn)[row] * v[DI(efc_dof)[row]];
  const int ci = DI(efc_id)[row];
  const int nd = DI(con_nd)[ci];
  const int* dofs = DI(con_dof) + ci * kL;
  const float* Jr = DF(efc_J) + row * kL;
  float a = 0.f;
  FOR_KL(l, nd) a += Jr[l] * v[dofs[l]];
  return a;
}

template <class SP>
__device__ __noinline__ void k_make_constraint(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  float *J = DF(efc_J), *epos = DF(efc_pos), *emargin = DF(efc_margin), *ediag = DF(efc_diag), *efloss = DF(efc_floss),
        *esgn = DF(efc_sgn);
  int *etype = DI(efc_type), *eid = DI(efc_id), *eitem = DI(efc_item), *edof = DI(efc_dof);
  const float *dinvw = MF(dof_invweight0), *qpos = DF(qpos);
  int ne = 0, nitem = 0;
  // --- dof friction loss rows (static list)
  {
    const int* fl = MI(floss_dof);
    const float* flv = MF(dof_frictionloss);
    const int nf = M.nfloss;
    for (int k = lane; k < nf; k += 32) {
      const int dof = fl[k];
      edof[k] = dof; esgn[k] = 1.f;
      epos[k] = 0; emargin[k] = 0; ediag[k] = dinvw[dof]; etype[k] = CNSTR_FRICTION_DOF; eid[k] = dof;
      efloss[k] = flv[dof]; eitem[k] = k;
    }
    ne = nf; nitem = nf;
  }
  // --- joint limits (slide / hinge): lane per limited joint, ordered compaction
  {
    const int *lj = MI(limit_jnt), *jqadr = MI(jnt_qposadr), *jdadr = MI(jnt_dofadr);
    const float *jrange = MF(jnt_range), *jmargin = MF(jnt_margin);
    for (int base = 0; base < M.nlimit; base += 32) {
      const int k = base + lane;
      int cnt = 0, j = 0;
      float dist[2], sgn[2];
      if (k < M.nlimit) {
        j = lj[k];
        const float q = qpos[jqadr[j]];
        for (int side = -1; side <= 1; side += 2) {
          const float dd = side * (jrange[2 * j + (side + 1) / 2] - q);
          if (dd < jmargin[j]) { dist[cnt] = dd; sgn[cnt] = (float)-side; cnt++; }
        }
      }
      const int incl = warp_incl_scan(cnt, lane);
      const int total = __shfl_sync(kFull, incl, 31);
      for (int q = 0; q < cnt; q++) {
        const int r = ne + incl - cnt + q;
        if (r >= M.maxefc) break;
        edof[r] = jdadr[j]; esgn[r] = sgn[q];
        epos[r] = dist[q]; emargin[r] = jmargin[j]; ediag[r] = dinvw[jdadr[j]]; etype[r] = CNSTR_LIMIT_JOINT;
        eid[r] = j; efloss[r] = 0; eitem[nitem + incl - cnt + q] = r;
      }
      if (total > M.maxefc - ne) c.warn = 1;   // constraint buffer full (mjWARN_CNSTRFULL) -> rollout failure
      const int added = min(total, M.maxefc - ne);
      ne += added; nitem += added;
      __syncwarp();
    }
  }
  c.nlim = ne - M.nfloss;
  // --- contacts: row addresses are assigned sequentially (a contact that does not fit is dropped, later
  //     smaller ones may still fit: same rule as the oracle); dof lists = union of the two bodies' chains
  int *cadr = DI(con_adr), *cdim = DI(con_dim), *cnd = DI(con_nd), *cdofl = DI(con_dof), *cloc = DI(con_loc),
      *cboff = DI(con_boff);
  const int *g1a = DI(con_g1), *g2a = DI(con_g2), *gbody = MI(geom_bodyid);
  const bool pyramidal = M.cone == CONE_PYRAMIDAL;
  for (int w = lane; w < c.ncon * nv; w += 32) cloc[w] = -1;
  __syncwarp();
  {
    const int *chadr = MI(chain_adr), *chnum = MI(chain_num), *chdof = MI(chain_dof);
    const int *tadr = MI(tendon_adr), *tnum = MI(tendon_num), *wdof = MI(wrap_dof);
    for (int ci = lane; ci < c.ncon; ci += 32) {
      int nd = 0;
      if (g1a[ci] < 0) {   // tendon-limit pseudo-contact: the wrapped dofs
        const int t = -g1a[ci] - 1;
        for (int w = tadr[t]; w < tadr[t] + tnum[t]; w++) {
          const int dof = wdof[w];
          if (cloc[ci * nv + dof] < 0 && nd < kL) { cloc[ci * nv + dof] = nd; cdofl[ci * kL + nd] = dof; nd++; }
        }
        cnd[ci] = nd;
        continue;
      }
      // contact between two moving bodies: the relative Jacobian vanishes identically on their COMMON ancestor dofs
      // (same point, same motion axis, opposite signs), so the dof list is the symmetric difference of the two chains
      const int ba = gbody[g1a[ci]], bbb = gbody[g2a[ci]];
      const unsigned clo = (unsigned)MI(body_dofmask_lo)[ba] & (unsigned)MI(body_dofmask_lo)[bbb];
      const unsigned chi = (unsigned)MI(body_dofmask_hi)[ba] & (unsigned)MI(body_dofmask_hi)[bbb];
      for (int s2 = 0; s2 < 2; s2++) {
        const int bb = s2 ? bbb : ba;
        for (int q = 0; q < chnum[bb]; q++) {
          const int dof = chdof[chadr[bb] + q];
          const bool common = dof < 32 ? ((clo >> dof) & 1u) : ((chi >> (dof - 32)) & 1u);
          if (common) continue;
          if (cloc[ci * nv + dof] < 0 && nd < kL) { cloc[ci * nv + dof] = nd; cdofl[ci * kL + nd] = dof; nd++; }
        }
      }
      cnd[ci] = nd;
    }
  }
  __syncwarp();
  int efc_ovf = 0;
  if (lane == 0) {
    int r = ne, it = nitem, bo = 0;
    for (int ci = 0; ci < c.ncon; ci++) {
      const int condim = cdim[ci];
      const bool pyr = pyramidal && condim > 1;
      const int nrow = pyr ? 2 * (condim - 1) : condim;   // pyramidal cone: two opposing edges per friction direction
      cboff[ci] = bo;
      if (r + nrow > M.maxefc) { cadr[ci] = -1; efc_ovf = 1; continue; }
      cadr[ci] = r;
      if (pyr) { for (int k = 0; k < nrow; k++) eitem[it++] = r + k; }   // independent one-sided rows
      else eitem[it++] = r;                                               // one work item per contact
      r += nrow;
      bo += cnd[ci] * (cnd[ci] + 1) / 2;
    }
    cboff[c.ncon] = bo;
    ne = r; nitem = it;
  }
  ne = __shfl_sync(kFull, ne, 0);
  nitem = __shfl_sync(kFull, nitem, 0);
  if (__shfl_sync(kFull, efc_ovf, 0)) c.warn = 1;   // mjWARN_CNSTRFULL
  __syncwarp();
  {
    const int *rootid = MI(body_rootid), *mlo = MI(body_dofmask_lo), *mhi = MI(body_dofmask_hi);
    const float *cpos = DF(con_pos), *cframe = DF(con_frame), *scom = DF(subtree_com), *cdof = DF(cdof),
                *binvw = MF(body_invweight0);
    // dense copies of the contact rows feed the register-blocked Hessian assembly (zeros off the chains)
    float* Jd = DF(efc_Jd);
    const int nvp = (nv + 3) & ~3;   // dense row stride, 16-byte aligned for vector loads
    MJPC_ROLL
    for (int w = lane + (M.nfloss + c.nlim) * nvp; w < ne * nvp; w += 32) Jd[w] = 0.f;
    __syncwarp();
    // compact Jacobian entries: one (contact, local dof) pair per lane
    const int *tadr2 = MI(tendon_adr), *tnum2 = MI(tendon_num), *wdof2 = MI(wrap_dof);
    const float* wcoef = MF(wrap_coef);
    const int nwork = c.ncon * kL;
    for (int w = lane; w < nwork; w += 32) {
      const int ci = w / kL, l = w - ci * kL;
      const int adr = cadr[ci];
      if (adr < 0 || l >= cnd[ci]) continue;
      const int i = cdofl[ci * kL + l];
      const int dim = cdim[ci];
      if (g1a[ci] < 0) {   // tendon limit: J = -side * coef on the wrapped dofs
        const int t = -g1a[ci] - 1;
        float v = 0.f;
        MJPC_ROLL
        for (int w2 = tadr2[t]; w2 < tadr2[t] + tnum2[t]; w2++) if (wdof2[w2] == i) v += -DF(con_mu)[ci] * wcoef[w2];
        J[adr * kL + l] = v;
        Jd[adr * nvp + i] = v;
        continue;
      }
      const int b1 = gbody[g1a[ci]], b2 = gbody[g2a[ci]];
      float jp[3] = {0, 0, 0}, jr[3] = {0, 0, 0};
      const float* cd = cdof + 6 * i;
      for (int s2 = 0; s2 < 2; s2++) {
        const int bb = s2 ? b2 : b1;
        if (bb <= 0) continue;
        const unsigned lo = (unsigned)mlo[bb], hi = (unsigned)mhi[bb];
        const bool on = i < 32 ? ((lo >> i) & 1u) : ((hi >> (i - 32)) & 1u);
        if (!on) continue;
        float off[3], t[3];
        for (int q = 0; q < 3; q++) off[q] = cpos[3 * ci + q] - scom[3 * rootid[bb] + q];
        cross3(t, cd, off);
        const float sg = s2 ? 1.f : -1.f;
        for (int q = 0; q < 3; q++) { jp[q] += sg * (cd[3 + q] + t[q]); jr[q] += sg * cd[q]; }
      }
      const float* fr = cframe + 9 * ci;
      if (pyramidal && dim > 1) {
        const float* mu = DF(con_friction) + 5 * ci;
        const float vn = dot3(fr, jp);
        for (int k = 1; k < dim; k++) {
          const float* ax = fr + 3 * (k % 3);
          const float vt = mu[k - 1] * (k < 3 ? dot3(ax, jp) : dot3(ax, jr));
          const int r0 = adr + 2 * (k - 1);
          J[r0 * kL + l] = vn + vt; Jd[r0 * nvp + i] = vn + vt;
          J[(r0 + 1) * kL + l] = vn - vt; Jd[(r0 + 1) * nvp + i] = vn - vt;
        }
        continue;
      }
      for (int k = 0; k < dim; k++) {
        const float* ax = fr + 3 * (k % 3);
        const float v = k < 3 ? dot3(ax, jp) : dot3(ax, jr);
        J[(adr + k) * kL + l] = v;
        Jd[(adr + k) * nvp + i] = v;
      }
    }
    // per-row scalars: one contact per lane
    for (int ci = lane; ci < c.ncon; ci += 32) {
      const int adr = cadr[ci];
      if (adr < 0) continue;
      if (g1a[ci] < 0) {
        epos[adr] = DF(con_dist)[ci]; emargin[adr] = DF(con_margin)[ci];
        ediag[adr] = MF(tendon_invweight0)[-g1a[ci] - 1];
        etype[adr] = CNSTR_CONTACT_FRICTIONLESS; eid[adr] = ci; efloss[adr] = 0;
        continue;
      }
      const int b1 = gbody[g1a[ci]], b2 = gbody[g2a[ci]];
      const int dim = cdim[ci];
      const float tran = binvw[2 * b1] + binvw[2 * b2], rot = binvw[2 * b1 + 1] + binvw[2 * b2 + 1];
      if (pyramidal && dim > 1) {
        const float* mu = DF(con_friction) + 5 * ci;
        for (int k = 1; k < dim; k++)
          for (int e = 0; e < 2; e++) {
            const int r = adr + 2 * (k - 1) + e;
            epos[r] = DF(con_dist)[ci]; emargin[r] = DF(con_margin)[ci];
            ediag[r] = tran + mu[k - 1] * mu[k - 1] * (k < 3 ? tran : rot);
            etype[r] = CNSTR_CONTACT_FRICTIONLESS;   // a pyramid edge is a one-sided quadratic row
            eid[r] = ci; efloss[r] = 0;
          }
        continue;
      }
      for (int k = 0; k < dim; k++) {
        const int r = adr + k;
        epos[r] = k == 0 ? DF(con_dist)[ci] : 0.f;
        emargin[r] = DF(con_margin)[ci];
        ediag[r] = k >= 3 ? rot : tran;
        etype[r] = dim == 1 ? CNSTR_CONTACT_FRICTIONLESS : CNSTR_CONTACT_ELLIPTIC;
        eid[r] = ci; efloss[r] = 0;
      }
    }
  }
  __syncwarp();
  // --- impedance / regularisation per row
  {
    float *R = DF(efc_R), *K = DF(efc_K), *B = DF(efc_B), *imp_a = DF(efc_imp);
    for (int i = lane; i < ne; i += 32) {
      const float *solref, *solimp;
      const int id = eid[i];
      bool friction_row = false;
      const int ty = etype[i];
      bool zero_dmin = false;   // MakeDifferentiable zeroes solimp[0] of joints and geoms (not of dofs / tendons)
      if (ty == CNSTR_FRICTION_DOF) { solref = MF(dof_solref) + 2 * id; solimp = MF(dof_solimp) + 5 * id; friction_row = true; }
      else if (ty == CNSTR_LIMIT_JOINT) { solref = MF(jnt_solref) + 2 * id; solimp = MF(jnt_solimp) + 5 * id; zero_dmin = CM(c).differentiable != 0.f; }
      else {
        solref = DF(con_solref) + 2 * id; solimp = DF(con_solimp) + 5 * id;
        friction_row = (ty == CNSTR_CONTACT_ELLIPTIC && i > cadr[id]);
        zero_dmin = CM(c).differentiable != 0.f && g1a[id] >= 0;   // geometric contacts only (tendon limits keep theirs)
      }
      const float imp = get_impedance(solimp, epos[i], emargin[i], zero_dmin);
      const float dmax = fminf(kMaxImp, fmaxf(kMinImp, solimp[1]));
      float Kk, Bb;
      if (solref[0] > 0) {
        float tc = solref[0];
        const float dr = solref[1];
        if (!M.disable_refsafe) tc = fmaxf(tc, 2 * CM(c).timestep);
        Kk = 1 / fmaxf(kMinVal, dmax * dmax * tc * tc * dr * dr);
        Bb = 2 / fmaxf(kMinVal, dmax * tc);
      } else {
        Kk = -solref[0] / fmaxf(kMinVal, dmax * dmax);
        Bb = -solref[1] / fmaxf(kMinVal, dmax);
      }
      if (friction_row) Kk = 0;
      K[i] = Kk; B[i] = Bb; imp_a[i] = imp;
      R[i] = fmaxf(kMinVal, (1 - imp) * ediag[i] / imp);
    }
    __syncwarp();
    for (int ci = lane; ci < c.ncon; ci += 32) {
      const int a = cadr[ci], dim = cdim[ci];
      if (a < 0 || dim == 1) continue;
      const float* fr = DF(con_friction) + 5 * ci;
      if (pyramidal) {
        // all edges share R = 2 mu^2 R_first; from here on con_dim is the contact's ROW count
        const float mu = fr[0] * sqrtf(1.f / fmaxf(kMinVal, CM(c).impratio));
        const float Rpy = 2.f * mu * mu * R[a];
        MJPC_ROLL
        for (int j = 0; j < 2 * (dim - 1); j++) R[a + j] = Rpy;
        DF(con_mu)[ci] = mu;
        cdim[ci] = 2 * (dim - 1);
        continue;
      }
      R[a + 1] = R[a] / fmaxf(kMinVal, CM(c).impratio);
      DF(con_mu)[ci] = fr[0] * sqrtf(R[a + 1] / R[a]);
      MJPC_ROLL
      for (int j = 1; j < dim - 1; j++) R[a + j + 1] = R[a + 1] * fr[0] * fr[0] / (fr[j] * fr[j]);
    }
    __syncwarp();
    float* D = DF(efc_D);
    MJPC_ROLL
    for (int i = lane; i < ne; i += 32) D[i] = 1 / R[i];
  }
  // --- wrench-space form of the rows of ONE-SIDED contacts (one geom on a body without dofs): J[row][i] = w_row . cdof_i
  //     for every dof i in the moving body's chain, w_row = side * (off x axis ; axis) for a translational direction and
  //     side * (axis ; 0) for a rotational one, off = contact point - com-frame origin.  The Newton Hessian of these
  //     rows is then assembled as a composite "contact inertia" over the kinematic tree (k_hessian) instead of one rank-1
  //     update per row.  Rows of contacts between two moving bodies and of tendon limits keep the row-by-row path
  //     (efc_drow).
  {
    int *cside = DI(con_side), *cmb = DI(con_mbody), *drow = DI(efc_drow);
    const int* chnum = MI(chain_num);
    const int* rootid = MI(body_rootid);
    const float *cpos = DF(con_pos), *cframe = DF(con_frame), *scom = DF(subtree_com);
    float* W6 = DF(efc_w);
    for (int ci = lane; ci < c.ncon; ci += 32) {
      int side = 0, mb = 0;
      if (g1a[ci] >= 0) {
        const int b1 = gbody[g1a[ci]], b2 = gbody[g2a[ci]];
        if (chnum[b1] == 0 && chnum[b2] > 0) { side = 1; mb = b2; }
        else if (chnum[b2] == 0 && chnum[b1] > 0) { side = -1; mb = b1; }
      }
      cside[ci] = side; cmb[ci] = (side != 0 && cadr[ci] >= 0) ? mb : -1;   // -1: not part of the composite form
    }
    __syncwarp();
    const int r0 = M.nfloss + c.nlim;
    int nd = 0;
    for (int base = r0; base < ne; base += 32) {
      const int i = base + lane;
      bool dense = false;
      if (i < ne) {
        const int ci = eid[i];
        const int side = cside[ci];
        if (side == 0) dense = true;
        else {
          const int k = i - cadr[ci], nrows = cdim[ci], mb = cmb[ci];   // rows exist only for contacts with cadr >= 0
          const float* fr = cframe + 9 * ci;
          float off[3];
          for (int q = 0; q < 3; q++) off[q] = cpos[3 * ci + q] - scom[3 * rootid[mb] + q];
          float w[6];
          auto axis_w = [&](int a, float* o) {   // direction a of the contact frame: 0..2 translational, 3..5 rotational
            const float* ax = fr + 3 * (a % 3);
            if (a < 3) { cross3(o, off, ax); o[3] = ax[0]; o[4] = ax[1]; o[5] = ax[2]; }
            else { o[0] = ax[0]; o[1] = ax[1]; o[2] = ax[2]; o[3] = o[4] = o[5] = 0.f; }
          };
          if (pyramidal && nrows > 1) {   // pyramid edge: normal +- mu_k * tangent_k
            float wt[6];
            const int kk = k / 2 + 1;
            axis_w(0, w); axis_w(kk, wt);
            const float sm = ((k & 1) ? -1.f : 1.f) * DF(con_friction)[5 * ci + kk - 1];
            for (int q = 0; q < 6; q++) w[q] += sm * wt[q];
          } else {
            axis_w(k, w);
          }
          for (int q = 0; q < 6; q++) W6[6 * i + q] = (float)side * w[q];
        }
      }
      const unsigned mask = __ballot_sync(kFull, dense);
      if (dense) drow[nd + __popc(mask & ((1u << lane) - 1u))] = i;
      nd += __popc(mask);
    }
    c.ndrow = nd;
  }
  c.nefc = ne;
  c.nitem = nitem;
  __syncwarp();
}

// ------------------------------------------------------------------------------------------ velocity stage
template <class SP>
__device__ __noinline__ void k_com_vel(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  float *cvel = DF(cvel), *cdof = DF(cdof), *cdof_dot = DF(cdof_dot), *qvel = DF(qvel);
  if (lane < 6) cvel[lane] = 0;
  __syncwarp();
  const int *level_adr = MI(level_adr), *level_body = MI(level_body), *parentid = MI(body_parentid),
            *jntadr = MI(body_jntadr), *jntnum = MI(body_jntnum), *jtype = MI(jnt_type), *jdadr = MI(jnt_dofadr);
  for (int l = 0; l < M.nlevel; l++) {
    const int a = level_adr[l], e = level_adr[l + 1];
    for (int k = a + lane; k < e; k += 32) {
      const int b = level_body[k];
      float v[6];
      for (int q = 0; q < 6; q++) v[q] = cvel[6 * parentid[b] + q];
      for (int j = jntadr[b]; j < jntadr[b] + jntnum[b]; j++) {
        int da = jdadr[j];
        const int t = jtype[j];
        if (t == JNT_FREE) {
          for (int kk = 0; kk < 3; kk++)
            for (int q = 0; q < 6; q++) { cdof_dot[6 * (da + kk) + q] = 0; v[q] += cdof[6 * (da + kk) + q] * qvel[da + kk]; }
          da += 3;
        }
        if (t == JNT_FREE || t == JNT_BALL) {
          for (int kk = 0; kk < 3; kk++) cross_motion(cdof_dot + 6 * (da + kk), v, cdof + 6 * (da + kk));
          for (int kk = 0; kk < 3; kk++)
            for (int q = 0; q < 6; q++) v[q] += cdof[6 * (da + kk) + q] * qvel[da + kk];
        } else {
          cross_motion(cdof_dot + 6 * da, v, cdof + 6 * da);
          for (int q = 0; q < 6; q++) v[q] += cdof[6 * da + q] * qvel[da];
        }
      }
      for (int q = 0; q < 6; q++) cvel[6 * b + q] = v[q];
    }
    __syncwarp();
  }
  // subtree linear velocity
  const int *rootid = MI(body_rootid), *subend = MI(body_subtreeend);
  const float *mass = MF(body_mass), *submass = MF(body_subtreemass);
  float *blin = DF(body_linvel), *slin = DF(subtree_linvel), *xipos = DF(xipos), *scom = DF(subtree_com);
  for (int b = lane; b < M.nbody; b += 32) {
    float off[3], wx[3];
    for (int q = 0; q < 3; q++) off[q] = xipos[3 * b + q] - scom[3 * rootid[b] + q];
    cross3(wx, cvel + 6 * b, off);
    for (int q = 0; q < 3; q++) blin[3 * b + q] = mass[b] * (cvel[6 * b + 3 + q] + wx[q]);
  }
  __syncwarp();
  for (int b = lane; b < M.nbody; b += 32) {
    float s[3] = {0, 0, 0};
    MJPC_ROLL
    for (int q = subend[b] - 1; q >= b; q--)
      for (int k = 0; k < 3; k++) s[k] += blin[3 * q + k];
    for (int k = 0; k < 3; k++) slin[3 * b + k] = s[k] / fmaxf(kMinVal, submass[b]);
  }
  __syncwarp();
}

// passive forces, RNE bias, actuation, qfrc_smooth, qacc_smooth
template <class SP>
__device__ __noinline__ void k_smooth_forces(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  float *qvel = DF(qvel), *qpos = DF(qpos), *passive = DF(qfrc_passive);
  const float* damping = MF(dof_damping);
  for (int i = lane; i < nv; i += 32) passive[i] = -damping[i] * qvel[i];
  __syncwarp();
  {
    const float *stiff = MF(jnt_stiffness), *qspring = MF(qpos_spring);
    const int *jtype = MI(jnt_type), *jdadr = MI(jnt_dofadr), *jqadr = MI(jnt_qposadr);
    for (int j = lane; j < M.njnt; j += 32) {
      if (stiff[j] == 0) continue;
      const int t = jtype[j];
      if (t == JNT_SLIDE || t == JNT_HINGE) passive[jdadr[j]] -= stiff[j] * (qpos[jqadr[j]] - qspring[jqadr[j]]);
    }
  }
  // RNE with qacc = 0
  float *cacc = DF(cacc), *cfrc = DF(cfrc), *cfs = DF(cfrc_sub), *cvel = DF(cvel), *cdof_dot = DF(cdof_dot),
        *cinert = DF(cinert), *cdof = DF(cdof);
  if (lane < 6) cacc[lane] = lane < 3 ? 0.f : -CM(c).gravity[lane - 3];
  __syncwarp();
  const int *level_adr = MI(level_adr), *level_body = MI(level_body), *parentid = MI(body_parentid),
            *dofadr = MI(body_dofadr), *dofnum = MI(body_dofnum), *subend = MI(body_subtreeend);
  for (int l = 0; l < M.nlevel; l++) {
    const int a = level_adr[l], e = level_adr[l + 1];
    for (int k = a + lane; k < e; k += 32) {
      const int b = level_body[k];
      float acc[6];
      for (int q = 0; q < 6; q++) acc[q] = cacc[6 * parentid[b] + q];
      for (int i = dofadr[b]; i < dofadr[b] + dofnum[b]; i++)
        for (int q = 0; q < 6; q++) acc[q] += cdof_dot[6 * i + q] * qvel[i];
      for (int q = 0; q < 6; q++) cacc[6 * b + q] = acc[q];
      float f1[6], iv[6], f2[6];
      mul_inert_vec(f1, cinert + 10 * b, acc);
      mul_inert_vec(iv, cinert + 10 * b, cvel + 6 * b);
      cross_force(f2, cvel + 6 * b, iv);
      for (int q = 0; q < 6; q++) cfrc[6 * b + q] = f1[q] + f2[q];
    }
    __syncwarp();
  }
  for (int b = 1 + lane; b < M.nbody; b += 32) {
    float s[6] = {0, 0, 0, 0, 0, 0};
    for (int q = subend[b] - 1; q >= b; q--)
      for (int k = 0; k < 6; k++) s[k] += cfrc[6 * q + k];
    for (int k = 0; k < 6; k++) cfs[6 * b + k] = s[k];
  }
  __syncwarp();
  const int* dbody = MI(dof_bodyid);
  float* bias = DF(qfrc_bias);
  for (int i = lane; i < nv; i += 32) {
    float s = 0;
    for (int q = 0; q < 6; q++) s += cdof[6 * i + q] * cfs[6 * dbody[i] + q];
    bias[i] = s;
  }
  // actuation (joint transmission; one actuator per joint assumed not required: atomics avoided by per-dof gather)
  float *qact = DF(qfrc_actuator), *aforce = DF(actuator_force), *ctrl = DF(ctrl);
  {
    const int *trnid = MI(actuator_trnid), *biastype = MI(actuator_biastype), *ctrllim = MI(actuator_ctrllimited),
              *frclim = MI(actuator_forcelimited), *jqadr = MI(jnt_qposadr), *jdadr = MI(jnt_dofadr);
    const float *gear = MF(actuator_gear), *gainprm = MF(actuator_gainprm), *biasprm = MF(actuator_biasprm),
                *ctrlrange = MF(actuator_ctrlrange), *frcrange = MF(actuator_forcerange);
    // transmission: a joint (mjTRN_JOINT) or a fixed tendon (mjTRN_TENDON: length / velocity / moment through the
    // tendon's wrap coefficients - e.g. the coupled distal finger joints of the Shadow Hand)
    const int *trntype = MI(actuator_trntype), *tadr = MI(tendon_adr), *tnum = MI(tendon_num), *wq = MI(wrap_qposadr),
              *wdof = MI(wrap_dof);
    const float* wcoef = MF(wrap_coef);
    for (int i = lane; i < M.nu; i += 32) {
      float u = ctrl[i];
      if (ctrllim[i]) u = fmaxf(ctrlrange[2 * i], fminf(ctrlrange[2 * i + 1], u));
      const int j = trnid[i];
      float force = gainprm[3 * i] * u;
      if (biastype[i] == 1) {
        float length, vel;
        if (trntype[i] == 1) {
          length = 0.f; vel = 0.f;
          MJPC_ROLL
          for (int w = tadr[j]; w < tadr[j] + tnum[j]; w++) { length += wcoef[w] * qpos[wq[w]]; vel += wcoef[w] * qvel[wdof[w]]; }
          length *= gear[i]; vel *= gear[i];
        } else {
          length = gear[i] * qpos[jqadr[j]]; vel = gear[i] * qvel[jdadr[j]];
        }
        force += biasprm[3 * i] + biasprm[3 * i + 1] * length + biasprm[3 * i + 2] * vel;
      }
      if (frclim[i]) force = fmaxf(frcrange[2 * i], fminf(frcrange[2 * i + 1], force));
      aforce[i] = force;
    }
    __syncwarp();
    for (int d = lane; d < nv; d += 32) {
      float s = 0;
      MJPC_ROLL
      for (int i = 0; i < M.nu; i++) {
        if (trntype[i] == 1) {
          const int t = trnid[i];
          MJPC_ROLL
          for (int w = tadr[t]; w < tadr[t] + tnum[t]; w++) if (wdof[w] == d) s += gear[i] * wcoef[w] * aforce[i];
        } else if (jdadr[trnid[i]] == d) {
          s += gear[i] * aforce[i];
        }
      }
      qact[d] = s;
    }
  }
  __syncwarp();
  float* smooth = DF(qfrc_smooth);
  for (int i = lane; i < nv; i += 32) smooth[i] = passive[i] - bias[i] + qact[i];
  if (c.xfrc_on) {
    // mj_xfrcAccumulate: force / torque at the centre of mass of every body in the subtree of the dof's body
    // (DFS order: a contiguous body range), mapped through the com-based motion axis of the dof
    const float *xf = DF(xfrc), *cdof = DF(cdof), *xipos = DF(xipos), *scom = DF(subtree_com);
    const int *dbody = MI(dof_bodyid), *subend = MI(body_subtreeend), *rootid = MI(body_rootid);
    for (int i = lane; i < nv; i += 32) {
      const int b0 = dbody[i];
      const float* cd = cdof + 6 * i;
      float a = 0.f;
      MJPC_ROLL
      for (int b = b0; b < subend[b0]; b++) {
        float off[3], t[3];
        for (int q = 0; q < 3; q++) off[q] = xipos[3 * b + q] - scom[3 * rootid[b] + q];
        cross3(t, cd, off);
        const float* f = xf + 6 * b;
        for (int q = 0; q < 3; q++) a += (cd[3 + q] + t[q]) * f[q] + cd[q] * f[3 + q];
      }
      smooth[i] += a;
    }
  }
  __syncwarp();
  spd_solve<SP>(c, SP::kTreeFactor ? DF(qM) : DF(qLD), DF(ldinv), DF(qacc_smooth), smooth, true);
}

// constraint reference acceleration aref = -B*vel - K*imp*(pos - margin)
template <class SP>
__device__ __noinline__ void k_reference(Ctx& c) {
  const int lane = c.lane;
  const float *qvel = DF(qvel), *K = DF(efc_K), *B = DF(efc_B), *imp = DF(efc_imp), *pos = DF(efc_pos),
              *margin = DF(efc_margin);
  float* aref = DF(efc_aref);
  const int nsimple = SP::model(c).nfloss + c.nlim;
  for (int i = lane; i < c.nefc; i += 32) {
    const float v = row_dot<SP>(c, i, nsimple, qvel);
    aref[i] = -B[i] * v - K[i] * imp[i] * (pos[i] - margin[i]);
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------ primal Newton solver
// Evaluate constraint cost at jar; writes force/state; returns warp-uniform cost. If hess, also writes the
// per-row Hessian weights hw[] (H += hw[r] * J_r^T J_r) and, for contacts in the cone zone, two extra
// "effective rows" per contact (the cone Hessian is rank-1 + weighted identity + rank-1 in scaled coordinates):
//   Dm*S*(v v^T + c1*P + c2*ut ut^T)*S,  v = (1, -mu*u/T), ut = (0, u), c1 = mu^2 - mu*N/T, c2 = mu*N/T^3 - mu^2/T^2
//   X_v = sum_a S_a v_a J_a (weight Dm),  X_u = sum_{a>=1} S_a u_a J_a (weight Dm*c2),  hw[a>=1] = Dm*c1*S_a^2
template <class SP>
__device__ __noinline__ float k_update_constraint(Ctx& c, bool hess) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float *jar = DF(efc_jar), *D = DF(efc_D), *R = DF(efc_R), *floss = DF(efc_floss), *J = DF(efc_J);
  float *force = DF(efc_force), *X = DF(efc_W), *hw = DF(efc_hw), *xw = DF(efc_hc);
  int *state = DI(efc_state);
  const int *etype = DI(efc_type), *eid = DI(efc_id), *item = DI(efc_item), *cdim = DI(con_dim);
  float cost = 0;
  for (int it = lane; it < c.nitem; it += 32) {
    const int i = item[it];
    const int ty = etype[i];
    const float Di = D[i], x = jar[i];
    if (ty == CNSTR_FRICTION_DOF) {
      const float f = floss[i], rf = R[i] * f;
      float w = 0.f;
      if (x <= -rf) { cost += f * (-0.5f * rf - x); force[i] = f; state[i] = STATE_LINEARNEG; }
      else if (x >= rf) { cost += f * (-0.5f * rf + x); force[i] = -f; state[i] = STATE_LINEARPOS; }
      else { cost += 0.5f * Di * x * x; force[i] = -Di * x; state[i] = STATE_QUADRATIC; w = Di; }
      hw[i] = w;
    } else if (ty == CNSTR_LIMIT_JOINT || ty == CNSTR_CONTACT_FRICTIONLESS) {
      if (x < 0) { cost += 0.5f * Di * x * x; force[i] = -Di * x; state[i] = STATE_QUADRATIC; hw[i] = Di; }
      else { force[i] = 0; state[i] = STATE_SATISFIED; hw[i] = 0.f; }
    } else {
      const int ci = eid[i];
      const int dim = cdim[ci];
      const float mu = DF(con_mu)[ci];
      const float* fr = DF(con_friction) + 5 * ci;
      float u[6];
      u[0] = jar[i] * mu;
      float tt = 0;
      FOR_DIM(j, 1, dim) { u[j] = jar[i + j] * fr[j - 1]; tt += u[j] * u[j]; }
      const float N = u[0], Tn = sqrtf(tt);
      if (N >= mu * Tn || (Tn <= 0 && N >= 0)) {
        FOR_DIM(j, 0, dim) { force[i + j] = 0; state[i + j] = STATE_SATISFIED; hw[i + j] = 0.f; }
      } else if (mu * N + Tn <= 0 || (Tn <= 0 && N < 0)) {
        FOR_DIM(j, 0, dim) {
          cost += 0.5f * D[i + j] * jar[i + j] * jar[i + j];
          force[i + j] = -D[i + j] * jar[i + j];
          state[i + j] = STATE_QUADRATIC;
          hw[i + j] = D[i + j];
        }
      } else {
        const float Dm = Di / (mu * mu * (1 + mu * mu));
        const float NmT = N - mu * Tn;
        cost += 0.5f * Dm * NmT * NmT;
        const float f0 = -Dm * NmT * mu;
        const float iT = 1.0f / Tn;
        force[i] = f0;
        FOR_DIM(j, 1, dim) force[i + j] = -f0 * iT * u[j] * fr[j - 1];
        FOR_DIM(j, 0, dim) state[i + j] = STATE_CONE;
        if (hess) {
          const float c1 = mu * mu - mu * N * iT;
          hw[i] = 0.f;
          FOR_DIM(j, 1, dim) hw[i + j] = Dm * c1 * fr[j - 1] * fr[j - 1];
          // coefficients of the two effective rows, stored per contact: [S_a v_a (6), S_a u_a (6), wv, wu]
          float* q = xw + 36 * ci;
          q[0] = mu; q[6] = 0.f;
          FOR_DIM(j, 1, dim) { q[j] = -fr[j - 1] * mu * u[j] * iT; q[6 + j] = fr[j - 1] * u[j]; }
          q[12] = Dm;
          q[13] = Dm * (mu * N * iT * iT * iT - mu * mu * iT * iT);
        }
      }
    }
  }
  cost = warp_sum(cost);
  __syncwarp();
  return cost;
}

// Newton Hessian for compile-time NV: one rolled pass over the structurally non-zero lower-triangle entries (hpair
// tables), entry e on thread e of the group per round; every active constraint row and every cone effective row adds
// its rank-1 term, read as a dense row from shared memory (broadcast loads, no bank conflicts).  NQ (entries per lane
// of one warp) is not read: it only keeps k_hessian's two nv = 18 instances apart.
template <class SP, int NV, int NQ, bool kHelpers = false>
__device__ __forceinline__ void hessian_dense_reg(Ctx& c) {
  auto&& M = SP::model(c);
  using G = WideGroup<SP, kHelpers>;   // the thread group that assembles (the warp, all W warps, or the helpers: dev_data.cuh)
  const int lane = G::lane(c);         // index within that group
  constexpr int WN = 32 * G::kWarps;
  constexpr int NVP = (NV + 3) / 4 * 4;
  const float *qM = DF(qM), *hw = DF(efc_hw), *Jd = DF(efc_Jd), *Xd = DF(efc_Xd), *xw = DF(efc_hc);
  float* H = DF(qH);
  const int *frow = MI(floss_row), *edof = DI(efc_dof), *state = DI(efc_state), *cadr = DI(con_adr),
            *hi = MI(hpair_i), *hj = MI(hpair_j), *cside = DI(con_side), *cdim = DI(con_dim);
  const int NE = M.nhpair, ncon = c.ncon;
  // ---- one-sided contacts: composite contact "inertia".  With J[row][i] = w_row . cdof_i on the moving body's chain,
  //      sum_rows (weights) J^T J = cdof_r^T ( sum over contacts below body(r) of W_c ) cdof_s,  W_c (6x6) = sum_a hw_a
  //      w_a w_a^T + cone terms - the same subtree-composite structure as the joint-space inertia itself (k_crb).
  float* Wc = DF(efc_blk);        // [ncon][21] lower triangles (the generic path's block scratch, unused here)
  float* g = DF(dofbuf);          // [nv][6]   (k_crb's scratch, free after qM was formed)
  const float* W6 = DF(efc_w);
  {
    // cone effective rows in wrench space: V = sum_a q_a w_a, U = sum_a q_{6+a} w_a  -> efc_hc[36 ci + 14 ..]
    float* xwm = DF(efc_hc);
    MJPC_ROLL
    for (int w = lane; w < ncon * 6; w += WN) {
      const int ci = w / 6, p = w - 6 * ci;
      const int a0 = cadr[ci];
      float v = 0.f, u = 0.f;
      if (a0 >= 0 && cside[ci] != 0 && state[a0] == STATE_CONE) {
        const int dim = cdim[ci];
        const float* q = xw + 36 * ci;
        FOR_DIM(a, 0, dim) { const float wa = W6[6 * (a0 + a) + p]; v += q[a] * wa; u += q[6 + a] * wa; }
      }
      xwm[36 * ci + 14 + p] = v; xwm[36 * ci + 20 + p] = u;   // zeros for non-cone contacts: read (times 0) below
    }
    G::bar();
    // (straight-line: clamped indices, weights selected to zero instead of branches - every taken branch costs a
    // reconvergence (BSSY/BSYNC ~30 cycles) with a single resident warp)
    constexpr int kMaxRows = 10;   // pyramidal condim 6; elliptic contacts have <= 6 rows
    const bool pyr = M.cone == CONE_PYRAMIDAL;
    const int nwork = ncon * 21;
    MJPC_ROLL
    for (int base = 0; base < nwork; base += WN) {
      const int w = min(base + lane, nwork - 1);
      const int ci = w / 21, e = w - 21 * ci;
      const int p = (e >= 1) + (e >= 3) + (e >= 6) + (e >= 10) + (e >= 15);
      const int q2 = e - p * (p + 1) / 2;
      const int a0r = cadr[ci];
      const bool on = a0r >= 0 && cside[ci] != 0;
      const int a0 = max(a0r, 0);
      const int nrows = on ? cdim[ci] : 0;
      float acc = 0.f;
#pragma unroll 1
      for (int a = 0; a < kMaxRows; a++) {
        if (a >= 6 && !pyr) break;                       // compile-time for a static spec
        const int r = min(a0 + a, M.maxefc - 1);
        const float t = hw[r] * W6[6 * r + p] * W6[6 * r + q2];   // may read rows of other constraints: selected away
        acc += a < nrows ? t : 0.f;                                // (a select, never a multiply by zero: NaN-safe)
      }
      const float* q = xw + 36 * ci;
      const float tc = q[12] * q[14 + p] * q[14 + q2] + q[13] * q[20 + p] * q[20 + q2];
      acc += (on && state[a0] == STATE_CONE) ? tc : 0.f;
      if (base + lane < nwork) Wc[w] = acc;
    }
    G::bar();
    // g_i = (sum of W_c over the contacts on bodies in the subtree of dof i's body) cdof_i, one (dof, component) per lane
    const int *subend = MI(body_subtreeend), *cmb = DI(con_mbody), *dbody = MI(dof_bodyid);
    const float* cdof = DF(cdof);
    MJPC_ROLL
    for (int w = lane; w < NV * 6; w += WN) {
      const int i = w / 6, k = w - 6 * i;
      const int b = dbody[i], se = subend[b];
      int idx[6];
      float cd[6];
#pragma unroll
      for (int l = 0; l < 6; l++) { idx[l] = k >= l ? k * (k + 1) / 2 + l : l * (l + 1) / 2 + k; cd[l] = cdof[6 * i + l]; }
      float a = 0.f;
      MJPC_ROLL
      for (int ci = 0; ci < ncon; ci++) {
        const int mb = cmb[ci];                       // -1 for two-sided / dropped contacts
        const float* Wk = Wc + 21 * ci;
        float d = 0.f;
#pragma unroll
        for (int l = 0; l < 6; l++) d += Wk[idx[l]] * cd[l];
        a += (mb >= b && mb < se) ? d : 0.f;
      }
      g[w] = a;
    }
    G::bar();
  }
  // one rolled loop over the pattern entries (code footprint), H written directly
  if (NE != NV * (NV + 1) / 2) {   // entries outside the pattern (the dense factor reads them); nothing to clear for a full pattern
    MJPC_ROLL
    for (int w = lane; w < NV * NV; w += WN) H[w] = 0.f;
    G::bar();
  }
  {
    const float* cdof = DF(cdof);
    const int* dbody2 = MI(dof_bodyid);
    const int* drow = DI(efc_drow);
#pragma unroll 1
    for (int e0 = 0; e0 < NE; e0 += WN) {
      const int e = min(e0 + lane, NE - 1);
      const int r = hi[e], sdof = hj[e];
      float a = qM[r * NV + sdof];
      // the composite form holds for (dof, ancestor dof) pairs only - the pattern of M itself; entries that exist in
      // the Hessian pattern because a pair of moving bodies CAN touch (e.g. two legs) get nothing from one-sided contacts
      const int br = dbody2[r];
      const unsigned mlo_r = (unsigned)MI(body_dofmask_lo)[br], mhi_r = (unsigned)MI(body_dofmask_hi)[br];
      const bool anc = sdof < 32 ? ((mlo_r >> sdof) & 1u) : ((mhi_r >> (sdof - 32)) & 1u);
      const float *gr = g + 6 * r, *cs = cdof + 6 * sdof;
      float dsum = 0.f;
#pragma unroll
      for (int l = 0; l < 6; l++) dsum += gr[l] * cs[l];
      a += anc ? dsum : 0.f;
      if (r == sdof) {
        const int fr = frow[r];
        if (fr >= 0) a += hw[fr];
        MJPC_ROLL
        for (int k = M.nfloss; k < M.nfloss + c.nlim; k++) { const float hk = hw[k]; a += edof[k] == r ? hk : 0.f; }
      }
      MJPC_ROLL
      for (int k = 0; k < c.ndrow; k++) {
        const int row = drow[k];
        const float* j = Jd + row * NVP;
        a += hw[row] * j[r] * j[sdof];
      }
      if (c.ndrow > 0) {
        MJPC_ROLL
        for (int ci = 0; ci < ncon; ci++) {
          const int a0 = cadr[ci];
          if (a0 < 0 || cside[ci] != 0 || state[a0] != STATE_CONE) continue;   // warp-uniform
          const float wv = xw[36 * ci + 12], wu = xw[36 * ci + 13];
          const float* xv = Xd + (2 * ci) * NVP;
          const float* xu = xv + NVP;
          a += wv * xv[r] * xv[sdof] + wu * xu[r] * xu[sdof];
        }
      }
      if (e0 + lane < NE) { H[r * NV + sdof] = a; H[sdof * NV + r] = a; }
    }
  }
  G::bar();
}

// row i of (NV x NV row-major matrix) times vector, compile-time NV, 8-byte vector loads (NV even)
template <int NV>
__device__ __forceinline__ float mat_row_dot(const float* Mrow, const float* v) {
  float a = 0.f;
  if (NV % 2 == 0) {
    const float2* m2 = reinterpret_cast<const float2*>(Mrow);
    const float2* v2 = reinterpret_cast<const float2*>(v);
#pragma unroll
    for (int k = 0; k < NV / 2; k++) { const float2 x = m2[k], y = v2[k]; a += x.x * y.x + x.y * y.y; }
  } else {
#pragma unroll
    for (int k = 0; k < NV; k++) a += Mrow[k] * v[k];
  }
  return a;
}

// dense-row variants of J*v and J^T*force for compile-time NV (vectorised, fully unrolled)
template <class SP, int NV>
__device__ __forceinline__ float row_dot_dense(Ctx& c, int row, int nsimple, const float* v) {
  constexpr int NVP = (NV + 3) / 4 * 4;
  // both forms are evaluated and one is selected (no divergent region): simple rows touch one dof, contact rows are
  // dense; the dense rows of simple constraints are never written, hence the select and not a sum
  const float simple = DF(efc_sgn)[row] * v[row < nsimple ? DI(efc_dof)[row] : 0];   // efc_dof is only written for simple rows
  const float dense = mat_row_dot<NV>(DF(efc_Jd) + row * NVP, v);   // NVP is a multiple of 4: rows are 16-byte aligned
  return row < nsimple ? simple : dense;
}
template <class SP, int NV>
__device__ __forceinline__ void jt_force_dense(Ctx& c, float* out) {
  auto&& M = SP::model(c);
  const int lane = c.lane;
  constexpr int NVP = (NV + 3) / 4 * 4;
  const float *Jd = DF(efc_Jd), *force = DF(efc_force), *esgn = DF(efc_sgn);
  const int *frow = MI(floss_row), *edof = DI(efc_dof);
  const int nf = M.nfloss, nl = c.nlim, ne = c.nefc;
  {
    const int li = lane < NV ? lane : NV - 1;   // all lanes run, clamped; the store is predicated
    float a = 0.f;
    const int fr = frow[li];
    const float ff = force[max(fr, 0)];
    a += fr >= 0 ? ff : 0.f;
    for (int q = nf; q < nf + nl; q++) { const float t = esgn[q] * force[q]; a += edof[q] == li ? t : 0.f; }
    for (int row = nf + nl; row < ne; row++) a += Jd[row * NVP + li] * force[row];
    if (lane < NV) out[lane] = a;
  }
  __syncwarp();
}

// size dispatch: a static spec knows nv at compile time (dense, fully unrolled rows); the generic spec keeps the
// runtime fast path for nv == 18 and otherwise the compact rows
template <class SP>
__device__ __forceinline__ float m_row_dot(const float* qM, int i, const float* v, int nv) {
  if constexpr (SP::kNV > 0) return mat_row_dot<SP::kNV>(qM + i * SP::kNV, v);
  else {
    if (nv == 18) return mat_row_dot<18>(qM + i * 18, v);
    float a = 0;
    for (int j = 0; j < nv; j++) a += qM[i * nv + j] * v[j];
    return a;
  }
}
template <class SP>
__device__ __forceinline__ float j_row_dot(Ctx& c, int row, int nsimple, const float* v, int nv) {
  if constexpr (SP::kNV > 0) return row_dot_dense<SP, SP::kNV>(c, row, nsimple, v);
  else return nv == 18 ? row_dot_dense<SP, 18>(c, row, nsimple, v) : row_dot<SP>(c, row, nsimple, v);
}
// Ma = M*qacc, jar = J*qacc - aref, gauss; returns total cost (uniform). If hess: qH = M + J^T diag(hw) J + cone rows,
// assembled in two balanced stages: (1) every contact's small symmetric block (its chain dofs) into scratch,
// one (contact, block entry) per lane; (2) every structurally non-zero Hessian entry gathers the blocks that
// contain it (deterministic order, no atomics).
template <class SP>
__device__ __noinline__ float k_total_cost(Ctx& c, const float* qacc, bool hess, float* gauss_out, float step = 0.f) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float *qM = DF(qM), *J = DF(efc_J), *aref = DF(efc_aref), *smooth = DF(qfrc_smooth), *qas = DF(qacc_smooth);
  float *Ma = DF(Ma), *jar = DF(efc_jar);
  const int nsimple = M.nfloss + c.nlim;
  float g = 0;
  if (step != 0.f) {
    // qacc moved by step * search: M qacc and J qacc - aref follow from the products the line search already formed
    const float *Mv = DF(Mv), *Jv = DF(efc_Jv);
    for (int b0 = 0; b0 < nv; b0 += 32) {
      const int i = min(b0 + lane, nv - 1);
      const bool on = b0 + lane < nv;
      const float a = Ma[i] + step * Mv[i];
      __syncwarp();
      if (on) Ma[i] = a;
      g += on ? (a - smooth[i]) * (qacc[i] - qas[i]) : 0.f;
    }
    const int ne = c.nefc;
    for (int b0 = 0; b0 < ne; b0 += 32) {
      const int i = min(b0 + lane, ne - 1);
      const float v = jar[i] + step * Jv[i];
      __syncwarp();
      if (b0 + lane < ne) jar[i] = v;
    }
  } else {
    for (int b0 = 0; b0 < nv; b0 += 32) {
      const int i = min(b0 + lane, nv - 1);
      const bool on = b0 + lane < nv;
      const float a = m_row_dot<SP>(qM, i, qacc, nv);
      if (on) Ma[i] = a;
      g += on ? (a - smooth[i]) * (qacc[i] - qas[i]) : 0.f;
    }
    const int ne = c.nefc;
    for (int b0 = 0; b0 < ne; b0 += 32) {
      const int i = min(b0 + lane, ne - 1);
      const float v = j_row_dot<SP>(c, i, nsimple, qacc, nv) - aref[i];
      if (b0 + lane < ne) jar[i] = v;
    }
  }
  g = 0.5f * warp_sum(g);
  __syncwarp();
  const float cc = k_update_constraint<SP>(c, hess);
  *gauss_out = g;
  return cc + g;
}

// Newton Hessian H = M + J^T diag(hw) J + cone blocks at the point last evaluated by k_total_cost(.., hess=true)
// (which leaves the row weights hw and the per-cone coefficients in efc_hc).  Kept apart from the cost evaluation
// so that the solver only assembles and factorises H when another iteration is actually taken.
// ONE out-of-line copy of the static-spec assembly per kernel: the one-warp kernel runs it on its warp (k_hessian), the
// helper-warp kernel on its helper warps alone (wide_helper_loop) while the main warp forms the gradient (k_solve).
// Every work item is computed by one thread in a fixed order whatever the group's size, so the values are the same.
template <class SP>
__device__ __noinline__ void hessian_static(Ctx& c) {
  hessian_dense_reg<SP, SP::kNV, (SP::kNHPair + 31) / 32, (SP::kWide > 1)>(c);
}

// The main warp's part of the assembly: the effective rows of cone contacts that the dense rank-1 pass reads (only
// present with contacts between two moving bodies / tendon limits on the register-blocked path).  Reads efc_J, efc_hc
// [36 ci + 0 .. 13], efc_state, con_*; writes efc_W, efc_Xd.
template <class SP>
__device__ __forceinline__ void hessian_cone_rows(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float* J = DF(efc_J);
  float *X = DF(efc_W);
  const int *state = DI(efc_state), *cdim = DI(con_dim);
  const float* xw = DF(efc_hc);
  const bool tree_path = SP::kNV > 0 || nv == 18;   // hessian_dense_reg: one-sided contacts go through the composite form
  if (!tree_path || c.ndrow > 0) {
    // effective rows of cone contacts (compact): one (contact, local dof) pair per lane
    const int *cadr = DI(con_adr), *cnd = DI(con_nd), *cside = DI(con_side);
    const int total = c.ncon * kL;
    for (int w = lane; w < total; w += 32) {
      const int ci = w / kL, l = w - ci * kL;
      const int a0 = cadr[ci];
      if (a0 < 0 || l >= cnd[ci] || state[a0] != STATE_CONE || (tree_path && cside[ci] != 0)) continue;
      const int dim = cdim[ci];
      const float* q = xw + 36 * ci;
      float xv = 0.f, xu = 0.f;
      FOR_DIM(a, 0, dim) {
        const float jv = J[(a0 + a) * kL + l];
        xv += q[a] * jv;
        xu += q[6 + a] * jv;
      }
      X[(2 * ci) * kL + l] = xv;
      X[(2 * ci + 1) * kL + l] = xu;
    }
    if (SP::kNV > 0 || nv == 18) {   // dense copies for the register-blocked assembly
      const int nvp = (nv + 3) & ~3;
      float* Xd = DF(efc_Xd);
      const int* cloc = DI(con_loc);
      __syncwarp();
      for (int w = lane; w < c.ncon * nv; w += 32) {
        const int ci = w / nv, i = w - ci * nv;
        const int a0 = cadr[ci];
        if (a0 < 0 || state[a0] != STATE_CONE || cside[ci] != 0) continue;
        const int l = cloc[w];
        Xd[(2 * ci) * nvp + i] = l >= 0 ? X[(2 * ci) * kL + l] : 0.f;
        Xd[(2 * ci + 1) * nvp + i] = l >= 0 ? X[(2 * ci + 1) * kL + l] : 0.f;
      }
    }
    __syncwarp();
  }
}

template <class SP>
__device__ __noinline__ void k_hessian(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float *qM = DF(qM), *J = DF(efc_J);
  hessian_cone_rows<SP>(c);
  if constexpr (SP::kNV > 0) {
    static_assert(SP::kWide == 1, "helper-warp kernels assemble on the helpers (k_solve)");
    hessian_static<SP>(c);
    return;
  }
  if (nv == 18 && M.nhpair <= 128) {
    hessian_dense_reg<SP, 18, 4>(c);
  } else if (nv == 18) {
    hessian_dense_reg<SP, 18, 6>(c);
  } else {
    const float *X = DF(efc_W), *hw = DF(efc_hw), *xw = DF(efc_hc);
    float *H = DF(qH), *blk = DF(efc_blk);
    const int *hi = MI(hpair_i), *hj = MI(hpair_j), *frow = MI(floss_row), *state = DI(efc_state), *edof = DI(efc_dof),
              *cadr = DI(con_adr), *cdim = DI(con_dim), *cnd = DI(con_nd), *cloc = DI(con_loc), *cboff = DI(con_boff);
    const int ncon = c.ncon, nf = M.nfloss, nl = c.nlim;
    // M + diagonal rows
    for (int w = lane; w < nv * nv; w += 32) H[w] = 0.f;   // entries outside the pattern (the factor fills them)
    __syncwarp();
    for (int e = lane; e < M.nhpair; e += 32) {
      const int r = hi[e], s2 = hj[e];
      float a = qM[r * nv + s2];
      if (r == s2) {
        const int fr = frow[r];
        if (fr >= 0) a += hw[fr];
        for (int q = nf; q < nf + nl; q++)
          if (edof[q] == r) a += hw[q];
      }
      H[r * nv + s2] = a;
    }
    __syncwarp();
    int c0 = 0;
    while (c0 < ncon) {
      // chunk of contacts whose blocks fit the scratch buffer
      int c1 = c0 + 1;
      while (c1 < ncon && cboff[c1 + 1] - cboff[c0] <= 1024) c1++;
      const int base = cboff[c0], nblk = cboff[c1] - base;
      // stage 1
      int ci = c0;
      for (int t0 = 0; t0 < nblk; t0 += 32) {
        const int t = t0 + lane;
        while (ci + 1 < c1 && cboff[ci + 1] - base <= t0) ci++;   // warp-uniform lower bound
        int cj = ci;
        while (cj + 1 < c1 && cboff[cj + 1] - base <= t) cj++;
        if (t < nblk) {
          const int a0 = cadr[cj];
          float acc = 0.f;
          if (a0 >= 0) {
            const int tt = t - (cboff[cj] - base);
            int la = (int)((sqrtf(8.f * tt + 1.f) - 1.f) * 0.5f);
            while ((la + 1) * (la + 2) / 2 <= tt) la++;
            while (la * (la + 1) / 2 > tt) la--;
            const int lb = tt - la * (la + 1) / 2;
            const int dim = cdim[cj];
            const float* Ja = J + a0 * kL + la;
            const float* Jb = J + a0 * kL + lb;
            for (int k = 0; k < dim; k++) acc += hw[a0 + k] * Ja[k * kL] * Jb[k * kL];
            if (state[a0] == STATE_CONE) {
              const float* q = xw + 36 * cj;
              acc += q[12] * X[(2 * cj) * kL + la] * X[(2 * cj) * kL + lb] + q[13] * X[(2 * cj + 1) * kL + la] * X[(2 * cj + 1) * kL + lb];
            }
          }
          blk[t] = acc;
        }
      }
      __syncwarp();
      // stage 2
      for (int e = lane; e < M.nhpair; e += 32) {
        const int r = hi[e], s2 = hj[e];
        float a = H[r * nv + s2];
        for (int cq = c0; cq < c1; cq++) {
          const int lr = cloc[cq * nv + r], ls = cloc[cq * nv + s2];
          if ((lr | ls) < 0 || cadr[cq] < 0) continue;
          const int mx = max(lr, ls), mn = min(lr, ls);
          a += blk[cboff[cq] - base + mx * (mx + 1) / 2 + mn];
        }
        H[r * nv + s2] = a;
      }
      __syncwarp();
      c0 = c1;
    }
    for (int e = lane; e < M.nhpair; e += 32) { const int r = hi[e], s2 = hj[e]; H[s2 * nv + r] = H[r * nv + s2]; }
    __syncwarp();
  }
}

// Helper warps of a W-warp trajectory group (dev_data.cuh): wait for the main warp's command, run the phase among
// themselves and report it done; the main warp meets them at the join when it needs the result.
template <class SP>
__device__ __noinline__ void wide_helper_loop(Ctx& c) {
  if constexpr (SP::kWide > 1) {
    for (;;) {
      wide_bar<SP>();
      const WideBox& b = wide_box();
      const int cmd = b.cmd;
      if (cmd == WIDE_EXIT) return;
      c.ncon = b.ncon; c.nlim = b.nlim; c.ndrow = b.ndrow; c.nefc = b.nefc;
      if (cmd == WIDE_HESSIAN) hessian_static<SP>(c);
      wide_done<SP>();
    }
  }
}

struct LsPoint { float alpha, cost, d1, d2; };

template <class SP>
__device__ __noinline__ LsPoint k_ls_eval(Ctx& c, float g0, float g1, float g2, float alpha) {
  const int lane = c.lane;
  const float *jar = DF(efc_jar), *Jv = DF(efc_Jv), *D = DF(efc_D), *R = DF(efc_R), *floss = DF(efc_floss);
  const int *etype = DI(efc_type), *eid = DI(efc_id), *item = DI(efc_item), *cdim = DI(con_dim);
  float cost = 0, d1 = 0, d2 = 0;
  for (int it = lane; it < c.nitem; it += 32) {
    const int i = item[it];
    const int ty = etype[i];
    const float Di = D[i], jv = Jv[i], x = jar[i] + alpha * jv;
    if (ty == CNSTR_FRICTION_DOF) {
      const float f = floss[i], rf = R[i] * f;
      if (x <= -rf) { cost += f * (-0.5f * rf - x); d1 += -f * jv; }
      else if (x >= rf) { cost += f * (-0.5f * rf + x); d1 += f * jv; }
      else { cost += 0.5f * Di * x * x; d1 += Di * x * jv; d2 += Di * jv * jv; }
    } else if (ty == CNSTR_LIMIT_JOINT || ty == CNSTR_CONTACT_FRICTIONLESS) {
      if (x < 0) { cost += 0.5f * Di * x * x; d1 += Di * x * jv; d2 += Di * jv * jv; }
    } else {
      const int ci = eid[i];
      const int dim = cdim[ci];
      const float mu = DF(con_mu)[ci];
      const float* fr = DF(con_friction) + 5 * ci;
      const float U0 = jar[i] * mu, V0 = Jv[i] * mu;
      float UU = 0, UV = 0, VV = 0;
      FOR_DIM(j, 1, dim) {
        const float uj = jar[i + j] * fr[j - 1], vj = Jv[i + j] * fr[j - 1];
        UU += uj * uj; UV += uj * vj; VV += vj * vj;
      }
      const float N = U0 + alpha * V0;
      const float Tsqr = UU + alpha * (2 * UV + alpha * VV);
      const float Tn = Tsqr <= 0 ? 0.f : sqrtf(Tsqr);
      if (N >= mu * Tn || (Tn <= 0 && N >= 0)) {
      } else if (mu * N + Tn <= 0 || (Tn <= 0 && N < 0)) {
        FOR_DIM(j, 0, dim) {
          const float Dj = D[i + j], vj = Jv[i + j], xj = jar[i + j] + alpha * vj;
          cost += 0.5f * Dj * xj * xj; d1 += Dj * xj * vj; d2 += Dj * vj * vj;
        }
      } else {
        const float Dm = Di / (mu * mu * (1 + mu * mu));
        const float N1 = V0, T1 = (UV + alpha * VV) / Tn;
        const float T2 = VV / Tn - (UV + alpha * VV) * T1 / (Tn * Tn);
        const float NmT = N - mu * Tn;
        cost += 0.5f * Dm * NmT * NmT;
        d1 += Dm * NmT * (N1 - mu * T1);
        d2 += Dm * ((N1 - mu * T1) * (N1 - mu * T1) + NmT * (-mu * T2));
      }
    }
  }
  LsPoint p;
  p.alpha = alpha;
  p.cost = g0 + alpha * g1 + alpha * alpha * g2 + warp_sum(cost);
  p.d1 = g1 + 2 * alpha * g2 + warp_sum(d1);
  p.d2 = 2 * g2 + warp_sum(d2);
  return p;
}

// Per-lane cache of one work item's line-search data: everything that does not depend on alpha is folded once
// per line search so an evaluation is a handful of register operations plus three warp reductions.
struct LsItem {
  int kind;                 // 0 none, 1 friction-loss, 2 inequality (limit / frictionless), 3 elliptic contact
  float D, x0, jv, f, rf;   // kinds 1, 2
  float mu, U0, V0, UU, UV, VV, Q0, Q1, Q2, Dm;  // kind 3
};

template <class SP>
__device__ __forceinline__ LsItem ls_load_item(Ctx& c) {
  LsItem it;
  it.kind = 0;
  it.D = it.x0 = it.jv = it.f = it.rf = it.mu = it.U0 = it.V0 = it.UU = it.UV = it.VV = it.Q0 = it.Q1 = it.Q2 = it.Dm = 0.f;
  if (c.lane >= c.nitem) return it;
  const float *jar = DF(efc_jar), *Jv = DF(efc_Jv), *D = DF(efc_D), *R = DF(efc_R), *floss = DF(efc_floss);
  const int i = DI(efc_item)[c.lane];
  const int ty = DI(efc_type)[i];
  it.D = D[i]; it.x0 = jar[i]; it.jv = Jv[i];
  if (ty == CNSTR_FRICTION_DOF) { it.kind = 1; it.f = floss[i]; it.rf = R[i] * it.f; }
  else if (ty == CNSTR_LIMIT_JOINT || ty == CNSTR_CONTACT_FRICTIONLESS) { it.kind = 2; }
  else {
    it.kind = 3;
    const int ci = DI(efc_id)[i];
    const int dim = DI(con_dim)[ci];
    const float* fr = DF(con_friction) + 5 * ci;
    it.mu = DF(con_mu)[ci];
    it.U0 = jar[i] * it.mu; it.V0 = Jv[i] * it.mu;
    FOR_DIM(j, 1, dim) {
      const float uj = jar[i + j] * fr[j - 1], vj = Jv[i + j] * fr[j - 1];
      it.UU += uj * uj; it.UV += uj * vj; it.VV += vj * vj;
    }
    FOR_DIM(j, 0, dim) {
      const float Dj = D[i + j], xj = jar[i + j], vj = Jv[i + j];
      it.Q0 += Dj * xj * xj; it.Q1 += Dj * xj * vj; it.Q2 += Dj * vj * vj;
    }
    it.Dm = it.D / (it.mu * it.mu * (1 + it.mu * it.mu));
  }
  return it;
}

// Straight-line evaluation (selects, no branches): the three constraint kinds sit on different lanes, so a branchy
// version executes every path anyway and pays a reconvergence per path on top.  Divisions by Tn = 0 produce inf / NaN
// in lanes whose result is then selected away (never multiplied by zero).
// (selection by bit masks, not by ?: - the compiler turns chains of selects over the three kinds into divergent
// branches with a reconvergence point each (5 BSSY/BSYNC pairs in the first version of this function), and with the
// kinds spread over the lanes every branch is taken by somebody; the selected VALUES are the same, so are the results)
__device__ __forceinline__ float ls_pick(float a, bool ma, float b, bool mb, float c2, bool mc) {
  return __int_as_float((__float_as_int(a) & (ma ? -1 : 0)) | (__float_as_int(b) & (mb ? -1 : 0)) | (__float_as_int(c2) & (mc ? -1 : 0)));
}
__device__ __forceinline__ LsPoint ls_eval_cached(const LsItem& it, float g0, float g1, float g2, float alpha) {
  // kinds 1, 2: scalar row
  const float x = it.x0 + alpha * it.jv;
  const float qc = 0.5f * it.D * x * x, qd1 = it.D * x * it.jv, qd2 = it.D * it.jv * it.jv;
  const bool neg = x <= -it.rf, pos = x >= it.rf, mid = !(neg || pos);
  const float c1 = ls_pick(it.f * (-0.5f * it.rf - x), neg, it.f * (-0.5f * it.rf + x), pos && !neg, qc, mid);
  const float d11 = ls_pick(-it.f * it.jv, neg, it.f * it.jv, pos && !neg, qd1, mid);
  const bool act2 = x < 0.f;
  // kind 3: elliptic cone
  const float mu = it.mu;
  const float N = it.U0 + alpha * it.V0;
  const float Tsqr = it.UU + alpha * (2 * it.UV + alpha * it.VV);
  const float Tn = Tsqr <= 0 ? 0.f : sqrtf(Tsqr);
  const bool top = N >= mu * Tn || (Tn <= 0 && N >= 0);
  const bool bottom = !top && (mu * N + Tn <= 0 || (Tn <= 0 && N < 0));
  const bool middle = !top && !bottom;
  const float iT = 1.0f / Tn;
  const float N1 = it.V0, T1 = (it.UV + alpha * it.VV) * iT;
  const float T2 = it.VV * iT - (it.UV + alpha * it.VV) * T1 * iT * iT;
  const float NmT = N - mu * Tn, s1 = N1 - mu * T1;
  const int k = it.kind;
  const bool k1 = k == 1, k2 = (k == 2) && act2, k3b = (k == 3) && bottom, k3m = (k == 3) && middle;
  // (kind 3 contributes through exactly one of the bottom / middle zones or not at all; kinds 1 and 2 are exclusive)
  const float cost = ls_pick(c1, k1, qc, k2, ls_pick(0.5f * (it.Q0 + alpha * (2 * it.Q1 + alpha * it.Q2)), k3b, 0.5f * it.Dm * NmT * NmT, k3m, 0.f, false), k3b || k3m);
  const float d1 = ls_pick(d11, k1, qd1, k2, ls_pick(it.Q1 + alpha * it.Q2, k3b, it.Dm * NmT * s1, k3m, 0.f, false), k3b || k3m);
  const float d2 = ls_pick(qd2, k1 && mid, qd2, k2, ls_pick(it.Q2, k3b, it.Dm * (s1 * s1 + NmT * (-mu * T2)), k3m, 0.f, false), k3b || k3m);
  LsPoint p;
  p.alpha = alpha;
  p.cost = g0 + alpha * g1 + alpha * alpha * g2 + warp_sum(cost);
  p.d1 = g1 + 2 * alpha * g2 + warp_sum(d1);
  p.d2 = 2 * g2 + warp_sum(d2);
  return p;
}

// one shared copy of the evaluation for the ~6 call sites of the line search (the item travels by value in registers)
__device__ __noinline__ LsPoint ls_eval_cached_shared(LsItem it, float g0, float g1, float g2, float alpha) {
  return ls_eval_cached(it, g0, g1, g2, alpha);
}

template <class SP>
__device__ __noinline__ float k_line_search(Ctx& c, float g0, float g1, float g2, float snorm, float scale_inv) {
  auto&& M = SP::model(c);
  if (snorm < kMinVal) return 0.f;
  const bool cached = c.nitem <= 32;   // one work item per lane: the usual case
  const LsItem item = ls_load_item<SP>(c);
  auto ev = [&](float alpha) {
#if defined(MJPC_PHASE_TIMING) && MJPC_PHASE_MAP == 1
    c.tph[7]++;   // timer mapping 1: slot 7 counts the evaluations
#endif
    return cached ? ls_eval_cached_shared(item, g0, g1, g2, alpha) : k_ls_eval<SP>(c, g0, g1, g2, alpha);
  };
  const LsPoint p0 = ev(0.f);
  const float gtol = fmaxf(fmaxf(CM(c).tolerance, kTolFloor) * CM(c).ls_tolerance * snorm * scale_inv, 64 * 1.1920929e-7f * fabsf(p0.d1));
  if (p0.d2 <= kMinVal) return 0.f;
  // fp32 cannot resolve cost differences below ~eps * cost, which is where the last Newton iterations live.  The
  // 1-D cost is convex and p0.d1 < 0, so acceptance is decided on the derivative: |d1| < gtol is the minimiser, and a
  // point still on the descending side (d1 <= 0, alpha > 0) cannot be worse than alpha = 0 (same rule as the fp32
  // instantiation of the oracle, oracle/physics.h line_search).
  LsPoint p1 = ev(-p0.d1 / p0.d2);
  if (p0.cost < p1.cost && !(p1.d1 <= 0.f)) p1 = p0;
  if (fabsf(p1.d1) < gtol) return p1.alpha;
  int iter = 0;
  LsPoint p2 = p1;
  bool bracket = false;
  while (iter < M.ls_iterations) {
    iter++;
    p2 = p1;
    if (p1.d2 <= kMinVal) break;
    p1 = ev(p1.alpha - p1.d1 / p1.d2);
    if (fabsf(p1.d1) < gtol) return p1.alpha;
    if ((p1.d1 > 0) != (p2.d1 > 0)) { bracket = true; break; }
  }
  if (!bracket) return ((p1.d1 <= 0.f && p1.alpha > 0.f) || p1.cost < p0.cost) ? p1.alpha : 0.f;
  LsPoint lo = p1.d1 < 0 ? p1 : p2, hi = p1.d1 < 0 ? p2 : p1;
  while (iter < M.ls_iterations) {
    iter++;
    const LsPoint from = fabsf(lo.d1) < fabsf(hi.d1) ? lo : hi;
    float a = from.d2 > kMinVal ? from.alpha - from.d1 / from.d2 : 0.5f * (lo.alpha + hi.alpha);
    const float amin = fminf(lo.alpha, hi.alpha), amax = fmaxf(lo.alpha, hi.alpha);
    if (!(a > amin && a < amax)) a = 0.5f * (lo.alpha + hi.alpha);
    if (a == lo.alpha || a == hi.alpha) break;
    const LsPoint pm = ev(a);
    if (fabsf(pm.d1) < gtol) return pm.alpha;
    if (pm.d1 < 0) lo = pm; else hi = pm;
  }
  if (lo.alpha > 0.f) return lo.alpha;   // bracket closed to adjacent values: the descending end is an improvement
  return hi.cost < p0.cost ? hi.alpha : 0.f;
}

// out[dof] = sum over constraint rows of J[row][dof] * force[row], in two balanced stages (per contact, then per dof)
template <class SP>
__device__ __forceinline__ void jt_force(Ctx& c, float* out_or_null) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float *J = DF(efc_J), *force = DF(efc_force), *esgn = DF(efc_sgn);
  float* xf = DF(con_xf);
  const int *cadr = DI(con_adr), *cdim = DI(con_dim), *cnd = DI(con_nd), *cloc = DI(con_loc), *frow = MI(floss_row),
            *edof = DI(efc_dof);
  for (int w = lane; w < c.ncon * kL; w += 32) {
    const int ci = w / kL, l = w - ci * kL;
    const int a0 = cadr[ci];
    float a = 0.f;
    if (a0 >= 0 && l < cnd[ci]) {
      const int nrow = cdim[ci];   // the row count (pyramidal: 2 (condim - 1), up to 10)
      FOR_ROWS(k, nrow) a += J[(a0 + k) * kL + l] * force[a0 + k];
    }
    xf[w] = a;
  }
  __syncwarp();
  const int nf = M.nfloss, nl = c.nlim;
  for (int i = lane; i < nv; i += 32) {
    float a = 0.f;
    const int fr = frow[i];
    if (fr >= 0) a += force[fr];
    for (int q = nf; q < nf + nl; q++)
      if (edof[q] == i) a += esgn[q] * force[q];
    for (int ci = 0; ci < c.ncon; ci++) {
      const int l = cloc[ci * nv + i];
      if (l >= 0) a += xf[ci * kL + l];
    }
    out_or_null[i] = a;
  }
  __syncwarp();
}

template <class SP>
__device__ __noinline__ void jt_force_any(Ctx& c, float* out, int nv) {
  if constexpr (SP::kNV > 0) jt_force_dense<SP, SP::kNV>(c, out);
  else { if (nv == 18) jt_force_dense<SP, 18>(c, out); else jt_force<SP>(c, out); }
}

template <class SP>
__device__ __noinline__ void k_solve(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv, ne = c.nefc;
  float *qacc = DF(qacc), *qas = DF(qacc_smooth), *qws = DF(qacc_warmstart), *qfc = DF(qfrc_constraint);
  c.niter = 0;
  // (lane loops below run on ALL lanes with a clamped index and predicated stores: no divergent regions)
  if (ne == 0) {
    for (int i = lane; i < nv; i += 32) { qacc[i] = qas[i]; qfc[i] = 0; }
    __syncwarp();
    return;
  }
  PHASE_AT(c, 1, 8);
  float gauss, cost;
  if (!M.disable_warmstart) {
    // warm start (engine_forward: the better of qacc_warmstart and qacc_smooth).  The smooth point is evaluated
    // first so that, when the warm start wins (the usual case), the constraint state is already the chosen one.
    const float cs = k_total_cost<SP>(c, qas, false, &gauss);
    const float cw = k_total_cost<SP>(c, qws, true, &gauss);
    const bool warm = cw < cs;
    for (int b0 = 0; b0 < nv; b0 += 32) { const int i = min(b0 + lane, nv - 1); const float v = warm ? qws[i] : qas[i]; if (b0 + lane < nv) qacc[i] = v; }
    __syncwarp();
    cost = warm ? cw : k_total_cost<SP>(c, qacc, true, &gauss);
  } else {
    for (int i = lane; i < nv; i += 32) qacc[i] = qas[i];
    __syncwarp();
    cost = k_total_cost<SP>(c, qacc, true, &gauss);
  }
  PHASE_AT(c, 1, 4);
  const float scale_inv = CM(c).meaninertia * (float)max(1, nv);
  const float tol = fmaxf(CM(c).tolerance, kTolFloor);
  const int nsimple = M.nfloss + c.nlim;
  float *grad = DF(grad), *search = DF(search), *Mv = DF(Mv), *Ma = DF(Ma), *smooth = DF(qfrc_smooth), *Jv = DF(efc_Jv),
        *qM = DF(qM);
  float old = cost, prev_gradient = 3.0e38f, alpha = 0.f;
  int stalls = 0;
  bool qfc_current = false;
  // Helper-warp kernels: the Hessian at the current point is assembled by the helper warps while this warp forms the
  // gradient and the termination test.  The assembly reads only what the last k_total_cost(.., hess=true) and the
  // constraint rows left (qM, efc_hw, efc_hc, efc_w, efc_Jd, efc_Xd, efc_state, con_*, efc_dof, efc_drow, cdof) and
  // writes efc_hc[36 ci + 14 ..], efc_blk, dofbuf and qH, none of which J^T f, the gradient and the test touch (they
  // write qfrc_constraint and grad).  An assembly in flight when the test stops the solve is dropped: it is left
  // running while the step ends (Euler, outputs: they touch none of its arrays) and met by wide_settle before the next
  // step's kinematics, which rewrite what it reads.
  for (int iter = 0; iter <= M.iterations; iter++) {
    if constexpr (SP::kWide > 1) {
      if (iter < M.iterations) {
        hessian_cone_rows<SP>(c);
        wide_post_async<SP>(c, WIDE_HESSIAN);
        c.wide_pending = 1;
        PHASE_AT(c, 1, 5);
      }
    }
    // gradient at the current point; qfc doubles as the J^T force scratch and is the output when we stop here
    jt_force_any<SP>(c, qfc, nv);
    qfc_current = true;
    float g2 = 0, ga = 0;
    for (int b0 = 0; b0 < nv; b0 += 32) {
      const int i = min(b0 + lane, nv - 1);
      const bool on = b0 + lane < nv;
      const float a = Ma[i] - smooth[i] - qfc[i];
      if (on) grad[i] = a;
      g2 += on ? a * a : 0.f;
      const float m = fabsf(Ma[i]) + fabsf(smooth[i]) + fabsf(qfc[i]);
      ga += on ? m * m : 0.f;
    }
    const float gnorm2 = warp_sum(g2), gabs2 = warp_sum(ga);
    __syncwarp();
    if (iter > 0) {
      // fp32 termination (same rule as the fp32 oracle, oracle/physics.h solve_constraints): the gradient test has a
      // rounding floor; a cost decrease below the rounding of the cost itself is not evidence of convergence and only
      // stops the solver when a (near) full Newton step no longer shrinks the gradient
      const float improvement = (old - cost) / scale_inv, gradient = sqrtf(gnorm2) / scale_inv;
      const float gfloor = kGradFloor * 1.1920929e-7f * sqrtf(gabs2) / scale_inv;
      if (gradient < fmaxf(tol, gfloor)) break;
      const bool resolvable = fabsf(old - cost) > 16.f * 1.1920929e-7f * fabsf(cost);
      if (resolvable) { if (improvement < tol) break; stalls = 0; }
      else if (gradient > 0.5f * prev_gradient && (alpha > 0.5f || ++stalls >= 3)) break;
      prev_gradient = gradient;
    }
    PHASE_AT(c, 1, 0);
    if (iter == M.iterations) break;
    // Newton direction: assemble (or meet the helpers' assembly) + factorise the Hessian only now that another
    // iteration is taken
    PHASE(c, 4);
    if constexpr (SP::kWide > 1) wide_settle<SP>(c);
    else k_hessian<SP>(c);
    PHASE(c, 5);
    PHASE_AT(c, 1, 5);
    // fill check: only rows of contacts between two moving bodies and of tendon limits (efc_drow) can couple dofs of
    // different branches; without them H has qM's (dof, ancestor) pattern
    spd_solve<SP>(c, DF(qH), DF(hinv), search, grad, c.ndrow == 0);
    PHASE(c, 6);
    PHASE_AT(c, 1, 6);
    for (int b0 = 0; b0 < nv; b0 += 32) { const int i = min(b0 + lane, nv - 1); const float v = -search[i]; __syncwarp(); if (b0 + lane < nv) search[i] = v; }
    __syncwarp();
    float q1 = 0, q2 = 0, sn = 0;
    for (int b0 = 0; b0 < nv; b0 += 32) {
      const int i = min(b0 + lane, nv - 1);
      const bool on = b0 + lane < nv;
      const float a = m_row_dot<SP>(qM, i, search, nv);
      if (on) Mv[i] = a;
      const float si = on ? search[i] : 0.f;
      q1 += si * (Ma[i] - smooth[i]);
      q2 += 0.5f * si * a;
      sn += si * si;
    }
    for (int b0 = 0; b0 < ne; b0 += 32) {
      const int i = min(b0 + lane, ne - 1);
      const float v = j_row_dot<SP>(c, i, nsimple, search, nv);
      if (b0 + lane < ne) Jv[i] = v;
    }
    q1 = warp_sum(q1); q2 = warp_sum(q2); sn = sqrtf(warp_sum(sn));
    __syncwarp();
    PHASE_AT(c, 1, 1);
    alpha = k_line_search<SP>(c, gauss, q1, q2, sn, scale_inv);
    PHASE_AT(c, 1, 2);
    if (alpha == 0.f) break;
    for (int b0 = 0; b0 < nv; b0 += 32) { const int i = min(b0 + lane, nv - 1); const float v = qacc[i] + alpha * search[i]; __syncwarp(); if (b0 + lane < nv) qacc[i] = v; }
    __syncwarp();
    old = cost;
    cost = k_total_cost<SP>(c, qacc, true, &gauss, alpha);
    qfc_current = false;
    c.niter = iter + 1;
    PHASE_AT(c, 1, 3);
  }
  PHASE_AT(c, 1, 0);
  if (!qfc_current) jt_force_any<SP>(c, qfc, nv);
  PHASE_AT(c, 1, 0);
}

// ------------------------------------------------------------------------------------------ pipeline pieces
__device__ __forceinline__ bool k_bad(Ctx& c, const float* v, int n) {
  bool bad = false;
  for (int i = c.lane; i < n; i += 32) bad |= !(fabsf(v[i]) < kMaxVal);
  return __any_sync(kFull, bad);
}

// everything of mj_forward up to (not including) the sensor/residual callback
template <class SP>
__device__ __noinline__ void k_forward(Ctx& c) {
  PHASE(c, 7);            // everything between two forward passes (policy, residual, cost, Euler, output)
  k_kinematics<SP>(c);
  k_com_pos<SP>(c);
  k_crb<SP>(c);
  PHASE(c, 0);
  k_collision<SP>(c);
  PHASE(c, 1);
  k_make_constraint<SP>(c);
  PHASE(c, 2);
  k_com_vel<SP>(c);
  k_smooth_forces<SP>(c);
  k_reference<SP>(c);
  PHASE(c, 3);
  k_solve<SP>(c);
  PHASE(c, 4);
}

// semi-implicit Euler with implicit joint damping
template <class SP>
__device__ __noinline__ void k_euler(Ctx& c) {
  auto&& M = SP::model(c);
  const int lane = c.lane, nv = M.nv;
  const float h = CM(c).timestep;
  float *qacc = DF(qacc), *qvel = DF(qvel), *qpos = DF(qpos), *vt = DF(vtmp);
  const float* acc = qacc;
  if (M.any_damping && !M.disable_eulerdamp) {
    // (helper-warp kernels: an abandoned Hessian assembly may still be writing qH; qLD is free after join 1 until the
    // next step's k_crb)
    float *H = SP::kWide > 1 ? DF(qLD) : DF(qH), *qM = DF(qM), *smooth = DF(qfrc_smooth), *qfc = DF(qfrc_constraint);
    const float* damping = MF(dof_damping);
    MJPC_ROLL
    for (int w = lane; w < nv * nv; w += 32) {
      const int r = w / nv, s = w - r * nv;
      H[w] = qM[w] + (r == s ? h * damping[r] : 0.f);
    }
    for (int i = lane; i < nv; i += 32) vt[i] = smooth[i] + qfc[i];
    __syncwarp();
    spd_solve<SP>(c, H, DF(hinv), vt, vt, true);
    acc = vt;
  }
  for (int i = lane; i < nv; i += 32) qvel[i] += h * acc[i];
  __syncwarp();
  const int *jtype = MI(jnt_type), *jqadr = MI(jnt_qposadr), *jdadr = MI(jnt_dofadr);
  for (int j = lane; j < M.njnt; j += 32) {
    const int qa = jqadr[j], da = jdadr[j];
    const int t = jtype[j];
    if (t == JNT_FREE) {
      for (int q = 0; q < 3; q++) qpos[qa + q] += h * qvel[da + q];
      quat_integrate(qpos + qa + 3, qvel + da + 3, h);
    } else if (t == JNT_BALL) {
      quat_integrate(qpos + qa, qvel + da, h);
    } else {
      qpos[qa] += h * qvel[da];
    }
  }
  c.time += h;
  __syncwarp();
}

}  // namespace mjpc_dev
