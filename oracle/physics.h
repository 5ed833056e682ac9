// TEST INFRASTRUCTURE - CPU oracle (see oracle/model.h header).  "parity unpinned" for contact physics.
//
// physics.h: scalar-templated restatement of the forward-dynamics pipeline MJPC reaches through
// mj_step / mj_forward (call sites mjpc/trajectory.cc:158,198,257,297).  MuJoCo is an external,
// un-vendored dependency (CMakeLists.txt:55-58), so this follows its *published* pipeline
// (SURVEY.md Appendix C): kinematics, com-frame spatial quantities, composite rigid body inertia,
// collision (primitive pairs), soft-constraint assembly (solref/solimp impedance, diagApprox from
// invweight0, elliptic cones with impratio), RNE bias forces, actuation, primal Newton solver with
// exact line search, semi-implicit Euler with implicit joint damping.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <limits>
#include <vector>

#include <atomic>

#include "counted.h"
#include "model.h"

namespace oracle {

// diagnostics: histogram of Newton iterations per solve (all threads), read through oracle_solver_hist()
inline std::atomic<long>* solver_hist() { static std::atomic<long> h[64]; return h; }

template <class T> constexpr T kMinVal() { return (T)1e-15; }
// Solver tolerance floor: opt.tolerance (1e-8) is below what fp32 cost differences can resolve, so reduced
// precision terminates on max(opt.tolerance, 1e-6); inactive in fp64. Measured effect on returns: 1e-8 relative.
template <class T> constexpr T kTolFloor() { return sizeof(T) == 4 ? (T)1e-6 : (T)0; }
// Capsule-capsule parallel test: det = |a1|^2 |a2|^2 - (a1.a2)^2 = sin^2(angle) of the two unit axes.  In fp32 the
// rounding residual of det for exactly parallel axes is ~1e-7, far above mjMINVAL, and the nearest-point solve then
// divides rounding noise by rounding noise; reduced precision therefore treats det < 16 eps |a1|^2 |a2|^2 (angles
// below 1.4e-3 rad) as parallel, the same rule as the device.  fp64 keeps MuJoCo's mjMINVAL.
template <class T> inline bool capsules_parallel(T det, T ma, T mc) {
  return sizeof(T) == 4 ? mm::fabs(det) < (T)16 * mm::eps<T>() * ma * mc : mm::fabs(det) < kMinVal<T>();
}
constexpr double kMaxVal = 1e10;      // mjMAXVAL
constexpr double kMinImp = 0.0001, kMaxImp = 0.9999, kMinMu = 1e-5;
constexpr int kMaxConDim = 6;
// reduced-precision solver: the gradient cannot be driven below kGradFloor * eps * |terms| (see solve_constraints)
constexpr double kGradFloor = 16;

enum { CNSTR_FRICTION_DOF = 0, CNSTR_LIMIT_JOINT, CNSTR_CONTACT_FRICTIONLESS, CNSTR_CONTACT_ELLIPTIC, CNSTR_LIMIT_TENDON,
       CNSTR_CONTACT_PYRAMIDAL };
// one-sided quadratic rows: cost 0.5 D jar^2 when jar < 0 (limits, frictionless contacts, pyramid edges)
inline bool cnstr_inequality(int type) {
  return type == CNSTR_LIMIT_JOINT || type == CNSTR_CONTACT_FRICTIONLESS || type == CNSTR_LIMIT_TENDON ||
         type == CNSTR_CONTACT_PYRAMIDAL;
}
enum { STATE_SATISFIED = 0, STATE_QUADRATIC, STATE_LINEARNEG, STATE_LINEARPOS, STATE_CONE };

// ------------------------------------------------------------------------------------------ small math
template <class T> inline T dot3(const T* a, const T* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
template <class T> inline void cross3(T* r, const T* a, const T* b) {
  T x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
template <class T> inline T norm3(const T* a) { return mm::sqrt(dot3(a, a)); }
template <class T> inline T normalize3(T* a) {
  T n = norm3(a);
  if (n < kMinVal<T>()) { a[0] = 1; a[1] = 0; a[2] = 0; return n; }
  a[0] /= n; a[1] /= n; a[2] /= n;
  return n;
}
template <class T> inline void quat_mul(T* r, const T* a, const T* b) {
  T w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  T x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  T y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  T z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
template <class T> inline void quat_normalize(T* q) {
  T n = mm::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < kMinVal<T>()) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
template <class T> inline void quat2mat(T* m, const T* q) {
  T w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
template <class T> inline void rot_vec(T* r, const T* m, const T* v) {  // r = M v (row-major 3x3)
  T x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2],
    z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
template <class T> inline void rot_vec_T(T* r, const T* m, const T* v) {  // r = M^T v
  T x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2],
    z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
template <class T> inline void axis_angle_quat(T* q, const T* axis, T angle) {
  T s = mm::sin(angle * (T)0.5);
  q[0] = mm::cos(angle * (T)0.5); q[1] = axis[0] * s; q[2] = axis[1] * s; q[3] = axis[2] * s;
}
// q <- q * exp(w*h/2): integrate body-frame angular velocity.  As mju_quatIntegrate, the result is the normalised q
// (the identity for an all-zero q) times the rotation, a unit quaternion also when w = 0.
template <class T> inline void quat_integrate(T* q, const T* w, T h) {
  T ax[3] = {w[0], w[1], w[2]};
  T n = norm3(ax);
  if (n < kMinVal<T>()) { quat_normalize(q); return; }
  ax[0] /= n; ax[1] /= n; ax[2] /= n;
  T dq[4], r[4];
  axis_angle_quat(dq, ax, n * h);
  if (mm::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]) < kMinVal<T>()) { q[0] = 1; q[1] = q[2] = q[3] = 0; }
  quat_mul(r, q, dq);
  quat_normalize(r);
  q[0] = r[0]; q[1] = r[1]; q[2] = r[2]; q[3] = r[3];
}
// spatial helpers; motion vector = [ang(3); lin(3)], force vector = [torque(3); force(3)]
template <class T> inline void cross_motion(T* r, const T* v, const T* m) {
  T a[3], b[3], c[3];
  cross3(a, v, m); cross3(b, v, m + 3); cross3(c, v + 3, m);
  for (int k = 0; k < 3; k++) { r[k] = a[k]; r[3 + k] = b[k] + c[k]; }
}
template <class T> inline void cross_force(T* r, const T* v, const T* f) {
  T a[3], b[3], c[3];
  cross3(a, v, f); cross3(b, v + 3, f + 3); cross3(c, v, f + 3);
  for (int k = 0; k < 3; k++) { r[k] = a[k] + b[k]; r[3 + k] = c[k]; }
}
// inertia I = {Ixx,Iyy,Izz,Ixy,Ixz,Iyz, m*ox,m*oy,m*oz, m} about the frame origin
template <class T> inline void mul_inert_vec(T* r, const T* I, const T* v) {
  const T* w = v; const T* l = v + 3; const T* mo = I + 6;
  T a[3], b[3];
  cross3(a, mo, l); cross3(b, mo, w);
  r[0] = I[0] * w[0] + I[3] * w[1] + I[4] * w[2] + a[0];
  r[1] = I[3] * w[0] + I[1] * w[1] + I[5] * w[2] + a[1];
  r[2] = I[4] * w[0] + I[5] * w[1] + I[2] * w[2] + a[2];
  r[3] = I[9] * l[0] - b[0]; r[4] = I[9] * l[1] - b[1]; r[5] = I[9] * l[2] - b[2];
}
// orthonormal frame from unit normal (rows: normal, t1, t2)
template <class T> inline void make_frame(T* f) {
  T* x = f; T* y = f + 3; T* z = f + 6;
  if (x[1] > (T)-0.5 && x[1] < (T)0.5) { y[0] = 0; y[1] = 1; y[2] = 0; } else { y[0] = 0; y[1] = 0; y[2] = 1; }
  T d = dot3(x, y);
  for (int k = 0; k < 3; k++) y[k] -= d * x[k];
  normalize3(y);
  cross3(z, x, y);
}
// dense in-place Cholesky (lower) of n x n row-major; returns min pivot. A = L L^T
template <class T> inline T chol_factor(T* A, int n) {
  T minp = mm::big<T>();
  for (int j = 0; j < n; j++) {
    T s = A[j * n + j];
    for (int k = 0; k < j; k++) s -= A[j * n + k] * A[j * n + k];
    minp = mm::min(minp, s);
    if (s < kMinVal<T>()) s = kMinVal<T>();
    T l = mm::sqrt(s);
    A[j * n + j] = l;
    for (int i = j + 1; i < n; i++) {
      T t = A[i * n + j];
      for (int k = 0; k < j; k++) t -= A[i * n + k] * A[j * n + k];
      A[i * n + j] = t / l;
    }
  }
  return minp;
}
template <class T> inline void chol_solve(T* x, const T* L, const T* b, int n) {
  for (int i = 0; i < n; i++) {
    T s = b[i];
    for (int k = 0; k < i; k++) s -= L[i * n + k] * x[k];
    x[i] = s / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    T s = x[i];
    for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k];
    x[i] = s / L[i * n + i];
  }
}

// ------------------------------------------------------------------------------------------ data
template <class T>
struct Contact {
  T dist, pos[3], frame[9], includemargin, friction[5], solref[2], solimp[5], mu;
  int dim, geom1, geom2, efc_address;
};

template <class T>
struct Data {
  // state
  std::vector<T> qpos, qvel, ctrl, mocap_pos, mocap_quat, userdata, qacc_warmstart;
  T time = 0;
  // position-dependent
  std::vector<T> xpos, xquat, xmat, xipos, ximat, xanchor, xaxis, geom_xpos, geom_xmat, site_xpos, site_xmat,
      subtree_com, cinert, crb, cdof, qM, qLD;
  // velocity-dependent
  std::vector<T> cvel, cdof_dot, subtree_linvel, qfrc_passive, qfrc_bias;
  // forces / accelerations
  std::vector<T> actuator_force, qfrc_actuator, qfrc_smooth, qacc_smooth, qacc, qfrc_constraint;
  std::vector<T> xfrc_applied;   // [nbody][force 3, torque 3] world frame, applied at the body's centre of mass
  bool xfrc_active = false;      // NoisyRollout (trajectory.cc:147-155); false -> the array is ignored
  // constraints
  std::vector<Contact<T>> contact;
  int ncon = 0, nefc = 0, solver_niter = 0;
  std::vector<T> efc_J, efc_pos, efc_margin, efc_diagApprox, efc_R, efc_D, efc_KBIP, efc_aref, efc_vel, efc_force,
      efc_frictionloss;
  std::vector<int> efc_type, efc_id, efc_state;
  // task
  std::vector<T> residual;
  bool warning = false;
  int maxcon = 32, maxefc = 96;

  explicit Data(const Model<T>& m) {
    qpos.assign(m.qpos0.begin(), m.qpos0.end());
    qvel.assign(m.nv, 0); ctrl.assign(m.nu, 0); qacc_warmstart.assign(m.nv, 0);
    mocap_pos.assign(3 * m.nmocap, 0); mocap_quat.assign(4 * m.nmocap, 0); userdata.assign(m.nuserdata, 0);
    for (int b = 0; b < m.nbody; b++) {
      int k = m.body_mocapid[b];
      if (k >= 0) {
        for (int c = 0; c < 3; c++) mocap_pos[3 * k + c] = m.body_pos[3 * b + c];
        for (int c = 0; c < 4; c++) mocap_quat[4 * k + c] = m.body_quat[4 * b + c];
      }
    }
    xpos.assign(3 * m.nbody, 0); xquat.assign(4 * m.nbody, 0); xmat.assign(9 * m.nbody, 0);
    xipos.assign(3 * m.nbody, 0); ximat.assign(9 * m.nbody, 0); xanchor.assign(3 * m.njnt, 0);
    xaxis.assign(3 * m.njnt, 0); geom_xpos.assign(3 * m.ngeom, 0); geom_xmat.assign(9 * m.ngeom, 0);
    site_xpos.assign(3 * m.nsite, 0); site_xmat.assign(9 * m.nsite, 0); subtree_com.assign(3 * m.nbody, 0);
    cinert.assign(10 * m.nbody, 0); crb.assign(10 * m.nbody, 0); cdof.assign(6 * m.nv, 0);
    qM.assign(m.nv * m.nv, 0); qLD.assign(m.nv * m.nv, 0);
    cvel.assign(6 * m.nbody, 0); cdof_dot.assign(6 * m.nv, 0); subtree_linvel.assign(3 * m.nbody, 0);
    qfrc_passive.assign(m.nv, 0); qfrc_bias.assign(m.nv, 0); actuator_force.assign(m.nu, 0);
    qfrc_actuator.assign(m.nv, 0); qfrc_smooth.assign(m.nv, 0); qacc_smooth.assign(m.nv, 0);
    qacc.assign(m.nv, 0); qfrc_constraint.assign(m.nv, 0); xfrc_applied.assign(6 * m.nbody, 0);
    residual.assign(mm::max(m.num_residual, 1), 0);
  }
};

// ------------------------------------------------------------------------------------------ position stage
template <class T>
void kinematics(const Model<T>& m, Data<T>& d) {
  d.xquat[0] = 1; d.xmat[0] = d.xmat[4] = d.xmat[8] = 1;
  for (int b = 1; b < m.nbody; b++) {
    int p = m.body_parentid[b];
    T pos[3], quat[4];
    if (m.body_mocapid[b] >= 0) {
      int k = m.body_mocapid[b];
      for (int c = 0; c < 3; c++) pos[c] = d.mocap_pos[3 * k + c];
      for (int c = 0; c < 4; c++) quat[c] = d.mocap_quat[4 * k + c];
      quat_normalize(quat);
    } else {
      rot_vec(pos, &d.xmat[9 * p], &m.body_pos[3 * b]);
      for (int c = 0; c < 3; c++) pos[c] += d.xpos[3 * p + c];
      quat_mul(quat, &d.xquat[4 * p], &m.body_quat[4 * b]);
    }
    for (int j = m.body_jntadr[b]; j < m.body_jntadr[b] + m.body_jntnum[b]; j++) {
      int qa = m.jnt_qposadr[j];
      int t = m.jnt_type[j];
      if (t == JNT_FREE) {
        for (int c = 0; c < 3; c++) pos[c] = d.qpos[qa + c];
        for (int c = 0; c < 4; c++) quat[c] = d.qpos[qa + 3 + c];
        quat_normalize(quat);
        for (int c = 0; c < 3; c++) { d.xanchor[3 * j + c] = pos[c]; d.xaxis[3 * j + c] = (c == 2); }
        continue;
      }
      T R[9];
      quat2mat(R, quat);
      T anchor[3], axis[3];
      rot_vec(anchor, R, &m.jnt_pos[3 * j]);
      for (int c = 0; c < 3; c++) anchor[c] += pos[c];
      rot_vec(axis, R, &m.jnt_axis[3 * j]);
      for (int c = 0; c < 3; c++) { d.xanchor[3 * j + c] = anchor[c]; d.xaxis[3 * j + c] = axis[c]; }
      if (t == JNT_SLIDE) {
        T q = d.qpos[qa] - m.qpos0[qa];
        for (int c = 0; c < 3; c++) pos[c] += axis[c] * q;
      } else {
        T ql[4], qn[4];
        if (t == JNT_HINGE) {
          axis_angle_quat(ql, &m.jnt_axis[3 * j], d.qpos[qa] - m.qpos0[qa]);
        } else {
          for (int c = 0; c < 4; c++) ql[c] = d.qpos[qa + c];
          quat_normalize(ql);
        }
        quat_mul(qn, quat, ql);
        for (int c = 0; c < 4; c++) quat[c] = qn[c];
        quat2mat(R, quat);
        T off[3];
        rot_vec(off, R, &m.jnt_pos[3 * j]);
        for (int c = 0; c < 3; c++) pos[c] = anchor[c] - off[c];
      }
    }
    quat_normalize(quat);
    for (int c = 0; c < 3; c++) d.xpos[3 * b + c] = pos[c];
    for (int c = 0; c < 4; c++) d.xquat[4 * b + c] = quat[c];
    quat2mat(&d.xmat[9 * b], quat);
    T ip[3], iq[4];
    rot_vec(ip, &d.xmat[9 * b], &m.body_ipos[3 * b]);
    for (int c = 0; c < 3; c++) d.xipos[3 * b + c] = pos[c] + ip[c];
    quat_mul(iq, quat, &m.body_iquat[4 * b]);
    quat2mat(&d.ximat[9 * b], iq);
  }
  for (int g = 0; g < m.ngeom; g++) {
    int b = m.geom_bodyid[g];
    T p[3], q[4];
    rot_vec(p, &d.xmat[9 * b], &m.geom_pos[3 * g]);
    for (int c = 0; c < 3; c++) d.geom_xpos[3 * g + c] = d.xpos[3 * b + c] + p[c];
    quat_mul(q, &d.xquat[4 * b], &m.geom_quat[4 * g]);
    quat2mat(&d.geom_xmat[9 * g], q);
  }
  for (int s = 0; s < m.nsite; s++) {
    int b = m.site_bodyid[s];
    T p[3], q[4];
    rot_vec(p, &d.xmat[9 * b], &m.site_pos[3 * s]);
    for (int c = 0; c < 3; c++) d.site_xpos[3 * s + c] = d.xpos[3 * b + c] + p[c];
    quat_mul(q, &d.xquat[4 * b], &m.site_quat[4 * s]);
    quat2mat(&d.site_xmat[9 * s], q);
  }
}

template <class T>
void com_pos(const Model<T>& m, Data<T>& d) {
  for (int b = 0; b < m.nbody; b++)
    for (int c = 0; c < 3; c++) d.subtree_com[3 * b + c] = m.body_mass[b] * d.xipos[3 * b + c];
  for (int b = m.nbody - 1; b > 0; b--)
    for (int c = 0; c < 3; c++) d.subtree_com[3 * m.body_parentid[b] + c] += d.subtree_com[3 * b + c];
  for (int b = 0; b < m.nbody; b++) {
    if (m.body_subtreemass[b] < kMinVal<T>()) {
      for (int c = 0; c < 3; c++) d.subtree_com[3 * b + c] = d.xipos[3 * b + c];
    } else {
      for (int c = 0; c < 3; c++) d.subtree_com[3 * b + c] /= m.body_subtreemass[b];
    }
  }
  // body inertia about the root-subtree com, world orientation
  for (int b = 1; b < m.nbody; b++) {
    const T* R = &d.ximat[9 * b];
    const T* I = &m.body_inertia[3 * b];
    T mass = m.body_mass[b];
    T o[3];
    for (int c = 0; c < 3; c++) o[c] = d.xipos[3 * b + c] - d.subtree_com[3 * m.body_rootid[b] + c];
    T W[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        W[3 * i + j] = R[3 * i] * I[0] * R[3 * j] + R[3 * i + 1] * I[1] * R[3 * j + 1] + R[3 * i + 2] * I[2] * R[3 * j + 2];
    T oo = dot3(o, o);
    T* ci = &d.cinert[10 * b];
    ci[0] = W[0] + mass * (oo - o[0] * o[0]); ci[1] = W[4] + mass * (oo - o[1] * o[1]);
    ci[2] = W[8] + mass * (oo - o[2] * o[2]);
    ci[3] = W[1] - mass * o[0] * o[1]; ci[4] = W[2] - mass * o[0] * o[2]; ci[5] = W[5] - mass * o[1] * o[2];
    ci[6] = mass * o[0]; ci[7] = mass * o[1]; ci[8] = mass * o[2]; ci[9] = mass;
  }
  // motion dofs about the root-subtree com
  for (int j = 0; j < m.njnt; j++) {
    int b = m.jnt_bodyid[j];
    int da = m.jnt_dofadr[j];
    T off[3];
    for (int c = 0; c < 3; c++) off[c] = d.subtree_com[3 * m.body_rootid[b] + c] - d.xanchor[3 * j + c];
    const T* ax = &d.xaxis[3 * j];
    switch (m.jnt_type[j]) {
      case JNT_FREE:
        for (int k = 0; k < 3; k++) {
          T* cd = &d.cdof[6 * (da + k)];
          for (int c = 0; c < 6; c++) cd[c] = 0;
          cd[3 + k] = 1;
        }
        da += 3;
        [[fallthrough]];
      case JNT_BALL:
        for (int k = 0; k < 3; k++) {
          T* cd = &d.cdof[6 * (da + k)];
          T col[3] = {d.xmat[9 * b + k], d.xmat[9 * b + 3 + k], d.xmat[9 * b + 6 + k]};
          for (int c = 0; c < 3; c++) cd[c] = col[c];
          cross3(cd + 3, col, off);
        }
        break;
      case JNT_SLIDE: {
        T* cd = &d.cdof[6 * da];
        for (int c = 0; c < 3; c++) { cd[c] = 0; cd[3 + c] = ax[c]; }
        break;
      }
      default: {
        T* cd = &d.cdof[6 * da];
        for (int c = 0; c < 3; c++) cd[c] = ax[c];
        cross3(cd + 3, ax, off);
      }
    }
  }
}

template <class T>
void crb(const Model<T>& m, Data<T>& d) {
  int nv = m.nv;
  d.crb = d.cinert;
  for (int b = m.nbody - 1; b > 0; b--) {
    int p = m.body_parentid[b];
    if (p > 0)
      for (int c = 0; c < 10; c++) d.crb[10 * p + c] += d.crb[10 * b + c];
  }
  std::fill(d.qM.begin(), d.qM.end(), (T)0);
  for (int i = 0; i < nv; i++) {
    T buf[6];
    mul_inert_vec(buf, &d.crb[10 * m.dof_bodyid[i]], &d.cdof[6 * i]);
    T s = 0;
    for (int c = 0; c < 6; c++) s += d.cdof[6 * i + c] * buf[c];
    d.qM[i * nv + i] = s + m.dof_armature[i];
    for (int j = m.dof_parentid[i]; j >= 0; j = m.dof_parentid[j]) {
      T t = 0;
      for (int c = 0; c < 6; c++) t += d.cdof[6 * j + c] * buf[c];
      d.qM[i * nv + j] = d.qM[j * nv + i] = t;
    }
  }
  d.qLD = d.qM;
  chol_factor(d.qLD.data(), nv);
}

// ------------------------------------------------------------------------------------------ collision
template <class T>
struct RawContact { T dist, pos[3], normal[3]; };

template <class T>
int collide_plane_sphere(RawContact<T>* out, const T* pp, const T* pm, const T* sp, T r) {
  T n[3] = {pm[2], pm[5], pm[8]};
  T diff[3] = {sp[0] - pp[0], sp[1] - pp[1], sp[2] - pp[2]};
  T dist = dot3(diff, n) - r;
  out->dist = dist;
  for (int c = 0; c < 3; c++) { out->normal[c] = n[c]; out->pos[c] = sp[c] - n[c] * (r + dist * (T)0.5); }
  return 1;
}
template <class T>
int collide_plane_capsule(RawContact<T>* out, const T* pp, const T* pm, const T* cp, const T* cm, const T* size) {
  T axis[3] = {cm[2], cm[5], cm[8]};
  int n = 0;
  for (int s = -1; s <= 1; s += 2) {
    T e[3];
    for (int c = 0; c < 3; c++) e[c] = cp[c] + (T)s * size[1] * axis[c];
    n += collide_plane_sphere(out + n, pp, pm, e, size[0]);
  }
  return n;
}
template <class T>
int collide_plane_box(RawContact<T>* out, const T* pp, const T* pm, const T* bp, const T* bm, const T* size, T margin) {
  T nrm[3] = {pm[2], pm[5], pm[8]};
  int n = 0;
  for (int k = 0; k < 8 && n < 4; k++) {
    T loc[3] = {(k & 1 ? size[0] : -size[0]), (k & 2 ? size[1] : -size[1]), (k & 4 ? size[2] : -size[2])};
    T w[3];
    rot_vec(w, bm, loc);
    T corner[3], diff[3];
    for (int c = 0; c < 3; c++) { corner[c] = bp[c] + w[c]; diff[c] = corner[c] - pp[c]; }
    T dist = dot3(diff, nrm);
    if (dist > margin) continue;
    out[n].dist = dist;
    for (int c = 0; c < 3; c++) { out[n].normal[c] = nrm[c]; out[n].pos[c] = corner[c] - nrm[c] * dist * (T)0.5; }
    n++;
  }
  return n;
}
// plane-cylinder: deepest point of each end disk + two more points on the nearer disk at +-120 degrees
template <class T>
int collide_plane_cylinder(RawContact<T>* out, const T* pp, const T* pm, const T* cp, const T* cm, const T* size,
                           T margin) {
  T nrm[3] = {pm[2], pm[5], pm[8]};
  T axis[3] = {cm[2], cm[5], cm[8]};
  T r = size[0], h = size[1];
  T prj = dot3(axis, nrm);
  if (prj > 0) { for (int c = 0; c < 3; c++) axis[c] = -axis[c]; prj = -prj; }  // axis now points toward the plane
  // in-disk direction of steepest descent toward the plane
  T vec[3];
  for (int c = 0; c < 3; c++) vec[c] = -nrm[c] + axis[c] * prj;
  if (sizeof(T) == 4) {
    // reduced precision: vec is a difference of unit vectors of length sin(tilt); its rounding residual along the
    // axis (~eps) is not small against that length within ~1e-3 rad of the normal, and after scaling to r it moves
    // the rim points off the rim plane (0.4 mm at 1e-5 rad, r = 0.08).  Remove the axial part (same rule as the device).
    const T va = dot3(vec, axis);
    for (int c = 0; c < 3; c++) vec[c] -= axis[c] * va;
  }
  T len = norm3(vec);
  if (len < (T)1e-6) { vec[0] = cm[0]; vec[1] = cm[3]; vec[2] = cm[6]; len = 1; }  // axis parallel to normal
  for (int c = 0; c < 3; c++) vec[c] *= r / len;
  T side[3];
  cross3(side, vec, axis);
  T diff[3] = {cp[0] - pp[0], cp[1] - pp[1], cp[2] - pp[2]};
  T dist0 = dot3(diff, nrm);
  int n = 0;
  T cand[4][3];
  for (int c = 0; c < 3; c++) {
    cand[0][c] = axis[c] * h + vec[c];
    cand[1][c] = -axis[c] * h + vec[c];
    cand[2][c] = axis[c] * h - vec[c] * (T)0.5 + side[c] * (T)0.8660254037844386;
    cand[3][c] = axis[c] * h - vec[c] * (T)0.5 - side[c] * (T)0.8660254037844386;
  }
  for (int k = 0; k < 4; k++) {
    T dist = dist0 + dot3(cand[k], nrm);
    if (dist > margin) continue;
    out[n].dist = dist;
    for (int c = 0; c < 3; c++) { out[n].normal[c] = nrm[c]; out[n].pos[c] = cp[c] + cand[k][c] - nrm[c] * dist * (T)0.5; }
    n++;
  }
  return n;
}
template <class T>
int collide_sphere_sphere(RawContact<T>* out, const T* p1, T r1, const T* p2, T r2) {
  T dv[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  T len = norm3(dv);
  T n[3] = {1, 0, 0};
  if (len >= kMinVal<T>()) { n[0] = dv[0] / len; n[1] = dv[1] / len; n[2] = dv[2] / len; }
  T dist = len - r1 - r2;
  out->dist = dist;
  for (int c = 0; c < 3; c++) { out->normal[c] = n[c]; out->pos[c] = p1[c] + n[c] * (r1 + dist * (T)0.5); }
  return 1;
}
template <class T>
int collide_sphere_capsule(RawContact<T>* out, const T* sp, T sr, const T* cp, const T* cm, const T* csize) {
  T axis[3] = {cm[2], cm[5], cm[8]};
  T dv[3] = {sp[0] - cp[0], sp[1] - cp[1], sp[2] - cp[2]};
  T x = mm::max(-csize[1], mm::min(csize[1], dot3(dv, axis)));
  T q[3] = {cp[0] + axis[0] * x, cp[1] + axis[1] * x, cp[2] + axis[2] * x};
  return collide_sphere_sphere(out, sp, sr, q, csize[0]);
}
// [EXT] mjc_CapsuleCapsule restated: nearest points of the two axis segments (2x2 system, clamped), then a sphere test
// there; (nearly) parallel axes (capsules_parallel) test the segment ends instead and may return two contacts.  Only contacts with
// dist <= margin are returned (as mjraw_SphereSphere does).
template <class T>
int collide_capsule_capsule(RawContact<T>* out, const T* p1, const T* m1, const T* s1, const T* p2, const T* m2, const T* s2,
                            T margin) {
  const T a1[3] = {m1[2], m1[5], m1[8]}, a2[3] = {m2[2], m2[5], m2[8]};
  const T dif[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
  const T ma = dot3(a1, a1), mb = -dot3(a1, a2), mc = dot3(a2, a2), u = -dot3(a1, dif), v = dot3(a2, dif);
  const T det = ma * mc - mb * mb;
  const T r1 = s1[0], l1 = s1[1], r2 = s2[0], l2 = s2[1];
  auto clampT = [](T x, T lim) { return mm::max(-lim, mm::min(lim, x)); };
  auto sphere = [&](RawContact<T>* o, T x1, T x2) {
    T v1[3], v2[3];
    for (int c = 0; c < 3; c++) { v1[c] = p1[c] + a1[c] * x1; v2[c] = p2[c] + a2[c] * x2; }
    collide_sphere_sphere(o, v1, r1, v2, r2);
    return o->dist <= margin ? 1 : 0;
  };
  if (!capsules_parallel(det, ma, mc)) {
    T x1 = (mc * u - mb * v) / det, x2 = (ma * v - mb * u) / det;
    if (x1 > l1) { x1 = l1; x2 = (v - mb * l1) / mc; }
    else if (x1 < -l1) { x1 = -l1; x2 = (v + mb * l1) / mc; }
    if (x2 > l2) { x2 = l2; x1 = clampT((u - mb * l2) / ma, l1); }
    else if (x2 < -l2) { x2 = -l2; x1 = clampT((u + mb * l2) / ma, l1); }
    return sphere(out, x1, x2);
  }
  int n = sphere(out, l1, clampT((v - mb * l1) / mc, l2));
  n += sphere(out + n, -l1, clampT((v + mb * l1) / mc, l2));
  if (n >= 2) return n;
  n += sphere(out + n, clampT((u - mb * l2) / ma, l1), l2);
  if (n >= 2) return n;
  n += sphere(out + n, clampT((u + mb * l2) / ma, l1), -l2);
  return n;
}
template <class T>
int collide_sphere_box(RawContact<T>* out, const T* sp, T sr, const T* bp, const T* bm, const T* bs) {
  T dv[3] = {sp[0] - bp[0], sp[1] - bp[1], sp[2] - bp[2]};
  T loc[3], cl[3];
  rot_vec_T(loc, bm, dv);
  bool inside = true;
  for (int c = 0; c < 3; c++) {
    cl[c] = mm::max(-bs[c], mm::min(bs[c], loc[c]));
    if (cl[c] != loc[c]) inside = false;
  }
  T nl[3], dist, pl[3];
  if (!inside) {
    T dd[3] = {cl[0] - loc[0], cl[1] - loc[1], cl[2] - loc[2]};  // sphere centre -> closest box point
    T len = norm3(dd);
    for (int c = 0; c < 3; c++) nl[c] = dd[c] / len;
    dist = len - sr;
    for (int c = 0; c < 3; c++) pl[c] = cl[c] - nl[c] * dist * (T)0.5;
  } else {
    // centre inside the box: push out through the nearest face
    int k = 0; T best = bs[0] - mm::fabs(loc[0]);
    for (int c = 1; c < 3; c++) { T g = bs[c] - mm::fabs(loc[c]); if (g < best) { best = g; k = c; } }
    T sgn = loc[k] >= 0 ? (T)1 : (T)-1;
    nl[0] = nl[1] = nl[2] = 0; nl[k] = -sgn;
    dist = -best - sr;
    for (int c = 0; c < 3; c++) pl[c] = loc[c];
    pl[k] = (T)0.5 * (sgn * bs[k] + loc[k] - sgn * sr);  // midway between box face and deepest sphere point
  }
  T nw[3], pw[3];
  rot_vec(nw, bm, nl);
  rot_vec(pw, bm, pl);
  out->dist = dist;
  for (int c = 0; c < 3; c++) { out->normal[c] = nw[c]; out->pos[c] = bp[c] + pw[c]; }
  return 1;
}

template <class T>
void collision(const Model<T>& m, Data<T>& d) {
  d.contact.clear();
  d.ncon = 0;
  if (m.disable_contact) return;
  for (int p = 0; p < m.npair; p++) {
    int g1 = m.pair_geom1[p], g2 = m.pair_geom2[p];
    int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
    T margin = mm::max(m.geom_margin[g1], m.geom_margin[g2]);
    T gap = mm::max(m.geom_gap[g1], m.geom_gap[g2]);
    const T* p1 = &d.geom_xpos[3 * g1]; const T* p2 = &d.geom_xpos[3 * g2];
    const T* m1 = &d.geom_xmat[9 * g1]; const T* m2 = &d.geom_xmat[9 * g2];
    const T* s1 = &m.geom_size[3 * g1]; const T* s2 = &m.geom_size[3 * g2];
    // bounding-sphere filter
    if (t1 == GEOM_PLANE) {
      T n[3] = {m1[2], m1[5], m1[8]};
      T dv[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
      if (dot3(dv, n) > m.geom_rbound[g2] + margin) continue;
    } else {
      T dv[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
      T bound = m.geom_rbound[g1] + m.geom_rbound[g2] + margin;
      if (dot3(dv, dv) > bound * bound) continue;
    }
    RawContact<T> raw[4];
    int n = 0;
    if (t1 == GEOM_PLANE && t2 == GEOM_SPHERE) n = collide_plane_sphere(raw, p1, m1, p2, s2[0]);
    else if (t1 == GEOM_PLANE && t2 == GEOM_CAPSULE) n = collide_plane_capsule(raw, p1, m1, p2, m2, s2);
    else if (t1 == GEOM_PLANE && t2 == GEOM_BOX) n = collide_plane_box(raw, p1, m1, p2, m2, s2, margin);
    else if (t1 == GEOM_PLANE && t2 == GEOM_CYLINDER) n = collide_plane_cylinder(raw, p1, m1, p2, m2, s2, margin);
    else if (t1 == GEOM_SPHERE && t2 == GEOM_SPHERE) n = collide_sphere_sphere(raw, p1, s1[0], p2, s2[0]);
    else if (t1 == GEOM_SPHERE && t2 == GEOM_CAPSULE) n = collide_sphere_capsule(raw, p1, s1[0], p2, m2, s2);
    else if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) n = collide_sphere_box(raw, p1, s1[0], p2, m2, s2);
    else if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) n = collide_capsule_capsule(raw, p1, m1, s1, p2, m2, s2, margin);
    for (int k = 0; k < n; k++) {
      if (!(raw[k].dist < margin)) continue;
      // capacity: MuJoCo raises mjWARN_CONTACTFULL, which the rollout turns into failure (trajectory.cc:169-173)
      if ((int)d.contact.size() >= d.maxcon) { d.warning = true; continue; }
      Contact<T> c;
      c.dist = raw[k].dist;
      for (int a = 0; a < 3; a++) { c.pos[a] = raw[k].pos[a]; c.frame[a] = raw[k].normal[a]; }
      make_frame(c.frame);
      c.includemargin = margin - gap;
      c.geom1 = g1; c.geom2 = g2;
      // parameter mixing
      const T *f1 = &m.geom_friction[3 * g1], *f2 = &m.geom_friction[3 * g2];
      T fr[3];
      if (m.geom_priority[g1] != m.geom_priority[g2]) {
        int gp = m.geom_priority[g1] > m.geom_priority[g2] ? g1 : g2;
        c.dim = m.geom_condim[gp];
        for (int a = 0; a < 2; a++) c.solref[a] = m.geom_solref[2 * gp + a];
        for (int a = 0; a < 5; a++) c.solimp[a] = m.geom_solimp[5 * gp + a];
        for (int a = 0; a < 3; a++) fr[a] = m.geom_friction[3 * gp + a];
      } else {
        c.dim = mm::max(m.geom_condim[g1], m.geom_condim[g2]);
        T w1 = m.geom_solmix[g1], w2 = m.geom_solmix[g2], mix;
        if (w1 >= kMinVal<T>() && w2 >= kMinVal<T>()) mix = w1 / (w1 + w2);
        else if (w1 < kMinVal<T>() && w2 < kMinVal<T>()) mix = (T)0.5;
        else mix = w1 < kMinVal<T>() ? (T)0 : (T)1;
        const T *r1 = &m.geom_solref[2 * g1], *r2 = &m.geom_solref[2 * g2];
        if (r1[0] > 0 && r2[0] > 0) {
          for (int a = 0; a < 2; a++) c.solref[a] = mix * r1[a] + (1 - mix) * r2[a];
        } else {
          for (int a = 0; a < 2; a++) c.solref[a] = mm::min(r1[a], r2[a]);
        }
        for (int a = 0; a < 5; a++) c.solimp[a] = mix * m.geom_solimp[5 * g1 + a] + (1 - mix) * m.geom_solimp[5 * g2 + a];
        for (int a = 0; a < 3; a++) fr[a] = mm::max(f1[a], f2[a]);
      }
      for (int a = 0; a < 3; a++) fr[a] = mm::max(fr[a], (T)kMinMu);
      c.friction[0] = c.friction[1] = fr[0]; c.friction[2] = fr[1]; c.friction[3] = c.friction[4] = fr[2];
      c.mu = 0; c.efc_address = -1;
      d.contact.push_back(c);
    }
  }
  d.ncon = (int)d.contact.size();
}

// ------------------------------------------------------------------------------------------ constraints
// translational / rotational Jacobian of body b at world point (dense nv columns)
template <class T>
void jac_point(const Model<T>& m, const Data<T>& d, int b, const T* point, T* jacp, T* jacr) {
  int nv = m.nv;
  for (int i = 0; i < 3 * nv; i++) { jacp[i] = 0; jacr[i] = 0; }
  if (b <= 0) return;
  T off[3];
  for (int c = 0; c < 3; c++) off[c] = point[c] - d.subtree_com[3 * m.body_rootid[b] + c];
  // last dof of the nearest ancestor (inclusive) that has dofs
  int bb = b;
  while (bb > 0 && m.body_dofnum[bb] == 0) bb = m.body_parentid[bb];
  if (bb <= 0) return;
  for (int i = m.body_dofadr[bb] + m.body_dofnum[bb] - 1; i >= 0; i = m.dof_parentid[i]) {
    const T* cd = &d.cdof[6 * i];
    T t[3];
    cross3(t, cd, off);
    for (int c = 0; c < 3; c++) { jacp[c * nv + i] = cd[3 + c] + t[c]; jacr[c * nv + i] = cd[c]; }
  }
}

template <class T>
void get_impedance(const T* solimp_in, T pos, T margin, T* imp, T* impP) {
  T dmin = mm::min((T)kMaxImp, mm::max((T)kMinImp, solimp_in[0]));
  T dmax = mm::min((T)kMaxImp, mm::max((T)kMinImp, solimp_in[1]));
  T width = mm::max((T)0, solimp_in[2]);
  T mid = mm::min((T)kMaxImp, mm::max((T)kMinImp, solimp_in[3]));
  T power = mm::max((T)1, solimp_in[4]);
  if (dmin == dmax || width <= kMinVal<T>()) { *imp = (T)0.5 * (dmin + dmax); *impP = 0; return; }
  T x = (pos - margin) / width;
  if (x < 0) x = -x;
  if (x >= 1) { *imp = dmax; *impP = 0; return; }
  if (x == 0) { *imp = dmin; *impP = 0; return; }
  T y;
  if (power == 1) y = x;
  else if (x <= mid) y = mm::pow(x, power) / mm::pow(mid, power - 1);
  else y = 1 - mm::pow(1 - x, power) / mm::pow(1 - mid, power - 1);
  *imp = dmin + y * (dmax - dmin);
  *impP = 0;
}

template <class T>
void make_constraint(const Model<T>& m, Data<T>& d) {
  int nv = m.nv;
  d.efc_J.clear(); d.efc_pos.clear(); d.efc_margin.clear(); d.efc_diagApprox.clear(); d.efc_type.clear();
  d.efc_id.clear(); d.efc_frictionloss.clear();
  std::vector<T> row(nv), jp1(3 * nv), jr1(3 * nv), jp2(3 * nv), jr2(3 * nv);
  // every row is checked against the constraint buffer (the device's hard limit maxefc): a row that does not fit is
  // dropped and raises the warning (mjWARN_CNSTRFULL), which fails a rollout
  auto add_row = [&](const T* J, T pos, T margin, T diag, int type, int id, T floss) {
    if ((int)d.efc_pos.size() >= d.maxefc) { d.warning = true; return; }
    d.efc_J.insert(d.efc_J.end(), J, J + nv);
    d.efc_pos.push_back(pos); d.efc_margin.push_back(margin); d.efc_diagApprox.push_back(diag);
    d.efc_type.push_back(type); d.efc_id.push_back(id); d.efc_frictionloss.push_back(floss);
  };
  // dof friction loss
  if (!m.disable_frictionloss)
    for (int i = 0; i < nv; i++)
      if (m.dof_frictionloss[i] > 0) {
        std::fill(row.begin(), row.end(), (T)0);
        row[i] = 1;
        add_row(row.data(), 0, 0, m.dof_invweight0[i], CNSTR_FRICTION_DOF, i, m.dof_frictionloss[i]);
      }
  // joint limits (slide / hinge)
  if (!m.disable_limit)
    for (int j = 0; j < m.njnt; j++) {
      if (!m.jnt_limited[j]) continue;
      int t = m.jnt_type[j];
      if (t != JNT_SLIDE && t != JNT_HINGE) continue;
      T q = d.qpos[m.jnt_qposadr[j]];
      for (int side = -1; side <= 1; side += 2) {
        T dist = side * (m.jnt_range[2 * j + (side + 1) / 2] - q);
        if (dist < m.jnt_margin[j]) {
          std::fill(row.begin(), row.end(), (T)0);
          row[m.jnt_dofadr[j]] = (T)-side;
          add_row(row.data(), dist, m.jnt_margin[j], m.dof_invweight0[m.jnt_dofadr[j]], CNSTR_LIMIT_JOINT, j, 0);
        }
      }
    }
  // tendon limits (fixed tendons: length = sum coef * qpos, Jacobian = coef on the wrapped dofs)
  if (!m.disable_limit)
    for (int t = 0; t < m.ntendon; t++) {
      if (!m.tendon_limited[t]) continue;
      T len = 0;
      for (int w = m.tendon_adr[t]; w < m.tendon_adr[t] + m.tendon_num[t]; w++) len += m.wrap_coef[w] * d.qpos[m.wrap_qposadr[w]];
      for (int side = -1; side <= 1; side += 2) {
        T dist = side * (m.tendon_range[2 * t + (side + 1) / 2] - len);
        if (dist < m.tendon_margin[t]) {
          std::fill(row.begin(), row.end(), (T)0);
          for (int w = m.tendon_adr[t]; w < m.tendon_adr[t] + m.tendon_num[t]; w++) row[m.wrap_dof[w]] += (T)-side * m.wrap_coef[w];
          add_row(row.data(), dist, m.tendon_margin[t], m.tendon_invweight0[t], CNSTR_LIMIT_TENDON, t, 0);
        }
      }
    }
  // contacts
  const bool pyramidal = m.cone == 0;
  for (int ci = 0; ci < d.ncon; ci++) {
    Contact<T>& c = d.contact[ci];
    int dim = c.dim;
    const int nrow = (pyramidal && dim > 1) ? 2 * (dim - 1) : dim;
    if ((int)d.efc_pos.size() + nrow > d.maxefc) { c.efc_address = -1; d.warning = true; continue; }  // mjWARN_CNSTRFULL -> failure
    int b1 = m.geom_bodyid[c.geom1], b2 = m.geom_bodyid[c.geom2];
    jac_point(m, d, b1, c.pos, jp1.data(), jr1.data());
    jac_point(m, d, b2, c.pos, jp2.data(), jr2.data());
    T tran = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
    T rot = m.body_invweight0[2 * b1 + 1] + m.body_invweight0[2 * b2 + 1];
    c.efc_address = (int)d.efc_pos.size();
    if (pyramidal && dim > 1) {
      // pyramidal cone: rows Jn +- mu_k Jt_k for every friction direction, all with pos = dist;
      // diagApprox = tran + mu_k^2 * (tran | rot)
      std::vector<T> jn(nv), jt(nv);
      auto frame_row = [&](int k, T* out) {
        const T* ax = &c.frame[3 * (k % 3)];
        const bool is_rot = k >= 3;
        for (int i = 0; i < nv; i++) {
          T s2 = 0;
          for (int a = 0; a < 3; a++)
            s2 += ax[a] * (is_rot ? (jr2[a * nv + i] - jr1[a * nv + i]) : (jp2[a * nv + i] - jp1[a * nv + i]));
          out[i] = s2;
        }
      };
      frame_row(0, jn.data());
      for (int k = 1; k < dim; k++) {
        frame_row(k, jt.data());
        const T mu = c.friction[k - 1];
        const T diag = tran + mu * mu * (k < 3 ? tran : rot);
        for (int sgn = 1; sgn >= -1; sgn -= 2) {
          for (int i = 0; i < nv; i++) row[i] = jn[i] + sgn * mu * jt[i];
          add_row(row.data(), c.dist, c.includemargin, diag, CNSTR_CONTACT_PYRAMIDAL, ci, 0);
        }
      }
      continue;
    }
    for (int k = 0; k < dim; k++) {
      const T* ax = &c.frame[3 * (k % 3)];
      bool is_rot = k >= 3;
      for (int i = 0; i < nv; i++) {
        T s = 0;
        for (int a = 0; a < 3; a++) {
          T dj = is_rot ? (jr2[a * nv + i] - jr1[a * nv + i]) : (jp2[a * nv + i] - jp1[a * nv + i]);
          s += ax[a] * dj;
        }
        row[i] = s;
      }
      int type = dim == 1 ? CNSTR_CONTACT_FRICTIONLESS : CNSTR_CONTACT_ELLIPTIC;
      add_row(row.data(), k == 0 ? c.dist : (T)0, c.includemargin, is_rot ? rot : tran, type, ci, 0);
    }
  }
  d.nefc = (int)d.efc_pos.size();
  int ne = d.nefc;
  d.efc_R.assign(ne, 0); d.efc_D.assign(ne, 0); d.efc_KBIP.assign(4 * ne, 0); d.efc_aref.assign(ne, 0);
  d.efc_vel.assign(ne, 0); d.efc_force.assign(ne, 0); d.efc_state.assign(ne, 0);
  // impedance, regularisation
  for (int i = 0; i < ne; i++) {
    const T *solref, *solimp;
    int id = d.efc_id[i];
    bool friction_row = false;
    switch (d.efc_type[i]) {
      case CNSTR_FRICTION_DOF: solref = &m.dof_solref[2 * id]; solimp = &m.dof_solimp[5 * id]; friction_row = true; break;
      case CNSTR_LIMIT_JOINT: solref = &m.jnt_solref[2 * id]; solimp = &m.jnt_solimp[5 * id]; break;
      case CNSTR_LIMIT_TENDON: solref = &m.tendon_solref[2 * id]; solimp = &m.tendon_solimp[5 * id]; break;
      default:
        solref = d.contact[id].solref; solimp = d.contact[id].solimp;
        friction_row = (d.efc_type[i] == CNSTR_CONTACT_ELLIPTIC && i > d.contact[id].efc_address);
    }
    T imp, impP;
    get_impedance(solimp, d.efc_pos[i], d.efc_margin[i], &imp, &impP);
    T dmax = mm::min((T)kMaxImp, mm::max((T)kMinImp, solimp[1]));
    T K, B;
    if (solref[0] > 0) {
      T tc = solref[0], dr = solref[1];
      if (!m.disable_refsafe) tc = mm::max(tc, 2 * m.timestep);
      K = 1 / mm::max(kMinVal<T>(), dmax * dmax * tc * tc * dr * dr);
      B = 2 / mm::max(kMinVal<T>(), dmax * tc);
    } else {
      K = -solref[0] / mm::max(kMinVal<T>(), dmax * dmax);
      B = -solref[1] / mm::max(kMinVal<T>(), dmax);
    }
    if (friction_row) K = 0;
    d.efc_KBIP[4 * i] = K; d.efc_KBIP[4 * i + 1] = B; d.efc_KBIP[4 * i + 2] = imp; d.efc_KBIP[4 * i + 3] = impP;
    d.efc_R[i] = mm::max(kMinVal<T>(), (1 - imp) * d.efc_diagApprox[i] / imp);
  }
  // friction-cone adjustment of R (elliptic): R[1] = R[0]/impratio, R[j]*mu[j]^2 constant
  for (int ci = 0; ci < d.ncon; ci++) {
    Contact<T>& c = d.contact[ci];
    if (c.efc_address < 0 || c.dim == 1) continue;
    int a = c.efc_address;
    if (pyramidal) {
      // pyramidal: all edges share R = 2 mu^2 R_first with mu = friction[0] (impratio acts through mu)
      c.mu = c.friction[0] * mm::sqrt(1 / mm::max(kMinVal<T>(), m.impratio));
      const T Rpy = 2 * c.mu * c.mu * d.efc_R[a];
      for (int j = 0; j < 2 * (c.dim - 1); j++) d.efc_R[a + j] = Rpy;
      continue;
    }
    d.efc_R[a + 1] = d.efc_R[a] / mm::max(kMinVal<T>(), m.impratio);
    c.mu = c.friction[0] * mm::sqrt(d.efc_R[a + 1] / d.efc_R[a]);
    for (int j = 1; j < c.dim - 1; j++)
      d.efc_R[a + j + 1] = d.efc_R[a + 1] * c.friction[0] * c.friction[0] / (c.friction[j] * c.friction[j]);
  }
  for (int i = 0; i < ne; i++) d.efc_D[i] = 1 / d.efc_R[i];
}

// ------------------------------------------------------------------------------------------ velocity stage
template <class T>
void com_vel(const Model<T>& m, Data<T>& d) {
  for (int c = 0; c < 6; c++) d.cvel[c] = 0;
  for (int b = 1; b < m.nbody; b++) {
    T v[6];
    for (int c = 0; c < 6; c++) v[c] = d.cvel[6 * m.body_parentid[b] + c];
    for (int j = m.body_jntadr[b]; j < m.body_jntadr[b] + m.body_jntnum[b]; j++) {
      int da = m.jnt_dofadr[j];
      int t = m.jnt_type[j];
      if (t == JNT_FREE) {
        for (int k = 0; k < 3; k++) {
          for (int c = 0; c < 6; c++) { d.cdof_dot[6 * (da + k) + c] = 0; v[c] += d.cdof[6 * (da + k) + c] * d.qvel[da + k]; }
        }
        da += 3;
      }
      if (t == JNT_FREE || t == JNT_BALL) {
        for (int k = 0; k < 3; k++) cross_motion(&d.cdof_dot[6 * (da + k)], v, &d.cdof[6 * (da + k)]);
        for (int k = 0; k < 3; k++)
          for (int c = 0; c < 6; c++) v[c] += d.cdof[6 * (da + k) + c] * d.qvel[da + k];
      } else {
        cross_motion(&d.cdof_dot[6 * da], v, &d.cdof[6 * da]);
        for (int c = 0; c < 6; c++) v[c] += d.cdof[6 * da + c] * d.qvel[da];
      }
    }
    for (int c = 0; c < 6; c++) d.cvel[6 * b + c] = v[c];
  }
  // subtree linear velocity (for subtreelinvel sensors)
  for (int b = 0; b < m.nbody; b++) {
    T off[3], wx[3];
    for (int c = 0; c < 3; c++) off[c] = d.xipos[3 * b + c] - d.subtree_com[3 * m.body_rootid[b] + c];
    cross3(wx, &d.cvel[6 * b], off);
    for (int c = 0; c < 3; c++) d.subtree_linvel[3 * b + c] = m.body_mass[b] * (d.cvel[6 * b + 3 + c] + wx[c]);
  }
  for (int b = m.nbody - 1; b > 0; b--)
    for (int c = 0; c < 3; c++) d.subtree_linvel[3 * m.body_parentid[b] + c] += d.subtree_linvel[3 * b + c];
  for (int b = 0; b < m.nbody; b++)
    for (int c = 0; c < 3; c++) d.subtree_linvel[3 * b + c] /= mm::max(kMinVal<T>(), m.body_subtreemass[b]);
}

template <class T>
void passive(const Model<T>& m, Data<T>& d) {
  for (int i = 0; i < m.nv; i++) d.qfrc_passive[i] = -m.dof_damping[i] * d.qvel[i];
  for (int j = 0; j < m.njnt; j++) {
    if (m.jnt_stiffness[j] == 0) continue;
    int t = m.jnt_type[j];
    if (t == JNT_SLIDE || t == JNT_HINGE)
      d.qfrc_passive[m.jnt_dofadr[j]] -= m.jnt_stiffness[j] * (d.qpos[m.jnt_qposadr[j]] - m.qpos_spring[m.jnt_qposadr[j]]);
  }
}

// recursive Newton-Euler with qacc = 0: Coriolis + centrifugal + gravity
template <class T>
void rne(const Model<T>& m, Data<T>& d) {
  std::vector<T> cacc(6 * m.nbody, 0), cfrc(6 * m.nbody, 0);
  for (int c = 0; c < 3; c++) cacc[3 + c] = -m.gravity[c];
  for (int b = 1; b < m.nbody; b++) {
    T a[6];
    for (int c = 0; c < 6; c++) a[c] = cacc[6 * m.body_parentid[b] + c];
    for (int i = m.body_dofadr[b]; i < m.body_dofadr[b] + m.body_dofnum[b]; i++)
      for (int c = 0; c < 6; c++) a[c] += d.cdof_dot[6 * i + c] * d.qvel[i];
    for (int c = 0; c < 6; c++) cacc[6 * b + c] = a[c];
    T f1[6], iv[6], f2[6];
    mul_inert_vec(f1, &d.cinert[10 * b], a);
    mul_inert_vec(iv, &d.cinert[10 * b], &d.cvel[6 * b]);
    cross_force(f2, &d.cvel[6 * b], iv);
    for (int c = 0; c < 6; c++) cfrc[6 * b + c] = f1[c] + f2[c];
  }
  for (int b = m.nbody - 1; b > 0; b--) {
    int p = m.body_parentid[b];
    if (p > 0)
      for (int c = 0; c < 6; c++) cfrc[6 * p + c] += cfrc[6 * b + c];
  }
  for (int i = 0; i < m.nv; i++) {
    T s = 0;
    for (int c = 0; c < 6; c++) s += d.cdof[6 * i + c] * cfrc[6 * m.dof_bodyid[i] + c];
    d.qfrc_bias[i] = s;
  }
}

template <class T>
void actuation(const Model<T>& m, Data<T>& d) {
  std::fill(d.qfrc_actuator.begin(), d.qfrc_actuator.end(), (T)0);
  for (int i = 0; i < m.nu; i++) {
    T ctrl = d.ctrl[i];
    if (m.actuator_ctrllimited[i])
      ctrl = mm::max(m.actuator_ctrlrange[2 * i], mm::min(m.actuator_ctrlrange[2 * i + 1], ctrl));
    const int j = m.actuator_trnid[i];
    const bool tendon = m.actuator_trntype[i] == 1;    // mjTRN_TENDON: length / moment through the fixed tendon's coefficients
    T gear = m.actuator_gear[i];
    T force = m.actuator_gainprm[3 * i] * ctrl;
    if (m.actuator_biastype[i] == 1) {
      T length = 0, vel = 0;
      if (tendon) {
        for (int w = m.tendon_adr[j]; w < m.tendon_adr[j] + m.tendon_num[j]; w++) {
          length += m.wrap_coef[w] * d.qpos[m.wrap_qposadr[w]]; vel += m.wrap_coef[w] * d.qvel[m.wrap_dof[w]];
        }
        length *= gear; vel *= gear;
      } else {
        length = gear * d.qpos[m.jnt_qposadr[j]]; vel = gear * d.qvel[m.jnt_dofadr[j]];
      }
      force += m.actuator_biasprm[3 * i] + m.actuator_biasprm[3 * i + 1] * length + m.actuator_biasprm[3 * i + 2] * vel;
    }
    if (m.actuator_forcelimited[i])
      force = mm::max(m.actuator_forcerange[2 * i], mm::min(m.actuator_forcerange[2 * i + 1], force));
    d.actuator_force[i] = force;
    if (tendon) {
      for (int w = m.tendon_adr[j]; w < m.tendon_adr[j] + m.tendon_num[j]; w++) d.qfrc_actuator[m.wrap_dof[w]] += gear * m.wrap_coef[w] * force;
    } else {
      d.qfrc_actuator[m.jnt_dofadr[j]] += gear * force;
    }
  }
}

// ------------------------------------------------------------------------------------------ primal Newton solver
template <class T>
struct SolverCtx {
  int nv, ne;
  std::vector<T> jar, Ma, grad, Mgrad, search, Jv, Mv, H;
  T cost, gauss;
};

// per-row cost/force/state at jar; also cone Hessians if H != nullptr (H += J^T hess J over active rows)
template <class T>
T update_constraint(const Model<T>& m, Data<T>& d, const std::vector<T>& jar, T* H) {
  int nv = m.nv, ne = d.nefc;
  T cost = 0;
  for (int i = 0; i < ne; i++) {
    int type = d.efc_type[i];
    T D = d.efc_D[i], x = jar[i];
    if (type == CNSTR_FRICTION_DOF) {
      T f = d.efc_frictionloss[i], rf = d.efc_R[i] * f;
      if (x <= -rf) { cost += f * (-(T)0.5 * rf - x); d.efc_force[i] = f; d.efc_state[i] = STATE_LINEARNEG; }
      else if (x >= rf) { cost += f * (-(T)0.5 * rf + x); d.efc_force[i] = -f; d.efc_state[i] = STATE_LINEARPOS; }
      else { cost += (T)0.5 * D * x * x; d.efc_force[i] = -D * x; d.efc_state[i] = STATE_QUADRATIC; }
    } else if (cnstr_inequality(type)) {
      if (x < 0) { cost += (T)0.5 * D * x * x; d.efc_force[i] = -D * x; d.efc_state[i] = STATE_QUADRATIC; }
      else { d.efc_force[i] = 0; d.efc_state[i] = STATE_SATISFIED; }
    } else {  // elliptic cone, first row of the contact
      Contact<T>& c = d.contact[d.efc_id[i]];
      int dim = c.dim;
      T mu = c.mu;
      T u[kMaxConDim];
      u[0] = jar[i] * mu;
      T tt = 0;
      for (int j = 1; j < dim; j++) { u[j] = jar[i + j] * c.friction[j - 1]; tt += u[j] * u[j]; }
      T N = u[0], Tn = mm::sqrt(tt);
      if (N >= mu * Tn || (Tn <= 0 && N >= 0)) {            // top zone: nothing
        for (int j = 0; j < dim; j++) { d.efc_force[i + j] = 0; d.efc_state[i + j] = STATE_SATISFIED; }
      } else if (mu * N + Tn <= 0 || (Tn <= 0 && N < 0)) {   // bottom zone: quadratic
        for (int j = 0; j < dim; j++) {
          cost += (T)0.5 * d.efc_D[i + j] * jar[i + j] * jar[i + j];
          d.efc_force[i + j] = -d.efc_D[i + j] * jar[i + j];
          d.efc_state[i + j] = STATE_QUADRATIC;
        }
      } else {                                                // middle zone: cone
        T Dm = D / (mu * mu * (1 + mu * mu));
        T NmT = N - mu * Tn;
        cost += (T)0.5 * Dm * NmT * NmT;
        d.efc_force[i] = -Dm * NmT * mu;
        for (int j = 1; j < dim; j++) d.efc_force[i + j] = -d.efc_force[i] / Tn * u[j] * c.friction[j - 1];
        for (int j = 0; j < dim; j++) d.efc_state[i + j] = STATE_CONE;
        if (H) {
          T hc[kMaxConDim * kMaxConDim];
          T scl[kMaxConDim];
          scl[0] = mu;
          for (int j = 1; j < dim; j++) scl[j] = c.friction[j - 1];
          for (int a = 0; a < dim; a++)
            for (int b = 0; b < dim; b++) {
              T h;
              if (a == 0 && b == 0) h = 1;
              else if (a == 0) h = -mu * u[b] / Tn;
              else if (b == 0) h = -mu * u[a] / Tn;
              else h = mu * N / (Tn * Tn * Tn) * u[a] * u[b] + (a == b ? (mu * mu - mu * N / Tn) : (T)0);
              hc[a * dim + b] = Dm * scl[a] * scl[b] * h;
            }
          for (int a = 0; a < dim; a++)
            for (int b = 0; b < dim; b++) {
              T h = hc[a * dim + b];
              if (h == 0) continue;
              const T* Ja = &d.efc_J[(i + a) * nv];
              const T* Jb = &d.efc_J[(i + b) * nv];
              for (int r = 0; r < nv; r++)
                for (int s = 0; s < nv; s++) H[r * nv + s] += h * Ja[r] * Jb[s];
            }
        }
      }
      i += dim - 1;
    }
  }
  if (H)
    for (int i = 0; i < ne; i++)
      if (d.efc_state[i] == STATE_QUADRATIC) {
        const T* Ji = &d.efc_J[i * nv];
        T D = d.efc_D[i];
        for (int r = 0; r < nv; r++) {
          if (Ji[r] == 0) continue;
          for (int s = 0; s < nv; s++) H[r * nv + s] += D * Ji[r] * Ji[s];
        }
      }
  return cost;
}

template <class T> struct LsPoint { T alpha, cost, d1, d2; };

// 1-D cost along the search direction and its first two derivatives
template <class T>
LsPoint<T> ls_eval(const Model<T>& m, const Data<T>& d, const SolverCtx<T>& s, const T* qg, T alpha) {
  int ne = d.nefc;
  T cost = qg[0] + alpha * qg[1] + alpha * alpha * qg[2];
  T d1 = qg[1] + 2 * alpha * qg[2], d2 = 2 * qg[2];
  for (int i = 0; i < ne; i++) {
    int type = d.efc_type[i];
    T D = d.efc_D[i], jv = s.Jv[i], x = s.jar[i] + alpha * jv;
    if (type == CNSTR_FRICTION_DOF) {
      T f = d.efc_frictionloss[i], rf = d.efc_R[i] * f;
      if (x <= -rf) { cost += f * (-(T)0.5 * rf - x); d1 += -f * jv; }
      else if (x >= rf) { cost += f * (-(T)0.5 * rf + x); d1 += f * jv; }
      else { cost += (T)0.5 * D * x * x; d1 += D * x * jv; d2 += D * jv * jv; }
    } else if (cnstr_inequality(type)) {
      if (x < 0) { cost += (T)0.5 * D * x * x; d1 += D * x * jv; d2 += D * jv * jv; }
    } else {
      const Contact<T>& c = d.contact[d.efc_id[i]];
      int dim = c.dim;
      T mu = c.mu;
      T U0 = s.jar[i] * mu, V0 = s.Jv[i] * mu, UU = 0, UV = 0, VV = 0;
      for (int j = 1; j < dim; j++) {
        T uj = s.jar[i + j] * c.friction[j - 1], vj = s.Jv[i + j] * c.friction[j - 1];
        UU += uj * uj; UV += uj * vj; VV += vj * vj;
      }
      T N = U0 + alpha * V0;
      T Tsqr = UU + alpha * (2 * UV + alpha * VV);
      T Tn = Tsqr <= 0 ? (T)0 : mm::sqrt(Tsqr);
      if (N >= mu * Tn || (Tn <= 0 && N >= 0)) {
        // nothing
      } else if (mu * N + Tn <= 0 || (Tn <= 0 && N < 0)) {
        for (int j = 0; j < dim; j++) {
          T Dj = d.efc_D[i + j], xj = s.jar[i + j] + alpha * s.Jv[i + j], vj = s.Jv[i + j];
          cost += (T)0.5 * Dj * xj * xj; d1 += Dj * xj * vj; d2 += Dj * vj * vj;
        }
      } else {
        T Dm = D / (mu * mu * (1 + mu * mu));
        T N1 = V0, T1 = (UV + alpha * VV) / Tn;
        T T2 = VV / Tn - (UV + alpha * VV) * T1 / (Tn * Tn);
        T NmT = N - mu * Tn;
        cost += (T)0.5 * Dm * NmT * NmT;
        d1 += Dm * NmT * (N1 - mu * T1);
        d2 += Dm * ((N1 - mu * T1) * (N1 - mu * T1) + NmT * (-mu * T2));
      }
      i += dim - 1;
    }
  }
  return {alpha, cost, d1, d2};
}

template <class T>
T line_search(const Model<T>& m, const Data<T>& d, const SolverCtx<T>& s, const T* qg, T scale_inv) {
  int nv = m.nv;
  T snorm = 0;
  for (int i = 0; i < nv; i++) snorm += s.search[i] * s.search[i];
  snorm = mm::sqrt(snorm);
  if (snorm < kMinVal<T>()) return 0;
  LsPoint<T> p0 = ls_eval(m, d, s, qg, (T)0);
  // derivative tolerance; the relative floor (64 eps) guards reduced precision and is inactive in fp64
  T gtol = mm::max(mm::max(m.tolerance, kTolFloor<T>()) * m.ls_tolerance * snorm * scale_inv,
                    64 * mm::eps<T>() * mm::fabs(p0.d1));
  if (p0.d2 <= kMinVal<T>()) return 0;
  // Reduced precision cannot resolve cost differences below ~eps * cost, which is where the last one or two Newton
  // iterations live.  The 1-D cost is convex and p0.d1 < 0, so acceptance there is decided on the derivative: a
  // point with |d1| < gtol is the minimiser, and a point still on the descending side (d1 <= 0, alpha > 0) cannot be
  // worse than alpha = 0.  fp64 keeps the published cost comparisons (identical in exact arithmetic).
  constexpr bool robust = sizeof(T) == 4;
  LsPoint<T> p1 = ls_eval(m, d, s, qg, -p0.d1 / p0.d2);
  if (p0.cost < p1.cost && !(robust && p1.d1 <= 0)) p1 = p0;
  if (mm::fabs(p1.d1) < gtol) return p1.alpha;
  // Newton iterations on one side until the derivative changes sign
  int iter = 0;
  LsPoint<T> p2 = p1;
  bool bracket = false;
  while (iter < m.ls_iterations) {
    iter++;
    p2 = p1;
    if (p1.d2 <= kMinVal<T>()) break;
    p1 = ls_eval(m, d, s, qg, p1.alpha - p1.d1 / p1.d2);
    if (mm::fabs(p1.d1) < gtol) return (robust || p1.cost <= p0.cost) ? p1.alpha : (T)0;
    if ((p1.d1 > 0) != (p2.d1 > 0)) { bracket = true; break; }
  }
  if (!bracket) return ((robust && p1.d1 <= 0 && p1.alpha > 0) || p1.cost < p0.cost) ? p1.alpha : (T)0;
  // bracketed refinement: safeguarded Newton
  LsPoint<T> lo = p1.d1 < 0 ? p1 : p2, hi = p1.d1 < 0 ? p2 : p1;
  while (iter < m.ls_iterations) {
    iter++;
    const LsPoint<T>& from = mm::fabs(lo.d1) < mm::fabs(hi.d1) ? lo : hi;
    T a = from.d2 > kMinVal<T>() ? from.alpha - from.d1 / from.d2 : (T)0.5 * (lo.alpha + hi.alpha);
    T amin = mm::min(lo.alpha, hi.alpha), amax = mm::max(lo.alpha, hi.alpha);
    if (!(a > amin && a < amax)) a = (T)0.5 * (lo.alpha + hi.alpha);
    if (a == lo.alpha || a == hi.alpha) break;
    LsPoint<T> pm = ls_eval(m, d, s, qg, a);
    if (mm::fabs(pm.d1) < gtol) return (robust || pm.cost <= p0.cost) ? pm.alpha : (T)0;
    if (pm.d1 < 0) lo = pm; else hi = pm;
  }
  if (robust) {   // bracket closed to adjacent values: the descending end is a guaranteed improvement
    if (lo.alpha > 0) return lo.alpha;
    return hi.cost < p0.cost ? hi.alpha : (T)0;
  }
  const LsPoint<T>& best = lo.cost < hi.cost ? lo : hi;
  return best.cost < p0.cost ? best.alpha : (T)0;
}

inline bool solver_trace() { static const bool on = std::getenv("ORACLE_SOLVER_TRACE") != nullptr; return on; }

template <class T>
void solve_constraints(const Model<T>& m, Data<T>& d) {
  int nv = m.nv, ne = d.nefc;
  d.solver_niter = 0;
  if (ne == 0) {
    d.qacc = d.qacc_smooth;
    std::fill(d.qfrc_constraint.begin(), d.qfrc_constraint.end(), (T)0);
    return;
  }
  SolverCtx<T> s;
  s.nv = nv; s.ne = ne;
  s.jar.assign(ne, 0); s.Ma.assign(nv, 0); s.grad.assign(nv, 0); s.Mgrad.assign(nv, 0); s.search.assign(nv, 0);
  s.Jv.assign(ne, 0); s.Mv.assign(nv, 0); s.H.assign(nv * nv, 0);
  auto mulM = [&](std::vector<T>& r, const std::vector<T>& v) {
    for (int i = 0; i < nv; i++) { T a = 0; for (int j = 0; j < nv; j++) a += d.qM[i * nv + j] * v[j]; r[i] = a; }
  };
  auto mulJ = [&](std::vector<T>& r, const std::vector<T>& v) {
    for (int i = 0; i < ne; i++) { T a = 0; for (int j = 0; j < nv; j++) a += d.efc_J[i * nv + j] * v[j]; r[i] = a; }
  };
  auto total_cost = [&](const std::vector<T>& qacc, bool hess) {
    mulM(s.Ma, qacc);
    mulJ(s.jar, qacc);
    for (int i = 0; i < ne; i++) s.jar[i] -= d.efc_aref[i];
    if (hess) s.H = d.qM;
    T c = update_constraint(m, d, s.jar, hess ? s.H.data() : nullptr);
    T g = 0;
    for (int i = 0; i < nv; i++) g += (s.Ma[i] - d.qfrc_smooth[i]) * (qacc[i] - d.qacc_smooth[i]);
    s.gauss = (T)0.5 * g;
    return c + s.gauss;
  };
  // warm start: keep qacc_warmstart only if it is better than the unconstrained acceleration
  if (!m.disable_warmstart) {
    T cw = total_cost(d.qacc_warmstart, false);
    T cs = total_cost(d.qacc_smooth, false);
    d.qacc = cw < cs ? d.qacc_warmstart : d.qacc_smooth;
  } else {
    d.qacc = d.qacc_smooth;
  }
  T scale_inv = m.meaninertia * (T)mm::max(1, nv);  // 1/scale
  auto gradient_and_direction = [&]() {
    // grad = Ma - qfrc_smooth - J^T force;  search = -H^-1 grad
    for (int i = 0; i < nv; i++) {
      T a = s.Ma[i] - d.qfrc_smooth[i];
      for (int r = 0; r < ne; r++) a -= d.efc_J[r * nv + i] * d.efc_force[r];
      s.grad[i] = a;
    }
    chol_factor(s.H.data(), nv);
    chol_solve(s.Mgrad.data(), s.H.data(), s.grad.data(), nv);
    for (int i = 0; i < nv; i++) s.search[i] = -s.Mgrad[i];
  };
  s.cost = total_cost(d.qacc, true);
  gradient_and_direction();
  T prev_gradient = std::numeric_limits<T>::max();
  int stalls = 0;
  for (int iter = 0; iter < m.iterations; iter++) {
    mulM(s.Mv, s.search);
    mulJ(s.Jv, s.search);
    T qg[3] = {s.gauss, 0, 0};
    for (int i = 0; i < nv; i++) {
      qg[1] += s.search[i] * (s.Ma[i] - d.qfrc_smooth[i]);
      qg[2] += (T)0.5 * s.search[i] * s.Mv[i];
    }
    T alpha = line_search(m, d, s, qg, scale_inv);
    if (alpha == 0) break;
    for (int i = 0; i < nv; i++) d.qacc[i] += alpha * s.search[i];
    T old = s.cost;
    s.cost = total_cost(d.qacc, true);
    gradient_and_direction();
    d.solver_niter = iter + 1;
    T gn = 0;
    for (int i = 0; i < nv; i++) gn += s.grad[i] * s.grad[i];
    T improvement = (old - s.cost) / scale_inv, gradient = mm::sqrt(gn) / scale_inv;
    const T tol = mm::max(m.tolerance, kTolFloor<T>());
    if (solver_trace()) {   // ORACLE_SOLVER_TRACE=1: one line per Newton iteration (diagnostics only)
      int ncone = 0, nquad = 0;
      for (int r = 0; r < ne; r++) { ncone += d.efc_state[r] == 4; nquad += d.efc_state[r] == 1; }
      std::fprintf(stderr, "  newton %2d  alpha %.4f  cost %.10g  improvement %.3e  gradient %.3e  (tol %.1e)  rows %d quad %d cone %d\n",
                   iter + 1, (double)alpha, (double)s.cost, (double)improvement, (double)gradient, (double)tol, ne, nquad, ncone);
    }
    if (sizeof(T) == 4) {
      // reduced precision: a cost decrease below the rounding of the cost itself is not evidence of convergence
      // (the gradient can still be 1e4 x tol there); such an iteration only stops the solver when the gradient no
      // longer shrinks.  Resolvable improvements follow the published rule.
      const bool resolvable = mm::fabs(old - s.cost) > 16 * mm::eps<T>() * mm::fabs(s.cost);
      // rounding floor of the gradient itself: eps x the magnitude of the terms it is the difference of
      T gabs = 0;
      for (int i = 0; i < nv; i++) { T a = mm::fabs(s.Ma[i]) + mm::fabs(d.qfrc_smooth[i]) + mm::fabs(s.Ma[i] - d.qfrc_smooth[i] - s.grad[i]); gabs += a * a; }
      const T gfloor = (T)kGradFloor * mm::eps<T>() * mm::sqrt(gabs) / scale_inv;
      if (gradient < mm::max(tol, gfloor)) break;
      // a (near) full Newton step that fails to shrink the gradient is the rounding floor; a short step is a kink
      // crossing (cone / friction-loss zone change) and the next step is a full one - allow a few of those
      if (resolvable) { if (improvement < tol) break; stalls = 0; }
      else if (gradient > (T)0.5 * prev_gradient && (alpha > (T)0.5 || ++stalls >= 3)) break;
      prev_gradient = gradient;
    } else if (improvement < tol || gradient < tol) break;
  }
  solver_hist()[std::min(d.solver_niter, 63)]++;
  for (int i = 0; i < nv; i++) {
    T a = 0;
    for (int r = 0; r < ne; r++) a += d.efc_J[r * nv + i] * d.efc_force[r];
    d.qfrc_constraint[i] = a;
  }
}

// ------------------------------------------------------------------------------------------ pipeline
template <class T> using ResidualCallback = void (*)(const Model<T>&, Data<T>&, T* residual);

template <class T>
void forward(const Model<T>& m, Data<T>& d, ResidualCallback<T> cb) {
  int nv = m.nv;
  kinematics(m, d);
  com_pos(m, d);
  crb(m, d);
  collision(m, d);
  make_constraint(m, d);
  com_vel(m, d);
  passive(m, d);
  rne(m, d);
  // reference acceleration of each constraint row: aref = -B*vel - K*imp*(pos - margin)
  for (int i = 0; i < d.nefc; i++) {
    T v = 0;
    for (int j = 0; j < nv; j++) v += d.efc_J[i * nv + j] * d.qvel[j];
    d.efc_vel[i] = v;
    d.efc_aref[i] = -d.efc_KBIP[4 * i + 1] * v - d.efc_KBIP[4 * i] * d.efc_KBIP[4 * i + 2] * (d.efc_pos[i] - d.efc_margin[i]);
  }
  actuation(m, d);
  for (int i = 0; i < nv; i++) d.qfrc_smooth[i] = d.qfrc_passive[i] - d.qfrc_bias[i] + d.qfrc_actuator[i];
  if (d.xfrc_active) {   // mj_xfrcAccumulate: Cartesian force / torque at each body's centre of mass -> joint space
    std::vector<T> jp(3 * nv), jr(3 * nv);
    for (int b = 1; b < m.nbody; b++) {
      const T* f = &d.xfrc_applied[6 * b];
      jac_point(m, d, b, &d.xipos[3 * b], jp.data(), jr.data());
      for (int i = 0; i < nv; i++)
        for (int c = 0; c < 3; c++) d.qfrc_smooth[i] += jp[c * nv + i] * f[c] + jr[c * nv + i] * f[3 + c];
    }
  }
  chol_solve(d.qacc_smooth.data(), d.qLD.data(), d.qfrc_smooth.data(), nv);
  solve_constraints(m, d);
  if (cb) cb(m, d, d.residual.data());  // mjcb_sensor at mjSTAGE_ACC (mjpc/app.cc:110-126)
}

template <class T>
bool bad(const std::vector<T>& v) {
  for (T x : v)
    if (!(mm::fabs(x) < (T)kMaxVal)) return true;  // catches NaN and |x| >= mjMAXVAL
  return false;
}

// semi-implicit Euler with implicit joint damping
template <class T>
void euler(const Model<T>& m, Data<T>& d) {
  int nv = m.nv;
  T h = m.timestep;
  std::vector<T> qacc = d.qacc;
  bool damped = false;
  for (int i = 0; i < nv; i++) damped |= m.dof_damping[i] > 0;
  if (damped && !m.disable_eulerdamp) {
    std::vector<T> MM = d.qM, f(nv);
    for (int i = 0; i < nv; i++) { MM[i * nv + i] += h * m.dof_damping[i]; f[i] = d.qfrc_smooth[i] + d.qfrc_constraint[i]; }
    chol_factor(MM.data(), nv);
    chol_solve(qacc.data(), MM.data(), f.data(), nv);
  }
  for (int i = 0; i < nv; i++) d.qvel[i] += h * qacc[i];
  for (int j = 0; j < m.njnt; j++) {
    int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
    switch (m.jnt_type[j]) {
      case JNT_FREE:
        for (int c = 0; c < 3; c++) d.qpos[qa + c] += h * d.qvel[da + c];
        quat_integrate(&d.qpos[qa + 3], &d.qvel[da + 3], h);
        break;
      case JNT_BALL: quat_integrate(&d.qpos[qa], &d.qvel[da], h); break;
      default: d.qpos[qa] += h * d.qvel[da];
    }
  }
  d.time += h;
}

// mj_step: checks -> forward -> checks -> integrate.  Any bad value raises d.warning, which the
// rollout turns into failure / return 1e6 (mjpc/trajectory.cc:169-173, utilities.cc:804-816).
template <class T>
void step(const Model<T>& m, Data<T>& d, ResidualCallback<T> cb) {
  if (bad(d.qpos) || bad(d.qvel)) { d.warning = true; return; }
  forward(m, d, cb);
  if (bad(d.qacc)) { d.warning = true; return; }
  d.qacc_warmstart = d.qacc;
  euler(m, d);
}

}  // namespace oracle
