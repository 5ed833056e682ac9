// TEST INFRASTRUCTURE - measurement sensors on the CPU oracle (oracle/physics.h), fp64 or fp32.
//
// The same single step as the oracle's step_batch (forward, warning on a bad qacc, warm start from qacc, Euler), with an
// optional xfrc_applied [B][nbody][6] for the step (mj_xfrcAccumulate, as the plants' disturbances apply it), plus
// the measurement sensors [start, start + count) of each pre-step state, read after the constraint solve as mj_step's
// sensor stage reads them:
//   jointpos / jointvel  qpos[jnt_qposadr] / qvel[jnt_dofadr]
//   framepos             site_xpos, xipos (body), xpos (xbody) or geom_xpos
//   touch                MuJoCo's definition: the normal forces of the contacts with constraint rows that involve a
//                        geom of the site's body, counted when the contact point lies in the site's sphere zone or the
//                        ray from the point along the contact normal, oriented into the site's body, hits the zone.
//                        Normal force: the normal row (elliptic / frictionless) or the sum of the 2 (condim - 1)
//                        pyramid edges.
//   gyro / velocimeter   mj_objectVelocity of the site with flg_local: the body's com-based velocity cvel = (w, v)
//                        moved to the site (v - (site_xpos - subtree_com[root]) x w) and rotated by site_xmat'
//   accelerometer        mj_objectAcceleration of the site with flg_local: the body's post-constraint com-based
//                        acceleration (mj_rnePostConstraint's recursion cacc[b] = cacc[parent] + cdof_dot qvel +
//                        cdof qacc from cacc[world] = (0, -gravity)), moved and rotated like the velocity, plus
//                        (R' w) x (R' v_site)
// A frame is a site (site_xpos, site_xmat, xquat[site_body] site_quat), a body's inertial frame (xipos, ximat,
// xquat body_iquat), an xbody (xpos, xmat, xquat) or a geom (geom_xpos, geom_xmat, xquat[geom_body] geom_quat):
//   framequat            the frame's quaternion as listed
//   framex/y/zaxis       column 0 / 1 / 2 of the frame's matrix
//   framelinvel / -angvel  mj_objectVelocity in the world frame: cvel of the frame's body moved to the frame's position
//   framelinacc / -angacc  mj_objectAcceleration in the world frame: the post-constraint cacc moved the same way, plus
//                        w x v_frame on the linear part
//   subtreecom / subtreelinvel  subtree_com / subtree_linvel of the body
//   subtreeangmom        sum over the body's descendants j (and itself) of the spin ximat_j diag(I_j) ximat_j' w_j and
//                        the orbital part (xipos_j - subtree_com) x m_j (v_j - subtree_linvel), with v_j the velocity
//                        of j's centre of mass
//   ballquat / ballangvel  the ball joint's normalised quaternion / its 3 dof velocities
//   jointactuatorfrc     qfrc_actuator of a slide or hinge joint's dof
//   actuatorpos / -vel   gear times the joint's qpos / qvel, or times the fixed tendon's length / velocity
//   actuatorfrc          actuator_force (after the force limit)
//   tendonpos / -vel     the fixed tendon's sum coef qpos / sum coef qvel
//   magnetometer         site_xmat' opt.magnetic (MuJoCo's mj_sensorPos)
//   rangefinder          mj_ray(pnt = site_xpos, vec = column 2 of site_xmat, geomgroup NULL, flg_static 1,
//                        bodyexclude = the site's body): the least non-negative distance to a geom not of the site's
//                        body whose alpha is not 0, or -1.  The ray-geom distances are restated below from the
//                        surfaces' equations, in the precision of the model (fp32 arithmetic in the fp32 oracle).
// The sensor table is read from the blob's sensor_* / site_* entries.  Written from the definition, independently of
// the device's k_sensors; the oracle itself is not modified.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <vector>

#include "../oracle/physics.h"

using namespace oracle;

namespace {

enum { SENS_FRAMEPOS = 1, SENS_JOINTPOS = 2, SENS_TOUCH = 3, SENS_SUBTREECOM = 4, SENS_SUBTREELINVEL = 5,
       SENS_FRAMELINVEL = 6, SENS_FRAMEQUAT = 7, SENS_JOINTVEL = 9, SENS_ACCELEROMETER = 10, SENS_VELOCIMETER = 11,
       SENS_GYRO = 12, SENS_FRAMEANGVEL = 13, SENS_FRAMEXAXIS = 14, SENS_FRAMEYAXIS = 15, SENS_FRAMEZAXIS = 16,
       SENS_FRAMELINACC = 17, SENS_FRAMEANGACC = 18, SENS_SUBTREEANGMOM = 19, SENS_BALLQUAT = 20,
       SENS_BALLANGVEL = 21, SENS_JOINTACTUATORFRC = 22, SENS_ACTUATORPOS = 23, SENS_ACTUATORVEL = 24,
       SENS_ACTUATORFRC = 25, SENS_TENDONPOS = 26, SENS_TENDONVEL = 27, SENS_MAGNETOMETER = 28,
       SENS_RANGEFINDER = 29 };
enum { OBJ_BODY = 0, OBJ_XBODY = 1, OBJ_GEOM = 2, OBJ_SITE = 3 };

struct Table {
  std::vector<int> type, objtype, objid, dim, adr, site_type;
  std::vector<double> site_size;
  double magnetic[3] = {0, -0.5, 0};   // opt.magnetic, MuJoCo's default unless the blob has opt_magnetic
  std::vector<double> geom_alpha;      // empty: every geom has alpha 1
};

// ----------------------------------------------------------------------------------------------- ray casting
// t >= 0 of the ray p + t v (v unit) on each geom surface, in the geom's frame; -1: no such t.  A ray that starts
// inside a closed surface hits it on the way out.
template <class T>
T smallest(T a, T b) { return a < 0 ? b : (b < 0 ? a : std::min(a, b)); }

// plane z = 0, hit from its front (+z) side only, within |x| <= size0 and |y| <= size1 when those are positive
template <class T>
T ray_plane(const T* p, const T* v, const T* size) {
  if (!(v[2] < 0)) return -1;
  const T t = -p[2] / v[2];
  if (t < 0) return -1;
  const T x = p[0] + t * v[0], y = p[1] + t * v[1];
  if ((size[0] > 0 && std::fabs(x) > size[0]) || (size[1] > 0 && std::fabs(y) > size[1])) return -1;
  return t;
}

// |p + t v - c|^2 = r^2 in coordinates scaled by s (an ellipsoid of semi-axes s; a sphere: s = r, r = 1)
template <class T>
void quadric_roots(const T* p, const T* v, const T* c, const T* s, T* t0, T* t1) {
  T a = 0, b = 0, cc = -1;
  for (int k = 0; k < 3; k++) {
    const T pk = (p[k] - c[k]) / s[k], vk = v[k] / s[k];
    a += vk * vk; b += pk * vk; cc += pk * pk;
  }
  const T disc = b * b - a * cc;
  *t0 = *t1 = -1;
  if (disc < 0 || a <= 0) return;
  *t0 = (-b - std::sqrt(disc)) / a;
  *t1 = (-b + std::sqrt(disc)) / a;
}

template <class T>
T ray_ellipsoid(const T* p, const T* v, const T* size) {
  const T c[3] = {0, 0, 0};
  T t0, t1;
  quadric_roots(p, v, c, size, &t0, &t1);
  return t0 >= 0 ? t0 : (t1 >= 0 ? t1 : T(-1));
}

// the lateral surface x^2 + y^2 = r^2, |z| <= h
template <class T>
T ray_tube(const T* p, const T* v, T r, T h) {
  const T a = v[0] * v[0] + v[1] * v[1];
  if (a <= 0) return -1;
  const T b = p[0] * v[0] + p[1] * v[1], cc = p[0] * p[0] + p[1] * p[1] - r * r, disc = b * b - a * cc;
  if (disc < 0) return -1;
  T best = -1;
  for (T t : {(-b - std::sqrt(disc)) / a, (-b + std::sqrt(disc)) / a})
    if (t >= 0 && std::fabs(p[2] + t * v[2]) <= h) best = smallest(best, t);
  return best;
}

// capsule: the tube and the two hemispherical caps of radius r centred at z = +-h (each beyond its end)
template <class T>
T ray_capsule(const T* p, const T* v, const T* size) {
  const T r = size[0], h = size[1];
  T best = ray_tube(p, v, r, h);
  const T s[3] = {r, r, r};
  for (int side = -1; side <= 1; side += 2) {
    const T c[3] = {0, 0, side * h};
    T t[2];
    quadric_roots(p, v, c, s, &t[0], &t[1]);
    for (T x : t)
      if (x >= 0 && side * (p[2] + x * v[2]) >= h) best = smallest(best, x);
  }
  return best;
}

// cylinder: the tube and the two discs z = +-h of radius r
template <class T>
T ray_cylinder(const T* p, const T* v, const T* size) {
  const T r = size[0], h = size[1];
  T best = ray_tube(p, v, r, h);
  if (v[2] != 0)
    for (int side = -1; side <= 1; side += 2) {
      const T t = (side * h - p[2]) / v[2], x = p[0] + t * v[0], y = p[1] + t * v[1];
      if (t >= 0 && x * x + y * y <= r * r) best = smallest(best, t);
    }
  return best;
}

// box |x_k| <= size_k: each face plane x_k = +-size_k, hit inside the face's rectangle
template <class T>
T ray_box(const T* p, const T* v, const T* size) {
  T best = -1;
  for (int k = 0; k < 3; k++) {
    if (v[k] == 0) continue;
    for (int side = -1; side <= 1; side += 2) {
      const T t = (side * size[k] - p[k]) / v[k];
      if (t < 0) continue;
      bool in = true;
      for (int j = 0; j < 3; j++)
        if (j != k && std::fabs(p[j] + t * v[j]) > size[j]) in = false;
      if (in) best = smallest(best, t);
    }
  }
  return best;
}

template <class T>
double rangefinder(const Model<T>& m, const Data<T>& d, const Table& tab, int site) {
  const int body = m.site_bodyid[site];
  const T* R = &d.site_xmat[9 * site];
  const T v[3] = {R[2], R[5], R[8]};
  T best = -1;
  for (int g = 0; g < m.ngeom; g++) {
    if (m.geom_bodyid[g] == body || (!tab.geom_alpha.empty() && tab.geom_alpha[g] == 0)) continue;
    // the ray in the geom's frame: geom_xmat' (pnt - geom_xpos), geom_xmat' vec
    const T *gp = &d.geom_xpos[3 * g], *gm = &d.geom_xmat[9 * g], *size = &m.geom_size[3 * g];
    T lp[3] = {0, 0, 0}, lv[3] = {0, 0, 0};
    for (int a = 0; a < 3; a++)
      for (int k = 0; k < 3; k++) {
        lp[a] += gm[3 * k + a] * (d.site_xpos[3 * site + k] - gp[k]);
        lv[a] += gm[3 * k + a] * v[k];
      }
    T t;
    switch (m.geom_type[g]) {
      case GEOM_PLANE: t = ray_plane(lp, lv, size); break;
      case GEOM_SPHERE: { const T s[3] = {size[0], size[0], size[0]}; t = ray_ellipsoid(lp, lv, s); break; }
      case GEOM_CAPSULE: t = ray_capsule(lp, lv, size); break;
      case GEOM_ELLIPSOID: t = ray_ellipsoid(lp, lv, size); break;
      case GEOM_CYLINDER: t = ray_cylinder(lp, lv, size); break;
      case GEOM_BOX: t = ray_box(lp, lv, size); break;
      default: throw std::runtime_error("rangefinder: a geom type rays are not cast against");
    }
    best = smallest(best, t);
  }
  return best;
}

template <class T>
struct Sim {
  Model<T> model;
  Data<T> data;
  Sim(const void* blob, size_t n) : model(blob, n), data(model) {}
};

struct Handle {
  int precision;
  Table tab;
  std::unique_ptr<Sim<double>> s64;
  std::unique_ptr<Sim<float>> s32;
};

template <class T>
double touch(const Model<T>& m, const Data<T>& d, const Table& tab, int site) {
  if (tab.site_type[site] != 2) throw std::runtime_error("touch zone other than a sphere");
  const int body = m.site_bodyid[site];
  const double r = tab.site_size[3 * site];
  const bool pyramidal = m.cone == 0;
  double sum = 0;
  for (int i = 0; i < d.ncon; i++) {
    const Contact<T>& c = d.contact[i];
    if (c.geom1 < 0 || c.efc_address < 0) continue;
    const int b1 = m.geom_bodyid[c.geom1], b2 = m.geom_bodyid[c.geom2];
    if (b1 != body && b2 != body) continue;
    double f = 0;
    const int nrow = pyramidal && c.dim > 1 ? 2 * (c.dim - 1) : 1;
    for (int k = 0; k < nrow; k++) f += (double)d.efc_force[c.efc_address + k];
    if (!(f > 0)) continue;
    const double sg = b2 == body ? 1.0 : -1.0;   // the frame normal points from geom 1 into geom 2
    double oc[3], dir[3], b = 0, cc = -r * r;
    for (int q = 0; q < 3; q++) {
      oc[q] = (double)c.pos[q] - (double)d.site_xpos[3 * site + q];
      dir[q] = sg * (double)c.frame[q];
      b += oc[q] * dir[q];
      cc += oc[q] * oc[q];
    }
    if (cc <= 0 || (b < 0 && b * b - cc >= 0)) sum += f;
  }
  return sum;
}

// site_xmat' (vec moved from subtree_com[root] to the site) for a com-based motion vector vec = (angular, linear);
// out = (angular, linear) in the site frame
template <class T>
void site_motion(const Model<T>& m, const Data<T>& d, int site, const double* vec, double* out) {
  const int b = m.site_bodyid[site], root = m.body_rootid[b];
  double off[3], lin[3];
  for (int q = 0; q < 3; q++) off[q] = (double)d.site_xpos[3 * site + q] - (double)d.subtree_com[3 * root + q];
  lin[0] = vec[3] - (off[1] * vec[2] - off[2] * vec[1]);
  lin[1] = vec[4] - (off[2] * vec[0] - off[0] * vec[2]);
  lin[2] = vec[5] - (off[0] * vec[1] - off[1] * vec[0]);
  const T* R = &d.site_xmat[9 * site];
  for (int r = 0; r < 3; r++) {
    out[r] = out[3 + r] = 0;
    for (int k = 0; k < 3; k++) {
      out[r] += (double)R[3 * k + r] * vec[k];
      out[3 + r] += (double)R[3 * k + r] * lin[k];
    }
  }
}

// mj_rnePostConstraint's com-based body accelerations without contact or applied forces: cacc [nbody][6]
template <class T>
std::vector<double> post_constraint_acc(const Model<T>& m, const Data<T>& d) {
  std::vector<double> cacc(6 * (size_t)m.nbody, 0.0);
  for (int q = 0; q < 3; q++) cacc[3 + q] = -(double)m.gravity[q];
  for (int b = 1; b < m.nbody; b++) {
    double* a = &cacc[6 * (size_t)b];
    const double* ap = &cacc[6 * (size_t)m.body_parentid[b]];
    for (int q = 0; q < 6; q++) a[q] = ap[q];
    for (int i = m.body_dofadr[b]; i < m.body_dofadr[b] + m.body_dofnum[b]; i++)
      for (int q = 0; q < 6; q++)
        a[q] += (double)d.cdof_dot[6 * i + q] * (double)d.qvel[i] + (double)d.cdof[6 * i + q] * (double)d.qacc[i];
  }
  return cacc;
}

void qmul(double* r, const double* a, const double* b) {
  r[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  r[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  r[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  r[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

void cross(double* r, const double* a, const double* b) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}

// a frame sensor's object: position, rotation matrix (row-major), quaternion, and the body it moves with
struct Frame {
  double p[3], R[9], q[4];
  int body;
};

template <class T>
Frame frame(const Model<T>& m, const Data<T>& d, int objtype, int id) {
  Frame f;
  const T *p, *R, *local = nullptr;
  switch (objtype) {
    case OBJ_SITE: f.body = m.site_bodyid[id]; p = &d.site_xpos[3 * id]; R = &d.site_xmat[9 * id]; local = &m.site_quat[4 * id]; break;
    case OBJ_GEOM: f.body = m.geom_bodyid[id]; p = &d.geom_xpos[3 * id]; R = &d.geom_xmat[9 * id]; local = &m.geom_quat[4 * id]; break;
    case OBJ_XBODY: f.body = id; p = &d.xpos[3 * id]; R = &d.xmat[9 * id]; break;
    case OBJ_BODY: f.body = id; p = &d.xipos[3 * id]; R = &d.ximat[9 * id]; local = &m.body_iquat[4 * id]; break;
    default: throw std::runtime_error("frame sensor of an unknown object type");
  }
  double xq[4], lq[4];
  for (int q = 0; q < 4; q++) xq[q] = d.xquat[4 * f.body + q];
  for (int q = 0; q < 3; q++) f.p[q] = p[q];
  for (int q = 0; q < 9; q++) f.R[q] = R[q];
  if (local) {
    for (int q = 0; q < 4; q++) lq[q] = local[q];
    qmul(f.q, xq, lq);
  } else {
    for (int q = 0; q < 4; q++) f.q[q] = xq[q];
  }
  return f;
}

// the world-frame angular and linear velocity (w, v) of the point p moving with body b (mj_objectVelocity)
template <class T>
void point_velocity(const Model<T>& m, const Data<T>& d, int b, const double* p, double* w, double* v) {
  double off[3], t[3];
  for (int q = 0; q < 3; q++) { w[q] = d.cvel[6 * b + q]; off[q] = p[q] - (double)d.subtree_com[3 * m.body_rootid[b] + q]; }
  cross(t, off, w);
  for (int q = 0; q < 3; q++) v[q] = (double)d.cvel[6 * b + 3 + q] - t[q];
}

// a fixed tendon's length (vel false) or velocity
template <class T>
double tendon(const Model<T>& m, const Data<T>& d, int t, bool vel) {
  double x = 0;
  for (int w = m.tendon_adr[t]; w < m.tendon_adr[t] + m.tendon_num[t]; w++)
    x += (double)m.wrap_coef[w] * (vel ? (double)d.qvel[m.wrap_dof[w]] : (double)d.qpos[m.wrap_qposadr[w]]);
  return x;
}

template <class T>
void subtree_angmom(const Model<T>& m, const Data<T>& d, int body, double* L) {
  const T *com = &d.subtree_com[3 * body], *slin = &d.subtree_linvel[3 * body];
  L[0] = L[1] = L[2] = 0;
  for (int j = body; j < m.nbody; j++) {
    int k = j;
    while (k > body) k = m.body_parentid[k];
    if (k != body) continue;   // not a descendant
    double p[3], w[3], v[3], wl[3] = {0, 0, 0}, r[3], mv[3], t[3];
    for (int q = 0; q < 3; q++) p[q] = d.xipos[3 * j + q];
    point_velocity(m, d, j, p, w, v);
    const T* R = &d.ximat[9 * j];
    for (int a = 0; a < 3; a++)
      for (int q = 0; q < 3; q++) wl[a] += (double)R[3 * q + a] * w[q];
    for (int a = 0; a < 3; a++) wl[a] *= (double)m.body_inertia[3 * j + a];
    for (int q = 0; q < 3; q++) {
      for (int a = 0; a < 3; a++) L[q] += (double)R[3 * q + a] * wl[a];
      r[q] = p[q] - (double)com[q];
      mv[q] = (double)m.body_mass[j] * (v[q] - (double)slin[q]);
    }
    cross(t, r, mv);
    for (int q = 0; q < 3; q++) L[q] += t[q];
  }
}

template <class T>
void sensors(const Model<T>& m, const Data<T>& d, const Table& tab, int start, int count, double* out) {
  const int adr0 = tab.adr[start];
  std::vector<double> cacc;
  for (int s = start; s < start + count; s++) {
    double* o = out + (tab.adr[s] - adr0);
    const int id = tab.objid[s];
    switch (tab.type[s]) {
      case SENS_JOINTPOS: o[0] = d.qpos[m.jnt_qposadr[id]]; break;
      case SENS_JOINTVEL: o[0] = d.qvel[m.jnt_dofadr[id]]; break;
      case SENS_FRAMEPOS: {
        const std::vector<T>& p = tab.objtype[s] == OBJ_SITE ? d.site_xpos : tab.objtype[s] == OBJ_GEOM ? d.geom_xpos
                                  : tab.objtype[s] == OBJ_XBODY ? d.xpos : d.xipos;
        for (int q = 0; q < 3; q++) o[q] = p[3 * id + q];
        break;
      }
      case SENS_TOUCH: o[0] = touch(m, d, tab, id); break;
      case SENS_GYRO: case SENS_VELOCIMETER: case SENS_ACCELEROMETER: {
        if (tab.objtype[s] != OBJ_SITE) throw std::runtime_error("IMU sensor of an object other than a site");
        const int b = m.site_bodyid[id];
        double vel[6], v[6];
        for (int q = 0; q < 6; q++) vel[q] = d.cvel[6 * b + q];
        site_motion(m, d, id, vel, v);
        if (tab.type[s] == SENS_GYRO) { for (int q = 0; q < 3; q++) o[q] = v[q]; break; }
        if (tab.type[s] == SENS_VELOCIMETER) { for (int q = 0; q < 3; q++) o[q] = v[3 + q]; break; }
        if (cacc.empty()) cacc = post_constraint_acc(m, d);
        double a[6];
        site_motion(m, d, id, &cacc[6 * (size_t)b], a);
        o[0] = a[3] + v[1] * v[5] - v[2] * v[4];
        o[1] = a[4] + v[2] * v[3] - v[0] * v[5];
        o[2] = a[5] + v[0] * v[4] - v[1] * v[3];
        break;
      }
      case SENS_FRAMEQUAT: case SENS_FRAMEXAXIS: case SENS_FRAMEYAXIS: case SENS_FRAMEZAXIS: {
        const Frame f = frame(m, d, tab.objtype[s], id);
        if (tab.type[s] == SENS_FRAMEQUAT) { for (int q = 0; q < 4; q++) o[q] = f.q[q]; break; }
        const int col = tab.type[s] - SENS_FRAMEXAXIS;
        for (int q = 0; q < 3; q++) o[q] = f.R[3 * q + col];
        break;
      }
      case SENS_FRAMELINVEL: case SENS_FRAMEANGVEL: case SENS_FRAMELINACC: case SENS_FRAMEANGACC: {
        const Frame f = frame(m, d, tab.objtype[s], id);
        double w[3], v[3];
        point_velocity(m, d, f.body, f.p, w, v);
        if (tab.type[s] == SENS_FRAMEANGVEL) { for (int q = 0; q < 3; q++) o[q] = w[q]; break; }
        if (tab.type[s] == SENS_FRAMELINVEL) { for (int q = 0; q < 3; q++) o[q] = v[q]; break; }
        if (cacc.empty()) cacc = post_constraint_acc(m, d);
        const double* a = &cacc[6 * (size_t)f.body];
        if (tab.type[s] == SENS_FRAMEANGACC) { for (int q = 0; q < 3; q++) o[q] = a[q]; break; }
        double off[3], t[3], wv[3];
        for (int q = 0; q < 3; q++) off[q] = f.p[q] - (double)d.subtree_com[3 * m.body_rootid[f.body] + q];
        cross(t, off, a);
        cross(wv, w, v);
        for (int q = 0; q < 3; q++) o[q] = a[3 + q] - t[q] + wv[q];
        break;
      }
      case SENS_SUBTREECOM: for (int q = 0; q < 3; q++) o[q] = d.subtree_com[3 * id + q]; break;
      case SENS_SUBTREELINVEL: for (int q = 0; q < 3; q++) o[q] = d.subtree_linvel[3 * id + q]; break;
      case SENS_SUBTREEANGMOM: subtree_angmom(m, d, id, o); break;
      case SENS_BALLQUAT: {
        if (m.jnt_type[id] != 1) throw std::runtime_error("ballquat of a joint other than a ball joint");
        const int a = m.jnt_qposadr[id];
        double n = 0;
        for (int q = 0; q < 4; q++) n += (double)d.qpos[a + q] * (double)d.qpos[a + q];
        n = std::sqrt(n);
        for (int q = 0; q < 4; q++) o[q] = d.qpos[a + q] / n;
        break;
      }
      case SENS_BALLANGVEL:
        if (m.jnt_type[id] != 1) throw std::runtime_error("ballangvel of a joint other than a ball joint");
        for (int q = 0; q < 3; q++) o[q] = d.qvel[m.jnt_dofadr[id] + q];
        break;
      case SENS_JOINTACTUATORFRC: o[0] = d.qfrc_actuator[m.jnt_dofadr[id]]; break;
      case SENS_ACTUATORFRC: o[0] = d.actuator_force[id]; break;
      case SENS_ACTUATORPOS: case SENS_ACTUATORVEL: {
        const bool vel = tab.type[s] == SENS_ACTUATORVEL;
        const int j = m.actuator_trnid[id];
        double x;
        if (m.actuator_trntype[id] == 1) x = tendon(m, d, j, vel);
        else if (m.actuator_trntype[id] == 0) x = vel ? (double)d.qvel[m.jnt_dofadr[j]] : (double)d.qpos[m.jnt_qposadr[j]];
        else throw std::runtime_error("actuator transmission not evaluated");
        o[0] = (double)m.actuator_gear[id] * x;
        break;
      }
      case SENS_TENDONPOS: o[0] = tendon(m, d, id, false); break;
      case SENS_TENDONVEL: o[0] = tendon(m, d, id, true); break;
      case SENS_MAGNETOMETER: {
        if (tab.objtype[s] != OBJ_SITE) throw std::runtime_error("magnetometer of an object other than a site");
        const T* R = &d.site_xmat[9 * id];
        for (int r = 0; r < 3; r++) {
          T x = 0;
          for (int k = 0; k < 3; k++) x += R[3 * k + r] * (T)tab.magnetic[k];
          o[r] = x;
        }
        break;
      }
      case SENS_RANGEFINDER:
        if (tab.objtype[s] != OBJ_SITE) throw std::runtime_error("rangefinder of an object other than a site");
        o[0] = rangefinder(m, d, tab, id);
        break;
      default: throw std::runtime_error("sensor type not evaluated");
    }
  }
}

template <class T>
int step(Sim<T>& sim, const Table& tab, int B, const double* qpos, const double* qvel, const double* ctrl,
         const double* warmstart, const double* mocap, const double* times, int start, int count, double* next_qpos,
         double* next_qvel, double* qacc, double* sensordata, int* counts, const double* xfrc) {
  const Model<T>& m = sim.model;
  Data<T>& d = sim.data;
  const int nq = m.nq, nv = m.nv, nu = m.nu;
  const int dim = count ? tab.adr[start + count - 1] - tab.adr[start] + tab.dim[start + count - 1] : 0;
  for (int b = 0; b < B; b++) {
    for (int i = 0; i < nq; i++) d.qpos[i] = (T)qpos[(size_t)b * nq + i];
    for (int i = 0; i < nv; i++) d.qvel[i] = (T)qvel[(size_t)b * nv + i];
    for (int i = 0; i < nu; i++) d.ctrl[i] = (T)ctrl[(size_t)b * nu + i];
    for (int i = 0; i < m.nmocap; i++) {
      for (int c = 0; c < 3; c++) d.mocap_pos[3 * i + c] = (T)mocap[7 * i + c];
      for (int c = 0; c < 4; c++) d.mocap_quat[4 * i + c] = (T)mocap[7 * i + 3 + c];
    }
    for (int i = 0; i < nv; i++) d.qacc_warmstart[i] = warmstart ? (T)warmstart[(size_t)b * nv + i] : (T)0;
    std::fill(d.xfrc_applied.begin(), d.xfrc_applied.end(), (T)0);
    d.xfrc_active = xfrc != nullptr;
    if (xfrc) for (int i = 0; i < 6 * m.nbody; i++) d.xfrc_applied[i] = (T)xfrc[(size_t)b * 6 * m.nbody + i];
    d.time = (T)times[b];
    d.warning = false;
    forward<T>(m, d, nullptr);
    if (bad(d.qacc)) d.warning = true;
    if (sensordata) sensors(m, d, tab, start, count, sensordata + (size_t)b * dim);
    if (qacc) for (int i = 0; i < nv; i++) qacc[(size_t)b * nv + i] = d.qacc[i];
    if (counts) { counts[4 * b] = d.ncon; counts[4 * b + 1] = d.nefc; counts[4 * b + 2] = d.solver_niter; counts[4 * b + 3] = d.warning; }
    d.qacc_warmstart = d.qacc;
    euler<T>(m, d);
    if (next_qpos) for (int i = 0; i < nq; i++) next_qpos[(size_t)b * nq + i] = d.qpos[i];
    if (next_qvel) for (int i = 0; i < nv; i++) next_qvel[(size_t)b * nv + i] = d.qvel[i];
  }
  return 0;
}

}  // namespace

extern "C" {

void* sensor_oracle_create(const void* blob, size_t nbytes, int precision) {
  try {
    auto* h = new Handle;
    h->precision = precision;
    BlobReader b(blob, nbytes);
    h->tab.type = b.ints("sensor_type"); h->tab.objtype = b.ints("sensor_objtype"); h->tab.objid = b.ints("sensor_objid");
    h->tab.dim = b.ints("sensor_dim"); h->tab.adr = b.ints("sensor_adr"); h->tab.site_type = b.ints("site_type");
    h->tab.site_size = b.reals("site_size");
    int dt, cnt;
    int64_t off;
    if (b.find("opt_magnetic", &dt, &cnt, &off)) {
      const std::vector<double> mag = b.reals("opt_magnetic");
      for (int q = 0; q < 3; q++) h->tab.magnetic[q] = mag.at(q);
    }
    if (b.find("geom_alpha", &dt, &cnt, &off)) h->tab.geom_alpha = b.reals("geom_alpha");
    if (precision == 64) h->s64.reset(new Sim<double>(blob, nbytes));
    else h->s32.reset(new Sim<float>(blob, nbytes));
    return h;
  } catch (const std::exception&) {
    return nullptr;
  }
}

void sensor_oracle_destroy(void* h) { delete (Handle*)h; }

// B single steps; sensordata [B][dim of sensors start .. start + count); returns 0, or -1 when a sensor in the range
// is not evaluated (type, or a non-sphere touch zone) or the range is outside the model's sensors.  xfrc NULL: no
// applied wrench.
int sensor_oracle_step(void* hv, int B, const double* qpos, const double* qvel, const double* ctrl,
                       const double* warmstart, const double* mocap, const double* times, int start, int count,
                       double* next_qpos, double* next_qvel, double* qacc, double* sensordata, int* counts,
                       const double* xfrc) {
  Handle* h = (Handle*)hv;
  if (start < 0 || count < 0 || start + count > (int)h->tab.type.size()) return -1;
  try {
    if (h->precision == 64)
      return step(*h->s64, h->tab, B, qpos, qvel, ctrl, warmstart, mocap, times, start, count, next_qpos, next_qvel,
                  qacc, sensordata, counts, xfrc);
    return step(*h->s32, h->tab, B, qpos, qvel, ctrl, warmstart, mocap, times, start, count, next_qpos, next_qvel, qacc,
                sensordata, counts, xfrc);
  } catch (const std::exception&) {
    return -1;
  }
}

}  // extern "C"
