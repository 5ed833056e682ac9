// TEST INFRASTRUCTURE - measurement sensors on the CPU oracle (oracle/physics.h), fp64 or fp32.
//
// The same single step as the oracle's step_batch (forward, warning on a bad qacc, warm start from qacc, Euler) plus
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
// The sensor table is read from the blob's sensor_* / site_* entries.  Written from the definition, independently of
// the device's k_sensors; the oracle itself is not modified.
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <vector>

#include "../oracle/physics.h"

using namespace oracle;

namespace {

enum { SENS_FRAMEPOS = 1, SENS_JOINTPOS = 2, SENS_TOUCH = 3, SENS_JOINTVEL = 9, SENS_ACCELEROMETER = 10,
       SENS_VELOCIMETER = 11, SENS_GYRO = 12 };
enum { OBJ_BODY = 0, OBJ_XBODY = 1, OBJ_GEOM = 2, OBJ_SITE = 3 };

struct Table {
  std::vector<int> type, objtype, objid, dim, adr, site_type;
  std::vector<double> site_size;
};

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
      default: throw std::runtime_error("sensor type not evaluated");
    }
  }
}

template <class T>
int step(Sim<T>& sim, const Table& tab, int B, const double* qpos, const double* qvel, const double* ctrl,
         const double* warmstart, const double* mocap, const double* times, int start, int count, double* next_qpos,
         double* next_qvel, double* qacc, double* sensordata, int* counts) {
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
    d.xfrc_active = false;
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
    if (precision == 64) h->s64.reset(new Sim<double>(blob, nbytes));
    else h->s32.reset(new Sim<float>(blob, nbytes));
    return h;
  } catch (const std::exception&) {
    return nullptr;
  }
}

void sensor_oracle_destroy(void* h) { delete (Handle*)h; }

// B single steps; sensordata [B][dim of sensors start .. start + count); returns 0, or -1 when a sensor in the range
// is not evaluated (type, or a non-sphere touch zone) or the range is outside the model's sensors
int sensor_oracle_step(void* hv, int B, const double* qpos, const double* qvel, const double* ctrl,
                       const double* warmstart, const double* mocap, const double* times, int start, int count,
                       double* next_qpos, double* next_qvel, double* qacc, double* sensordata, int* counts) {
  Handle* h = (Handle*)hv;
  if (start < 0 || count < 0 || start + count > (int)h->tab.type.size()) return -1;
  try {
    if (h->precision == 64)
      return step(*h->s64, h->tab, B, qpos, qvel, ctrl, warmstart, mocap, times, start, count, next_qpos, next_qvel,
                  qacc, sensordata, counts);
    return step(*h->s32, h->tab, B, qpos, qvel, ctrl, warmstart, mocap, times, start, count, next_qpos, next_qvel, qacc,
                sensordata, counts);
  } catch (const std::exception&) {
    return -1;
  }
}

}  // extern "C"
