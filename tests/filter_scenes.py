"""An independent fp64 restatement of the Unscented and Kalman filters (the reference's mjpc/estimators/unscented.cc and
kalman.cc, with mju_subQuat, mju_quatIntegrate and mj_integratePos), and the scenes their tests run on.

It is written from the reference's definitions, not from mujoco_mpc_b200/estimator.py or csrc/estimator_kernels.cuh:
  * tangent-space arithmetic through the exponential map of fd_scenes (q (+) v = q exp(v), q1 (-) q0 = log(q0* q1) on
    the shortest arc), positions by joint, velocities added;
  * the Markley quaternion mean as numpy.linalg.eigh's eigenvector of the largest eigenvalue of
    K = sum 4 w_i q_i q_i' - (sum w_i) I (covariance weights), signed to agree with the nominal point's quaternion;
  * every update as the conditioning of a joint Gaussian: (next state, sensors of the pre-step state) with covariance
    [[S_ss + Q, S_sy], [S_ys, S_yy + R]] conditioned on the measurement gives mean (+) S_sy S_yy^-1 (y - y_mean) and
    S_ss - S_sy S_yy^-1 S_ys (unscented.cc: sensordata after mj_step belongs to the pre-step state, :365-390); the
    Kalman measurement conditions (x, C x + noise) the same way, and its prediction is A P A' + Q.
A factorisation fails on a pivot below PIVOT_MIN or one that is not finite, as the device's does.

Scenes (an appended <sensor> block after the particle-copy user sensor of joint_scenes.compile_scene, so the measured
sensors start at index 1):
  * slide: fd_scenes.slide_scene with jointpos and jointvel sensors: linear, so both filters are exact;
  * free_ball: a free body, a motorised slide and a ball joint in zero gravity, whose step is fd_scenes' closed form;
    sensors framepos / framequat of the free body, the slide's jointpos / jointvel and ballquat / ballangvel;
  * hinges(n): n root hinges (nv = n), each measured twice by jointpos and jointvel (ny = 4 n).
"""
import numpy as np

import fd_scenes as FD
import joint_scenes as JS

PIVOT_MIN = 1e-15
SENSOR_START = 1


class FactorError(Exception):
    pass


# --------------------------------------------------------------------------------------------- tangent arithmetic
def joints(m):
    """[(type, qposadr, dofadr)] of model m (0 free, 1 ball, 2 slide, 3 hinge)."""
    return [(int(m.jnt_type[j]), int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])) for j in range(m.njnt)]


def _qexp(q, v):
    out = FD.quat_mul(q, FD.quat_exp(v))
    return out / np.linalg.norm(out)


def _qlog(q1, q0):
    return FD.quat_log(FD.quat_mul(FD.quat_conj(q0), q1) / np.linalg.norm(q1) / np.linalg.norm(q0))


def plus(m, x, dx, scale=1.0):
    """x (+) scale dx for a state x [nq + nv] and tangent dx [2 nv]."""
    nq, nv = m.nq, m.nv
    x = np.array(x, float)
    dx = scale * np.asarray(dx, float)
    out = x.copy()
    for t, a, d in joints(m):
        if t == 0:
            out[a:a + 3] = x[a:a + 3] + dx[d:d + 3]
            out[a + 3:a + 7] = _qexp(x[a + 3:a + 7], dx[d + 3:d + 6])
        elif t == 1:
            out[a:a + 4] = _qexp(x[a:a + 4], dx[d:d + 3])
        else:
            out[a] = x[a] + dx[d]
    out[nq:] = x[nq:] + dx[nv:]
    return out


def minus(m, x1, x0):
    """x1 (-) x0 [2 nv]."""
    nq, nv = m.nq, m.nv
    x1, x0 = np.asarray(x1, float), np.asarray(x0, float)
    out = np.zeros(2 * nv)
    for t, a, d in joints(m):
        if t == 0:
            out[d:d + 3] = x1[a:a + 3] - x0[a:a + 3]
            out[d + 3:d + 6] = _qlog(x1[a + 3:a + 7], x0[a + 3:a + 7])
        elif t == 1:
            out[d:d + 3] = _qlog(x1[a:a + 4], x0[a:a + 4])
        else:
            out[d] = x1[a] - x0[a]
    out[nv:] = x1[nq:] - x0[nq:]
    return out


def quat_slots(m):
    """qpos addresses of every quaternion."""
    return [a + (3 if t == 0 else 0) for t, a, d in joints(m) if t in (0, 1)]


# --------------------------------------------------------------------------------------------- linear algebra
def factor(M):
    """Lower Cholesky factor; FactorError on a pivot below PIVOT_MIN or not finite."""
    M = np.asarray(M, float)
    if not np.all(np.isfinite(M)):
        raise FactorError("not finite")
    n = len(M)
    L = np.zeros_like(M)
    for j in range(n):
        d = M[j, j] - L[j, :j] @ L[j, :j]
        if not (np.isfinite(d) and d >= PIVOT_MIN):
            raise FactorError("pivot %d = %r" % (j, d))
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (M[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def condition(S_ss, S_sy, S_yy, innovation):
    """The Gaussian (s, y) conditioned on y: (tangent correction, covariance).  FactorError when S_yy does not factor."""
    factor(S_yy)
    G = np.linalg.solve(S_yy, S_sy.T).T       # S_sy S_yy^-1
    P = S_ss - G @ S_sy.T
    return G @ innovation, 0.5 * (P + P.T)


def finite_or_raise(*arrays):
    for a in arrays:
        if not np.all(np.isfinite(a)):
            raise FactorError("non-finite result")


# --------------------------------------------------------------------------------------------- Unscented
class UKFWeights:
    def __init__(self, ndstate, alpha, beta=2.0):
        lam = ndstate * (alpha ** 2 - 1.0)
        self.n = ndstate
        self.step = np.sqrt(ndstate + lam)
        self.wm0 = lam / (ndstate + lam)
        self.wc0 = self.wm0 + 1.0 - alpha ** 2 + beta
        self.w = 1.0 / (2.0 * (ndstate + lam))
        self.R = 2 * ndstate + 1

    def vec(self, w0):
        v = np.full(self.R, self.w)
        v[-1] = w0
        return v


def sigma_points(m, x, P, W):
    """[R][nq + nv]: x (+) step L[:, i], then x (+) -step L[:, i], nominal last; FactorError when P does not factor."""
    L = factor(P)
    rows = [plus(m, x, W.step * L[:, i]) for i in range(W.n)] + [plus(m, x, -W.step * L[:, i]) for i in range(W.n)]
    return np.array(rows + [np.array(x, float)])


def quaternion_mean(Q, wc, ref):
    """(mean, the eigenvalues of K ascending) of the quaternions Q [R][4]."""
    K = 4.0 * np.einsum("i,ij,ik->jk", wc, Q, Q) - wc.sum() * np.eye(4)
    lam, V = np.linalg.eigh(K)
    v = V[:, -1] / np.linalg.norm(V[:, -1])
    return (v if v @ ref >= 0 else -v), lam, K


def state_mean(m, nxt, W, quat_override=None):
    mean = W.vec(W.wm0) @ nxt
    wc = W.vec(W.wc0)
    info = {}
    for a in quat_slots(m):
        q, lam, K = quaternion_mean(nxt[:, a:a + 4], wc, nxt[-1, a:a + 4])
        mean[a:a + 4] = q if quat_override is None else quat_override[a:a + 4]
        info[a] = (lam, K)
    return mean, info


def ukf_update(m, W, nxt, ys, y, Q, Rn, quat_override=None):
    """The Unscented update from the stepped rows nxt [R][nq+nv], their pre-step sensors ys [R][ny] and the measurement
    y: (state, covariance, quaternion-mean info).  FactorError on a failed sensor factor or a non-finite result."""
    nxt, ys = np.asarray(nxt, float), np.asarray(ys, float)
    wm, wc = W.vec(W.wm0), W.vec(W.wc0)
    mean, info = state_mean(m, nxt, W, quat_override)
    ymean = wm @ ys
    ds = np.array([minus(m, r, mean) for r in nxt])
    dy = ys - ymean
    S_ss = np.diag(Q) + (ds.T * wc) @ ds
    S_sy = (ds.T * wc) @ dy
    S_yy = np.diag(Rn) + (dy.T * wc) @ dy
    corr, P = condition(S_ss, S_sy, S_yy, np.asarray(y, float) - ymean)
    x = plus(m, mean, corr)
    finite_or_raise(x, P)
    return x, P, info


# --------------------------------------------------------------------------------------------- Kalman
def kalman_rows(m, x, eps, centered):
    n = 2 * m.nv
    rows = [np.array(x, float)]
    for s in ([1.0, -1.0] if centered else [1.0]):
        for i in range(n):
            e = np.zeros(n)
            e[i] = s * eps
            rows.append(plus(m, x, e))
    return np.array(rows)


def kalman_measurement(m, x, P, ys, y, Rn, eps, centered):
    """(state, covariance) from the sensors ys [rows][ny] of kalman_rows."""
    n = 2 * m.nv
    ys = np.asarray(ys, float)
    h = 2 * eps if centered else eps
    C = np.stack([(ys[1 + i] - (ys[1 + n + i] if centered else ys[0])) / h for i in range(n)], axis=1)
    PCt = P @ C.T
    corr, Pn = condition(P, PCt, C @ PCt + np.diag(Rn), np.asarray(y, float) - ys[0])
    xn = plus(m, x, corr)
    finite_or_raise(xn, Pn)
    return xn, Pn


def kalman_prediction(m, P, nxt, Q, eps, centered):
    """(state, covariance) from the next states nxt [rows][nq+nv] of kalman_rows."""
    n = 2 * m.nv
    nxt = np.asarray(nxt, float)
    h = 2 * eps if centered else eps
    A = np.stack([minus(m, nxt[1 + i], nxt[1 + n + i] if centered else nxt[0]) / h for i in range(n)], axis=1)
    Pn = A @ P @ A.T + np.diag(Q)
    Pn = 0.5 * (Pn + Pn.T)
    finite_or_raise(nxt[0], Pn)
    return nxt[0].copy(), Pn


# --------------------------------------------------------------------------------------------- scenes
def _compile(text, sensors):
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.mjcf import compile_xml
    m0 = compile_xml(text.replace("{sensor}", ""))
    dim = m0.nq + m0.nv
    block = f'<sensor><user name="State" dim="{dim}" user="0 1 0 1"/>{"".join(sensors)}</sensor>'
    m = compile_xml(text.replace("{sensor}", block))
    m.task_residual_id = T.RESIDUAL_PARTICLE_COPY
    m.task_ids, m.task_state, m.ray_geoms = np.zeros(1, np.int32), np.zeros(1), np.zeros(0, np.int32)
    return m


class FilterScene:
    """A compiled model with measured sensors [SENSOR_START, SENSOR_START + nsensor), its fd_scenes step, a measurement
    function h(x) of the pre-step state and a nominal state."""

    def __init__(self, name, fd, sensors, h, x0):
        self.name, self.fd, self.h, self.x0 = name, fd, h, np.asarray(x0, float)
        self.m = _compile(fd.text(), sensors)
        self.nsensor = len(sensors)
        self.ny = len(h(self.x0))

    def step(self, x, u):
        m = self.m
        q, v = self.fd.step(np.asarray(x[:m.nq], float), np.asarray(x[m.nq:], float), np.asarray(u, float))
        return np.concatenate([q, v])


def slide():
    fd = FD.slide_scene()
    sensors = ['<jointpos joint="j0"/>', '<jointpos joint="j1"/>', '<jointvel joint="j0"/>', '<jointvel joint="j1"/>']
    return FilterScene("slide", fd, sensors, lambda x: np.asarray(x, float)[[0, 1, 2, 3]], fd.x)


def slide_linear_model(sc):
    """(F, G, H, c) of the slide: x' = F x + G u + c, y = H x (closed form, fd_scenes)."""
    F, Gm, _, _ = sc.fd.jacobians()
    x0, u0 = np.zeros(4), np.zeros(2)
    c = sc.step(x0, u0)
    return F, Gm, np.eye(4), c


def free_ball():
    bodies = [FD.Body("free", m=1.0, r=0.1), FD.Body("slide", m=1.0), FD.Body("ball", m=2.0, r=0.2)]
    q = np.concatenate([[0.1, 0.2, 1.0], JS.QROT, [0.05], FD.quat_mul(JS.QROT, FD.quat_exp(np.array([0.3, -0.2, 0.5])))])
    v = np.concatenate([[0.3, -0.2, 0.1], FD.W_ROT, [0.2], -0.8 * FD.W_ROT])
    fd = FD.FdScene("filter_free_ball", bodies, [FD.Motor(1, gear=1.0)], q, v, [0.4], gravity=False)
    sensors = ['<framepos objtype="xbody" objname="b0"/>', '<framequat objtype="xbody" objname="b0"/>',
               '<jointpos joint="j1"/>', '<jointvel joint="j1"/>', '<ballquat joint="j2"/>', '<ballangvel joint="j2"/>']

    def h(x):
        x = np.asarray(x, float)
        qf, qb = x[3:7] / np.linalg.norm(x[3:7]), x[8:12] / np.linalg.norm(x[8:12])
        return np.concatenate([x[0:3], qf, [x[7]], [x[12 + 6]], qb, x[12 + 7:12 + 10]])
    return FilterScene("free_ball", fd, sensors, h, np.concatenate([q, v]))


def hinges(n=34):
    bodies = [FD.Body("hinge", m=1.0 + 0.01 * k, r=0.05, axis="1 0 0", damping=0.1) for k in range(n)]
    fd = FD.FdScene("filter_hinges", bodies, [FD.Motor(0, gear=1.0)], 0.01 * np.arange(n), np.zeros(n), [0.0],
                    gravity=False)
    sensors = ([f'<jointpos joint="j{k}"/>' for k in range(n)] + [f'<jointvel joint="j{k}"/>' for k in range(n)]) * 2
    return FilterScene("hinges", fd, sensors, lambda x: np.concatenate([x, x]), fd.x)
