"""MJPC's Unscented (mjpc/estimators/unscented.cc) and Kalman (mjpc/estimators/kalman.cc) state estimators with their
steps on a step backend.  Both derive from ``_Filter`` (the reference's Estimator base), and their C++ wrappers from
``_CppFilter``.

The filter arithmetic is double precision on the host: a Cholesky factor of the covariance, weighted means and
covariances of at most 2 ndstate + 1 points and one Cholesky factor of the sensor covariance.  The sigma-point steps
(one mj_step per point, EvaluateSigmaPoints, unscented.cc:353-394) are what costs: the backend runs them all in one
call.  ``EngineBackend`` runs them as one launch of the CUDA engine (``Engine.step_sensors``); anything with the same
``step_sensors`` method can stand in for it.

Reference semantics restated (unscented.cc):
  settings      :31-168, Reset :171-290 (every setting through GetNumberOrDefault)
  SigmaPoints   :293-349   lower Cholesky factor L of P; point i = x (+) step L[:, i], point i + ndstate = x (-) step
                           L[:, i] (positions through mj_integratePos, velocities added); the nominal state is LAST
  Evaluate      :353-394   every point steps from the same time and ctrl; y_i = h(sigma_i) (sensors of the pre-step
                           state, after the constraint solve), s_i = f(sigma_i); means weight the last point w_mean0
  QuaternionMean:578-626   per free / ball joint the principal eigenvector of sum 4 w q q^T - (sum w) I, with the
                           COVARIANCE weights (as the reference does)
  Differences / Covariances / Update :397-574

Documented differences from the reference:
  * a failed factorisation (covariance or sensor covariance) raises ``EstimatorError`` naming the factor and leaves
    state, covariance and time untouched (the reference calls mju_error).  A factorisation fails on a pivot below
    CHOL_MIN_PIVOT or one that is not finite (the reference's mju_cholFactor(.., 0) accepts pivots >= 0);
  * an update whose new state or covariance would not be finite raises ``EstimatorError`` ("non-finite result") and
    leaves the filter untouched;
  * every sigma point warm-starts the constraint solver from the nominal point's qacc of the previous update (zeros
    after reset); the reference reuses one mjData, so each point starts from the previous point's qacc.  The Newton
    solution is unique to the solver tolerance, so this changes results only at that level;
  * ``update`` takes mocap (default: the model's), the reference's mjData keeps the model's;
  * ``update`` takes the measured slice [nsensordata] of the sensors, not the whole sensordata.

The Kalman filter (``Kalman``, kalman.cc) linearises by finite differences instead: the centre state and its
tangent-space perturbations x (+) eps e_i (then x (+) -eps e_i when centred) are one backend call per Jacobian, the
sensor Jacobian C from the pre-step sensors at the current state (UpdateMeasurement, :188-276), the dynamics Jacobian A
from the next states at the corrected state (UpdatePrediction, :279-323).  Its documented differences from the
reference are the Unscented filter's (the warm start is the centre state's qacc of the previous call), plus:
  * a failed sensor-covariance factorisation raises ``EstimatorError`` and leaves state, covariance and time untouched;
  * ``update_prediction`` uses the ctrl and mocap of the last measurement, as the reference's mjData does;
  * time: both calls run at ``time`` and ``update_prediction`` advances it by the timestep (the reference leaves its
    ``time`` member alone and its mjData's clock advances inside mj_step);
  * the finite differences default to KALMAN_CENTERED with KALMAN_EPSILON: the reference's 1e-6 one-sided is an fp64
    setting, and the engine steps in fp32 (DESIGN.md, "Kalman filter", has the sweep that chose them).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from .engine import EngineError, _CppObject, _d, _model_blobs, _pd, _pf
from .mjcf import JNT_BALL, JNT_FREE, SENS_MEASURED


class EstimatorError(RuntimeError):
    pass


CHOL_MIN_PIVOT = 1e-15   # the device factorisation's pivot threshold (csrc/estimator_kernels.cuh fb_chol_factor)


def cholesky(M, what):
    """Lower Cholesky factor of M; EstimatorError naming `what` when a pivot M_jj - sum_k<j L_jk^2 is below
    CHOL_MIN_PIVOT or any entry is not finite (LAPACK accepts any positive pivot and may return a NaN factor without
    raising)."""
    try:
        L = np.linalg.cholesky(M)
    except np.linalg.LinAlgError:
        L = None
    if L is None or not np.all(np.isfinite(L)) or \
            not np.all(np.diag(M) - np.sum(np.tril(L, -1) ** 2, axis=1) >= CHOL_MIN_PIVOT):
        raise EstimatorError(what + " factorisation failed")
    return L


def _finite_result(state, covariance):
    """(state, covariance), or EstimatorError when either is not finite (the filter then keeps what it had)."""
    if not (np.all(np.isfinite(state)) and np.all(np.isfinite(covariance))):
        raise EstimatorError("non-finite result (state or covariance)")
    return state, covariance


def _number(m, name, default):
    """GetNumberOrDefault (utilities.cc): the model's custom numeric `name`, else `default`."""
    v = m.numeric.get(name) if hasattr(m, "numeric") else None
    return float(v[0]) if v is not None and len(v) else default


# ------------------------------------------------------------------------------------------- quaternions / positions
def _quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
                     a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat_integrate(q, v, scale):
    """mju_quatIntegrate: q * exp(scale v / 2), normalised."""
    w = np.asarray(v, float) * scale
    a = np.linalg.norm(w)
    if a < 1e-15:
        return np.asarray(q, float) / np.linalg.norm(q)
    r = np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * w / a])
    out = _quat_mul(q, r)
    return out / np.linalg.norm(out)


def quat_sub(qa, qb):
    """mju_subQuat: the 3-vector v with qb * exp(v / 2) = qa (shortest arc)."""
    qb_inv = np.array([qb[0], -qb[1], -qb[2], -qb[3]])
    d = _quat_mul(qb_inv, qa)
    d = d / np.linalg.norm(d)
    if d[0] < 0:
        d = -d
    s = np.linalg.norm(d[1:])
    if s < 1e-15:
        return np.zeros(3)
    return 2 * np.arctan2(s, d[0]) * d[1:] / s


def integrate_pos(m, qpos, dq, scale=1.0):
    """mj_integratePos: qpos (+) scale dq, quaternions in the tangent space."""
    q = np.array(qpos, float)
    for j in range(m.njnt):
        a, d, t = m.jnt_qposadr[j], m.jnt_dofadr[j], m.jnt_type[j]
        if t == JNT_FREE:
            q[a:a + 3] += scale * dq[d:d + 3]
            q[a + 3:a + 7] = quat_integrate(q[a + 3:a + 7], dq[d + 3:d + 6], scale)
        elif t == JNT_BALL:
            q[a:a + 4] = quat_integrate(q[a:a + 4], dq[d:d + 3], scale)
        else:
            q[a] += scale * dq[d]
    return q


def differentiate_pos(m, q1, q2):
    """mj_differentiatePos with dt = 1: the tangent vector from q1 to q2."""
    out = np.zeros(m.nv)
    for j in range(m.njnt):
        a, d, t = m.jnt_qposadr[j], m.jnt_dofadr[j], m.jnt_type[j]
        if t == JNT_FREE:
            out[d:d + 3] = q2[a:a + 3] - q1[a:a + 3]
            out[d + 3:d + 6] = quat_sub(q2[a + 3:a + 7], q1[a + 3:a + 7])
        elif t == JNT_BALL:
            out[d:d + 3] = quat_sub(q2[a:a + 4], q1[a:a + 4])
        else:
            out[d] = q2[a] - q1[a]
    return out


def principal_eigenvector4(K, reference):
    """Principal eigenvector of a symmetric 4 x 4 matrix by cyclic Jacobi rotations, converged to rounding, with the
    sign that agrees with `reference` (stands for PrincipalEigenVector4, utilities.cc:1476+; the device filters run
    the same rotations)."""
    A = np.array(K, float)
    V = np.eye(4)
    for _ in range(50):
        if sum(A[p, q] ** 2 for p in range(4) for q in range(p + 1, 4)) < 1e-300:
            break
        for p in range(4):
            for q in range(p + 1, 4):
                if A[p, q] == 0:
                    continue
                th = (float(A[q, q]) - float(A[p, p])) / (2 * float(A[p, q]))
                t = 0.5 / th if abs(th) > 1e150 else (1.0 if th >= 0 else -1.0) / (abs(th) + np.sqrt(th * th + 1))
                c = 1 / np.sqrt(t * t + 1)
                s = t * c
                J = np.eye(4)
                J[p, p] = J[q, q] = c
                J[p, q], J[q, p] = s, -s
                A = J.T @ A @ J
                V = V @ J
    v = V[:, int(np.argmax(np.diag(A)))]
    v = v / np.linalg.norm(v)
    return v if np.dot(v, reference) >= 0 else -v


def quaternion_mean(quats, weights, reference):
    """Principal eigenvector of K = sum 4 w_i q_i q_i^T - (sum w) I (QuaternionMeans, unscented.cc:578-626), with the
    sign that agrees with `reference` (the nominal point's quaternion)."""
    Q = np.asarray(quats, float)
    w = np.asarray(weights, float)
    K = 4.0 * np.einsum("i,ij,ik->jk", w, Q, Q) - w.sum() * np.eye(4)
    return principal_eigenvector4(K, reference)


# ------------------------------------------------------------------------------------------------------- backends
class EngineBackend:
    """The sigma-point (Unscented) or finite-difference (Kalman) steps as one launch of the CUDA engine
    (mjpc_b200_step_sensors)."""

    def __init__(self, engine, sensor_start, nsensor, timestep):
        self.engine, self.sensor_start, self.nsensor = engine, int(sensor_start), int(nsensor)
        engine.set_options(timestep)   # the estimator's own timestep (estimator_timestep), as Reset sets it

    def step_sensors(self, states, ctrl, mocap, time, warmstart):
        o = self.engine.step_sensors(states, ctrl, mocap, time, self.sensor_start, self.nsensor, warmstart=warmstart)
        return (o["next_states"].astype(float), o["sensordata"].astype(float), o["qacc"].astype(float),
                int(np.count_nonzero(o["warning"])))

    @property
    def last_kernel_ms(self):
        return self.engine.last_kernel_ms


def measured_range(m, sensor_start, nsensor):
    """Check that sensors [sensor_start, sensor_start + nsensor) are ones the measurement path evaluates; returns the
    dimension of their sensordata slice."""
    if sensor_start < 0 or nsensor < 1 or sensor_start + nsensor > m.nsensor:
        raise EstimatorError("sensor range [%d, %d) outside the model's %d sensors"
                             % (sensor_start, sensor_start + nsensor, m.nsensor))
    for i in range(sensor_start, sensor_start + nsensor):
        if int(m.sensor_type[i]) not in SENS_MEASURED:
            raise EstimatorError("sensor %d (%s) is not a measured sensor type (jointpos, jointvel, touch, the frame, "
                                 "subtree, IMU, magnetometer, rangefinder, ball-joint, actuator and tendon sensors)" % (i, m.sensor_names[i]))
        if float(m.sensor_cutoff[i]) != 0.0:
            raise EstimatorError("sensor %d (%s): cutoff is not modelled" % (i, m.sensor_names[i]))
    return int(np.sum(m.sensor_dim[sensor_start:sensor_start + nsensor]))


# ------------------------------------------------------------------------------------------------------- the filter
def settings(m, sensor_start=None, nsensor=None, timestep=None, alpha=None, beta=None):
    """The filter settings, each left None defaulting from the model's numerics as GetNumberOrDefault does
    (unscented.cc:31-168): (sensor_start, nsensor, timestep, alpha, beta)."""
    return (int(_number(m, "estimator_sensor_start", 0) if sensor_start is None else sensor_start),
            int(_number(m, "estimator_number_sensor", m.nsensor) if nsensor is None else nsensor),
            float(_number(m, "estimator_timestep", float(m.opt_timestep)) if timestep is None else timestep),
            float(_number(m, "unscented_alpha", 1.0) if alpha is None else alpha),
            float(_number(m, "unscented_beta", 2.0) if beta is None else beta))


def reset_values(m, state=None, covariance_scale=None, process_scale=None, sensor_scale=None):
    """Reset's state (the home keyframe if the model has one, else qpos0 and zero qvel) and noise scales."""
    if state is None:
        if m.nkey and "home" in m.key_names:
            k = m.key_names.index("home")
            state = np.concatenate([m.key_qpos[k], m.key_qvel[k]])
        else:
            state = np.concatenate([m.qpos0, np.zeros(m.nv)])
    cs = _number(m, "estimator_covariance_initial_scale", 1e-4) if covariance_scale is None else covariance_scale
    ps = _number(m, "estimator_process_noise_scale", 1e-4) if process_scale is None else process_scale
    ss = _number(m, "estimator_sensor_noise_scale", 1e-4) if sensor_scale is None else sensor_scale
    return np.array(state, float), float(cs), float(ps), float(ss)


def _default_mocap(m):
    return np.concatenate([m.mocap_pos0, m.mocap_quat0], axis=1).reshape(-1) if m.nmocap else np.zeros(0)


class _Filter:
    """What the Unscented and Kalman filters share: the settings, sensor range and backend, reset, the noise, the
    warm-started backend step and its commit, the gain update and the tangent-space state addition."""

    def __init__(self, m, backend, sensor_start, nsensor, timestep):
        self.m = m
        self.sensor_start, self.nsensor, self.timestep = settings(m, sensor_start, nsensor, timestep)[:3]
        self.nsensordata = measured_range(m, self.sensor_start, self.nsensor)
        self.backend = backend(self.sensor_start, self.nsensor, self.timestep)
        self.ndstate = 2 * m.nv
        self.warnings = 0

    def reset(self, state=None, time=0.0, covariance_scale=None, process_scale=None, sensor_scale=None):
        """Reset: state = the home keyframe if the model has one, else qpos0 and zero qvel."""
        self.state, cs, ps, ss = reset_values(self.m, state, covariance_scale, process_scale, sensor_scale)
        self.time = float(time)
        self.covariance = cs * np.eye(self.ndstate)
        self.noise_process = np.full(self.ndstate, float(ps))
        self.noise_sensor = np.full(self.nsensordata, float(ss))
        self.qacc_warmstart = np.zeros(self.m.nv)
        self.warnings = 0

    def set_noise(self, process=None, sensor=None):
        """Diagonal process [ndstate] / sensor [nsensordata] noise; None keeps one."""
        if process is not None:
            self.noise_process = np.array(process, float)
        if sensor is not None:
            self.noise_sensor = np.array(sensor, float)

    def _step(self, states, ctrl, mocap):
        """One backend call: every state from `time`, ctrl and mocap, warm-started from the committed qacc."""
        warm = np.tile(self.qacc_warmstart, (len(states), 1))
        return self.backend.step_sensors(states, np.asarray(ctrl, float), mocap, self.time, warm)

    def _commit(self, qacc, nwarn):
        """After a successful update: the warm start from the centre's qacc and the call's warnings."""
        self.qacc_warmstart = qacc.copy()
        self.warnings += nwarn

    @staticmethod
    def _gain(X, S, P0, innovation):
        """(X S^-1 innovation, the symmetrised P0 - X S^-1 X'); EstimatorError when S does not factor."""
        L = cholesky(S, "sensor covariance")
        solve = lambda b: np.linalg.solve(L.T, np.linalg.solve(L, b))
        P = P0 - X @ solve(X.T)
        return X @ solve(innovation), 0.5 * (P + P.T)

    def _state_add(self, x, dx):
        """x (+) dx: positions through mj_integratePos, velocities added."""
        nq, nv = self.m.nq, self.m.nv
        new = np.empty_like(x)
        new[:nq] = integrate_pos(self.m, x[:nq], dx[:nv], 1.0)
        new[nq:] = x[nq:] + dx[nv:]
        return new


class Unscented(_Filter):
    """mjpc::Unscented.  `backend(sensor_start, nsensor, timestep)` returns the object that runs the sigma-point steps (see
    EngineBackend); settings left None default from the model's numerics as GetNumberOrDefault does."""

    def __init__(self, m, backend, sensor_start=None, nsensor=None, timestep=None, alpha=None, beta=None):
        super().__init__(m, backend, sensor_start, nsensor, timestep)
        self.alpha, self.beta = settings(m, alpha=alpha, beta=beta)[3:]
        self.nsigma = 2 * self.ndstate + 1
        # derived weights (unscented.cc:171-290)
        lam = self.ndstate * (self.alpha ** 2 - 1.0)
        self.sigma_step = np.sqrt(self.ndstate + lam)
        self.weight_mean0 = lam / (self.ndstate + lam)
        self.weight_covariance0 = self.weight_mean0 + 1.0 - self.alpha ** 2 + self.beta
        self.weight_sigma = 1.0 / (2.0 * (self.ndstate + lam))
        self.reset()

    def sigma_points(self):
        """SigmaPoints (unscented.cc:293-349): [nsigma][nq+nv], nominal last."""
        m = self.m
        nq, nv = m.nq, m.nv
        L = cholesky(self.covariance, "covariance")
        pts = np.zeros((self.nsigma, nq + nv))
        pts[-1] = self.state
        for i in range(self.ndstate):
            col = self.sigma_step * L[:, i]
            pts[i, :nq] = integrate_pos(m, self.state[:nq], col[:nv], 1.0)
            pts[i, nq:] = self.state[nq:] + col[nv:]
            pts[i + self.ndstate, :nq] = integrate_pos(m, self.state[:nq], col[:nv], -1.0)
            pts[i + self.ndstate, nq:] = self.state[nq:] - col[nv:]
        return pts

    def _weights(self, w0):
        w = np.full(self.nsigma, self.weight_sigma)
        w[-1] = w0
        return w

    def state_mean(self, states):
        """Weighted mean of the stepped states, quaternions by QuaternionMeans."""
        m = self.m
        mean = self._weights(self.weight_mean0) @ states
        wc = self._weights(self.weight_covariance0)
        for j in range(m.njnt):
            if m.jnt_type[j] in (JNT_FREE, JNT_BALL):
                a = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == JNT_FREE else 0)
                mean[a:a + 4] = quaternion_mean(states[:, a:a + 4], wc, states[-1, a:a + 4])
        return mean

    def update(self, ctrl, sensor, mocap=None):
        """One filter update from the measured sensor slice [nsensordata]; advances time by the timestep."""
        m = self.m
        nq, nv = m.nq, m.nv
        if mocap is None:
            mocap = _default_mocap(m)
        states, sensors, qacc, nwarn = self._step(self.sigma_points(), ctrl, mocap)
        wm = self._weights(self.weight_mean0)
        wc = self._weights(self.weight_covariance0)
        s_mean = self.state_mean(states)
        y_mean = wm @ sensors
        ds = np.zeros((self.nsigma, self.ndstate))
        for i in range(self.nsigma):
            ds[i, :nv] = differentiate_pos(m, s_mean[:nq], states[i, :nq])
            ds[i, nv:] = states[i, nq:] - s_mean[nq:]
        dy = sensors - y_mean
        cov_yy = np.diag(self.noise_sensor) + (dy.T * wc) @ dy
        cov_sy = (ds.T * wc) @ dy
        cov_ss = np.diag(self.noise_process) + (ds.T * wc) @ ds
        corr, P = self._gain(cov_sy, cov_yy, cov_ss, np.asarray(sensor, float) - y_mean)
        self.state, self.covariance = _finite_result(self._state_add(s_mean, corr), P)
        self.time = self.time + self.timestep
        self._commit(qacc[-1], nwarn)
        return self.state


def _get_filter(f, get):
    """(state, covariance, time, scalars) of the C++ filter object f, read by get(state, covariance, time, scalars)."""
    x, P = np.zeros(f.m.nq + f.m.nv), np.zeros((f.ndstate, f.ndstate))
    t, sc = C.c_double(), np.zeros(f._nscalars)
    f._check(get(_pd(x), _pd(P), C.byref(t), _pd(sc)))
    return x, P, t.value, sc


class _CppFilter(_CppObject):
    """What CppUnscented and CppKalman share: the C++ filter behind the generic mjpc_b200_estimator_* entry points (its
    reset, noise, set, update and get), the ctrl / sensor / mocap marshalling and the EstimatorError of a failed
    factorisation."""

    def close(self):
        if getattr(self, "h", None):
            self.lib.mjpc_b200_estimator_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.mjpc_b200_estimator_last_error(self.h).decode()
            if "factorisation" in msg or "non-finite result" in msg:
                raise EstimatorError(msg)
            raise EngineError(f"{self._prefix} error {rc}: {msg}")

    def reset(self, state=None, time=0.0, covariance_scale=None, process_scale=None, sensor_scale=None):
        x, cs, ps, ss = reset_values(self.m, state, covariance_scale, process_scale, sensor_scale)
        self._check(self.lib.mjpc_b200_estimator_reset(self.h, _pd(_d(x)), time, cs, ps, ss))

    def set_noise(self, process=None, sensor=None):
        self._check(self.lib.mjpc_b200_estimator_set_noise(self.h, _pd(_d(process)), _pd(_d(sensor))))

    def set(self, state, covariance, time):
        self._check(self.lib.mjpc_b200_estimator_set(self.h, _pd(_d(state)), _pd(_d(covariance)), time))

    def update(self, ctrl, sensor, mocap=None):
        self._check(self.lib.mjpc_b200_estimator_update(self.h, *self._args(ctrl, sensor, mocap)))
        return self.state

    def _args(self, ctrl, sensor, mocap):
        mc = None if mocap is None or len(mocap) == 0 else np.ascontiguousarray(mocap, np.float32)
        u = np.ascontiguousarray(np.atleast_1d(np.asarray(ctrl, float)))
        y = np.ascontiguousarray(sensor, np.float64)
        self._keep = (u, y, mc)
        return _pd(u), _pd(y), _pf(mc)

    def _get(self):
        return _get_filter(self, functools.partial(self.lib.mjpc_b200_estimator_get, self.h))

    @property
    def state(self):
        return self._get()[0]

    @property
    def covariance(self):
        return self._get()[1]

    @property
    def time(self):
        return self._get()[2]

    @property
    def warnings(self):
        return int(self._get()[3][3])


class CppUnscented(_CppFilter):
    """The C++ filter (mjpc_b200_unscented_create: csrc/host/estimator.{h,cc}, a one-filter bank whose arithmetic runs
    on the device) behind the same attributes as Unscented; settings resolve from the model's numerics exactly as
    Unscented's do."""
    _nscalars = 5

    def __init__(self, m, sensor_start=None, nsensor=None, timestep=None, alpha=None, beta=None, device=0):
        self.sensor_start, self.nsensor, self.timestep, self.alpha, self.beta = settings(m, sensor_start, nsensor,
                                                                                         timestep, alpha, beta)
        self.nsensordata = measured_range(m, self.sensor_start, self.nsensor)
        self._create("mjpc_b200_unscented", m, self.sensor_start, self.nsensor, C.c_double(self.timestep),
                     C.c_double(self.alpha), C.c_double(self.beta), int(device))
        self.ndstate, self.nsigma = 2 * m.nv, 4 * m.nv + 1
        self.reset()


# ------------------------------------------------------------------------------------------------------ Kalman
KALMAN_EPSILON = 1e-3    # the engine's finite differences (profiles/kalman_epsilon_sweep.py, DESIGN.md)
KALMAN_CENTERED = True


class Kalman(_Filter):
    """mjpc::Kalman.  `backend(sensor_start, nsensor, timestep)` returns the object that runs the steps (see
    EngineBackend); settings left None default from the model's numerics as GetNumberOrDefault does."""

    def __init__(self, m, backend, sensor_start=None, nsensor=None, timestep=None, epsilon=KALMAN_EPSILON,
                 centered=KALMAN_CENTERED):
        super().__init__(m, backend, sensor_start, nsensor, timestep)
        self.epsilon, self.centered = float(epsilon), bool(centered)
        self.nstates = (2 if self.centered else 1) * self.ndstate + 1
        self.reset()

    def reset(self, state=None, time=0.0, covariance_scale=None, process_scale=None, sensor_scale=None):
        """Reset (kalman.cc:113-185), and the ctrl and mocap of the last measurement = zeros and the model's mocap."""
        super().reset(state, time, covariance_scale, process_scale, sensor_scale)
        self.ctrl, self.mocap = np.zeros(self.m.nu), _default_mocap(self.m)

    def perturbed(self):
        """[nstates][nq+nv]: the state, then x (+) eps e_i for i < ndstate, then (centred) x (+) -eps e_i; positions
        through mj_integratePos, as mjd_transitionFD perturbs them."""
        m = self.m
        nq, nv, n = m.nq, m.nv, self.ndstate
        X = np.tile(self.state, (self.nstates, 1))
        for r in range(1, self.nstates):
            i, e = (r - 1) % n, self.epsilon if r - 1 < n else -self.epsilon
            if i < nv:
                d = np.zeros(nv)
                d[i] = 1.0
                X[r, :nq] = integrate_pos(m, self.state[:nq], d, e)
            else:
                X[r, nq + i - nv] += e
        return X

    def _column(self, plus, r):
        """Finite-difference column r of a Jacobian from the rows [nstates][...] of one step (difference `plus`)."""
        n, h = self.ndstate, (2 * self.epsilon if self.centered else self.epsilon)
        return plus(r + 1, r + 1 + n if self.centered else 0) / h

    def update_measurement(self, ctrl, sensor, mocap=None):
        """UpdateMeasurement (kalman.cc:188-276) from the measured sensor slice [nsensordata]."""
        mocap = _default_mocap(self.m) if mocap is None else np.asarray(mocap, float)
        nxt, y, qacc, nwarn = self._step(self.perturbed(), ctrl, mocap)
        C = np.stack([self._column(lambda a, b: y[a] - y[b], i) for i in range(self.ndstate)], axis=1)
        P = self.covariance
        PCt = P @ C.T
        S = C @ PCt + np.diag(self.noise_sensor)
        corr, Pn = self._gain(PCt, S, P, np.asarray(sensor, float) - y[0])
        self.state, self.covariance = _finite_result(self._state_add(self.state, corr), Pn)
        self.ctrl, self.mocap = np.atleast_1d(np.asarray(ctrl, float)).copy(), mocap
        self._commit(qacc[0], nwarn)
        return self.state

    def update_prediction(self):
        """UpdatePrediction (kalman.cc:279-323) with the ctrl and mocap of the last measurement; advances time."""
        m = self.m
        nq = m.nq
        nxt, _, qacc, nwarn = self._step(self.perturbed(), self.ctrl, self.mocap)

        def diff(a, b):
            return np.concatenate([differentiate_pos(m, nxt[b, :nq], nxt[a, :nq]), nxt[a, nq:] - nxt[b, nq:]])
        A = np.stack([self._column(diff, i) for i in range(self.ndstate)], axis=1)
        P = A @ self.covariance @ A.T + np.diag(self.noise_process)
        self.state, self.covariance = _finite_result(nxt[0].copy(), 0.5 * (P + P.T))
        self.time = self.time + self.timestep
        self._commit(qacc[0], nwarn)
        return self.state

    def update(self, ctrl, sensor, mocap=None):
        """update_measurement, then update_prediction: the state predicted for the next step."""
        self.update_measurement(ctrl, sensor, mocap)
        return self.update_prediction()


class CppKalman(_CppFilter):
    """The C++ filter (mjpc_b200_kalman_*: csrc/host/estimator.{h,cc}, a one-filter bank whose arithmetic runs on the
    device) behind the same attributes as Kalman; settings resolve from the model's numerics exactly as Kalman's do.
    update is the generic one: the measurement, then the prediction."""
    _nscalars = 6

    def __init__(self, m, sensor_start=None, nsensor=None, timestep=None, epsilon=KALMAN_EPSILON,
                 centered=KALMAN_CENTERED, device=0):
        self.sensor_start, self.nsensor, self.timestep = settings(m, sensor_start, nsensor, timestep)[:3]
        self.nsensordata = measured_range(m, self.sensor_start, self.nsensor)
        self.epsilon, self.centered = float(epsilon), bool(centered)
        self._create("mjpc_b200_kalman", m, self.sensor_start, self.nsensor, C.c_double(self.timestep),
                     C.c_double(self.epsilon), int(self.centered), int(device))
        self.ndstate = 2 * m.nv
        self.nstates = (2 if self.centered else 1) * self.ndstate + 1
        self.reset()

    def update_measurement(self, ctrl, sensor, mocap=None):
        self._check(self.lib.mjpc_b200_kalman_update_measurement(self.h, *self._args(ctrl, sensor, mocap)))
        return self.state

    def update_prediction(self):
        self._check(self.lib.mjpc_b200_kalman_update_prediction(self.h))
        return self.state


# ------------------------------------------------------------------------------------------------------ batched
class CppBatchEstimator(_CppObject):
    """num_filters independent filters of one kind on one engine handle, every update on the device
    (csrc/host/estimator.{h,cc}, mjpc_b200_batch_estimator_*).  kind: "kalman" or "unscented"; settings resolve
    from the model's numerics exactly as CppKalman's / CppUnscented's do.  Each filter starts as reset() leaves it.
    update returns the per-filter status (0, or MJPC_B200_ERR_BAD_ARGUMENT = -1 where a factorisation failed and the
    filter was left as it was); state / covariance / time / warnings take the filter index."""
    KINDS = {"kalman": 1, "unscented": 2}

    def __init__(self, m, kind, num_filters, sensor_start=None, nsensor=None, timestep=None, alpha=None, beta=None,
                 epsilon=KALMAN_EPSILON, centered=KALMAN_CENTERED, device=0):
        if kind not in self.KINDS:
            raise ValueError("kind must be one of %s" % sorted(self.KINDS))
        self.kind, self.num_filters = kind, int(num_filters)
        self.sensor_start, self.nsensor, self.timestep, self.alpha, self.beta = settings(m, sensor_start, nsensor,
                                                                                         timestep, alpha, beta)
        self.nsensordata = measured_range(m, self.sensor_start, self.nsensor)
        self.epsilon, self.centered = float(epsilon), bool(centered)
        self.ndstate = 2 * m.nv
        if kind == "unscented":
            prm, self._nscalars = (self.alpha, self.beta), 5
            self.rows = 2 * self.ndstate + 1
        else:
            prm, self._nscalars = (self.epsilon, float(self.centered)), 6
            self.rows = (2 if self.centered else 1) * self.ndstate + 1
        self._settings = np.array(prm, float)
        self._create("mjpc_b200_batch_estimator", m, self.KINDS[kind], self.num_filters, self.sensor_start,
                     self.nsensor, C.c_double(self.timestep), _pd(self._settings), int(device))
        for b in range(self.num_filters):
            self.reset(b)

    def _check(self, rc):
        if rc != 0:
            raise EngineError(f"{self._prefix} error {rc}: "
                              f"{self.lib.mjpc_b200_batch_estimator_last_error(self.h).decode()}")

    def reset(self, b, state=None, time=0.0, covariance_scale=None, process_scale=None, sensor_scale=None):
        x, cs, ps, ss = reset_values(self.m, state, covariance_scale, process_scale, sensor_scale)
        self._check(self.lib.mjpc_b200_batch_estimator_reset(self.h, b, _pd(_d(x)), time, cs, ps, ss))

    def set_models(self, models):
        """Filter b runs on compiled model models[b] from now on (len(models) == num_filters; the rule of
        Engine.set_model_variants); None or [] runs every filter on the bank's model again.  The filters' states are
        kept."""
        bufs, arr, n = _model_blobs(models)
        self._check(self.lib.mjpc_b200_batch_estimator_set_models(self.h, arr, n))

    def set_noise(self, b, process=None, sensor=None):
        self._check(self.lib.mjpc_b200_batch_estimator_set_noise(self.h, b, _pd(_d(process)), _pd(_d(sensor))))

    def set(self, b, state, covariance, time):
        self._check(self.lib.mjpc_b200_batch_estimator_set(self.h, b, _pd(_d(state)), _pd(_d(covariance)), time))

    def update(self, ctrl, sensor, mocap=None):
        """One update of every filter from ctrl [B][nu], sensor [B][nsensordata] and mocap [B][7 nmocap] (None: the
        model's); returns status [B]."""
        B = self.num_filters
        u = np.ascontiguousarray(np.asarray(ctrl, float).reshape(B, self.m.nu))
        y = np.ascontiguousarray(np.asarray(sensor, float).reshape(B, self.nsensordata))
        mc = None if mocap is None or np.size(mocap) == 0 else \
            np.ascontiguousarray(np.asarray(mocap, np.float32).reshape(B, -1))
        status = np.zeros(B, np.int32)
        self._check(self.lib.mjpc_b200_batch_estimator_update(self.h, _pd(u), _pd(y), _pf(mc),
                                                              status.ctypes.data_as(C.POINTER(C.c_int))))
        return status

    def get(self, b):
        """(state, covariance, time, scalars) of filter b."""
        return _get_filter(self, functools.partial(self.lib.mjpc_b200_batch_estimator_get, self.h, b))

    def debug_rows(self, phase, ctrl=None, mocap=None):
        """The bank's row kernel alone (mjpc_b200_batch_estimator_debug_rows; phase 0 Unscented, 1 Kalman measurement,
        2 Kalman prediction) from ctrl [B][nu] (None: zeros) and mocap (None: the model's): (qpos [B][rows][nq],
        qvel [B][rows][nv], the rows' warm starts [B][rows][nv], status [B])."""
        B, R, m = self.num_filters, self.rows, self.m
        u = np.ascontiguousarray(np.zeros((B, m.nu)) if ctrl is None else np.asarray(ctrl, float).reshape(B, m.nu))
        mc = None if mocap is None or np.size(mocap) == 0 else \
            np.ascontiguousarray(np.asarray(mocap, np.float32).reshape(B, -1))
        qpos, qvel = np.zeros((B, R, m.nq), np.float32), np.zeros((B, R, m.nv), np.float32)
        warm = np.zeros((B, R, m.nv), np.float32)
        status = np.zeros(B, np.int32)
        self._check(self.lib.mjpc_b200_batch_estimator_debug_rows(
            self.h, int(phase), _pd(u), _pf(mc), _pf(qpos), _pf(qvel), _pf(warm),
            status.ctypes.data_as(C.POINTER(C.c_int))))
        return qpos, qvel, warm, status

    def debug_finish(self, phase, sensor, next_qpos, next_qvel, qacc, sensordata, counts):
        """The phase's update kernel on the caller's step outputs (mjpc_b200_batch_estimator_debug_finish):
        sensor [B][nsensordata] (None for phase 2), next_qpos [B][rows][nq], next_qvel / qacc [B][rows][nv],
        sensordata [B][rows][nsensordata] (float32) and counts [B][rows][4] (int32); returns the raw status [B]."""
        B, R, m = self.num_filters, self.rows, self.m
        f32 = lambda a, n: np.ascontiguousarray(np.asarray(a, np.float32).reshape(B, R, n))
        nq, nv, ys, qa = f32(next_qpos, m.nq), f32(next_qvel, m.nv), f32(sensordata, self.nsensordata), f32(qacc, m.nv)
        cn = np.ascontiguousarray(np.asarray(counts, np.int32).reshape(B, R, 4))
        y = None if sensor is None else np.ascontiguousarray(np.asarray(sensor, float).reshape(B, self.nsensordata))
        status = np.zeros(B, np.int32)
        ip = C.POINTER(C.c_int)
        self._check(self.lib.mjpc_b200_batch_estimator_debug_finish(
            self.h, int(phase), _pd(y), _pf(nq), _pf(nv), _pf(qa), _pf(ys), cn.ctypes.data_as(ip),
            status.ctypes.data_as(ip)))
        return status

    def state(self, b):
        return self.get(b)[0]

    def covariance(self, b):
        return self.get(b)[1]

    def time(self, b):
        return self.get(b)[2]

    def warnings(self, b):
        return int(self.get(b)[3][3])
