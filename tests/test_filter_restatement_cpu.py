"""The fp64 filter restatement of tests/filter_scenes.py, pinned before it judges the device filters:
  * on the linear slide it is the textbook Kalman filter on the closed-form F and H (the Unscented filter at any alpha
    and the finite-difference Kalman filter are exact for a linear-Gaussian model): 1e-12;
  * on the slide and the free / ball scene it agrees with the Python mirror (mujoco_mpc_b200.estimator) stepping on
    the fp64 oracle, both fed the same steps: 1e-9;
  * its factorisation fails exactly where the device's does: a pivot below 1e-15 or not finite, and so does the
    mirror's.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter_scenes as FS  # noqa: E402
from estimator_backends import OracleSigmaBackend  # noqa: E402

from mujoco_mpc_b200.estimator import EstimatorError, Kalman, Unscented, cholesky  # noqa: E402

STEPS = 10


def _noise(n, seed):
    return np.random.default_rng(seed).normal(size=n)


def _textbook(F, G, H, c, x, P, u, y, Q, R):
    """One measurement-then-prediction step of the textbook Kalman filter (the UKF's joint Gaussian of the next state and
    the pre-step sensors conditions the same way)."""
    S = H @ P @ H.T + R
    K = np.linalg.solve(S, H @ P).T
    x = x + K @ (y - H @ x)
    P = P - K @ S @ K.T
    return F @ x + G @ u + c, F @ P @ F.T + Q


def _ukf_joint(F, G, H, c, x, P, u, y, Q, R):
    """The Unscented filter's update for a linear model: condition (F x + G u + c, H x) on y."""
    S = H @ P @ H.T + R
    K = F @ P @ H.T @ np.linalg.inv(S)
    return F @ x + G @ u + c + K @ (y - H @ x), F @ P @ F.T + Q - K @ H @ P @ F.T


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - b)) / (np.max(np.abs(b)) + 1e-300))


@pytest.mark.parametrize("alpha", [1.0, 0.5, 2.0])
def test_unscented_is_the_exact_filter_on_the_linear_slide(alpha):
    sc = FS.slide()
    m = sc.m
    F, G, H, c = FS.slide_linear_model(sc)
    W = FS.UKFWeights(4, alpha)
    x, P = sc.x0.copy(), np.diag([1e-2, 2e-2, 3e-2, 4e-2]) + 1e-3
    Q, R = np.array([1e-4, 2e-4, 3e-4, 4e-4]), np.array([1e-3, 1e-3, 2e-3, 2e-3])
    xr, Pr = x.copy(), P.copy()
    for t in range(STEPS):
        u = np.array([0.3, -0.2 + 0.1 * t])
        y = H @ xr + 0.05 * _noise(4, t)
        pts = FS.sigma_points(m, x, P, W)
        x, P, _ = FS.ukf_update(m, W, [sc.step(p, u) for p in pts], [sc.h(p) for p in pts], y, Q, R)
        xr, Pr = _ukf_joint(F, G, H, c, xr, Pr, u, y, np.diag(Q), np.diag(R))
        assert _rel(x, xr) < 1e-12 and _rel(P, Pr) < 1e-12, (t, _rel(x, xr), _rel(P, Pr))


@pytest.mark.parametrize("centered", [True, False])
def test_kalman_is_the_exact_filter_on_the_linear_slide(centered):
    sc = FS.slide()
    m = sc.m
    F, G, H, c = FS.slide_linear_model(sc)
    x, P = sc.x0.copy(), np.diag([1e-2, 2e-2, 3e-2, 4e-2]) + 1e-3
    Q, R = np.array([1e-4, 2e-4, 3e-4, 4e-4]), np.array([1e-3, 1e-3, 2e-3, 2e-3])
    xr, Pr = x.copy(), P.copy()
    eps = 1e-3
    for t in range(STEPS):
        u = np.array([0.3, -0.2 + 0.1 * t])
        y = H @ xr + 0.05 * _noise(4, t)
        rows = FS.kalman_rows(m, x, eps, centered)
        x, P = FS.kalman_measurement(m, x, P, [sc.h(r) for r in rows], y, R, eps, centered)
        rows = FS.kalman_rows(m, x, eps, centered)
        x, P = FS.kalman_prediction(m, P, [sc.step(r, u) for r in rows], Q, eps, centered)
        xr, Pr = _textbook(F, G, H, c, xr, Pr, u, y, np.diag(Q), np.diag(R))
        assert _rel(x, xr) < 1e-12 and _rel(P, Pr) < 1e-12, (t, _rel(x, xr), _rel(P, Pr))


class _Recorder:
    """An oracle backend that also keeps its last call's rows and outputs."""

    def __init__(self, m, s, n, ts):
        self.o = OracleSigmaBackend(m, s, n, ts)

    def step_sensors(self, states, ctrl, mocap, time, warmstart):
        out = self.o.step_sensors(states, ctrl, mocap, time, warmstart)
        self.last = (np.array(states, float), out)
        return out


@pytest.mark.parametrize("scene", ["slide", "free_ball"])
def test_unscented_matches_the_mirror_on_the_oracle(scene):
    sc = getattr(FS, scene)()
    m = sc.m
    rec = {}
    f = Unscented(m, lambda s, n, ts: rec.setdefault("b", _Recorder(m, s, n, ts)), sensor_start=FS.SENSOR_START,
                  nsensor=sc.nsensor, alpha=1.0, beta=2.0)
    f.reset(sc.x0, covariance_scale=1e-3, process_scale=1e-5, sensor_scale=1e-4)
    W = FS.UKFWeights(2 * m.nv, 1.0)
    u = np.zeros(m.nu) + 0.1
    for t in range(4):
        x0, P0 = f.state.copy(), f.covariance.copy()
        y = sc.h(sc.x0) + 1e-3 * _noise(sc.ny, t)
        f.update(u, y)
        rows, (nxt, ys, _, _) = rec["b"].last
        assert _rel(FS.sigma_points(m, x0, P0, W), rows) < 1e-13
        x, P, _ = FS.ukf_update(m, W, nxt, ys, y, f.noise_process, f.noise_sensor)
        assert _rel(x, f.state) < 1e-9 and _rel(P, f.covariance) < 1e-9, (t, _rel(x, f.state), _rel(P, f.covariance))


@pytest.mark.parametrize("scene", ["slide", "free_ball"])
@pytest.mark.parametrize("centered", [True, False])
def test_kalman_matches_the_mirror_on_the_oracle(scene, centered):
    sc = getattr(FS, scene)()
    m = sc.m
    rec = {}
    f = Kalman(m, lambda s, n, ts: rec.setdefault("b", _Recorder(m, s, n, ts)), sensor_start=FS.SENSOR_START,
               nsensor=sc.nsensor, epsilon=1e-4, centered=centered)
    f.reset(sc.x0, covariance_scale=1e-3, process_scale=1e-5, sensor_scale=1e-4)
    u = np.zeros(m.nu) + 0.1
    for t in range(3):
        x0, P0 = f.state.copy(), f.covariance.copy()
        y = sc.h(sc.x0) + 1e-3 * _noise(sc.ny, t)
        f.update_measurement(u, y)
        rows, (_, ys, _, _) = rec["b"].last
        assert _rel(FS.kalman_rows(m, x0, 1e-4, centered), rows) < 1e-13
        x, P = FS.kalman_measurement(m, x0, P0, ys, y, f.noise_sensor, 1e-4, centered)
        assert _rel(x, f.state) < 1e-9 and _rel(P, f.covariance) < 1e-9
        f.update_prediction()
        rows, (nxt, _, _, _) = rec["b"].last
        x2, P2 = FS.kalman_prediction(m, P, nxt, f.noise_process, 1e-4, centered)
        assert _rel(x2, f.state) < 1e-9 and _rel(P2, f.covariance) < 1e-9


@pytest.mark.parametrize("M,ok", [
    (np.diag([1.0, 1e-15]), True),
    (np.diag([1.0, 1e-15 * (1 - 2 ** -40)]), False),
    (np.diag([1.0, 1e-16]), False),
    (np.diag([1.0, 0.0]), False),
    (np.array([[np.nan, 0.0], [0.0, 1.0]]), False),
    (np.array([[1.0, np.nan], [np.nan, 1.0]]), False),
    (np.diag([np.inf, 1.0]), False),
    (np.diag([1.0, -1.0]), False),
])
def test_factorisation_threshold_and_non_finite_pivots(M, ok):
    """The restatement and the mirror accept the same pivots: >= 1e-15 and finite."""
    for fn, err in ((FS.factor, FS.FactorError), (lambda a: cholesky(a, "covariance"), EstimatorError)):
        if ok:
            fn(M)
        else:
            with pytest.raises(err):
                fn(M)


def test_mirror_refuses_a_non_finite_result_and_keeps_its_state():
    sc = FS.slide()
    m = sc.m
    f = Kalman(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts), sensor_start=FS.SENSOR_START, nsensor=sc.nsensor)
    f.reset(sc.x0, covariance_scale=1e-3)
    x, P, t = f.state.copy(), f.covariance.copy(), f.time
    y = sc.h(sc.x0)
    y[0] = np.inf
    with pytest.raises(EstimatorError, match="non-finite result"):
        f.update_measurement(np.zeros(m.nu), y)
    assert np.array_equal(f.state, x) and np.array_equal(f.covariance, P) and f.time == t
