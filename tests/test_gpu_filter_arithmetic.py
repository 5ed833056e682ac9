"""GPU: the device filter bank's fp64 arithmetic (csrc/estimator_kernels.cuh) against the independent fp64 restatement
of tests/filter_scenes.py, at its edges.

The bank's own kernels run on data the test chooses through two test hooks of CppBatchEstimator: debug_rows returns the
step rows (and their warm starts) the row kernel stages, and debug_finish runs a phase's update kernel on step outputs
the test defines.  That takes the physics out of the comparison and lets non-finite values reach the filter arithmetic
without a non-finite state ever entering a step launch.  The restatement is fed the same float rows and sensors the
device used.

Bars.  Rows: the device's float rows equal float32 of the restated fp64 rows to 1 float ulp.  Updates: each quantity
(state, covariance) is held to 4x the spread of the restatement over NEIGHBOURS copies of its float inputs moved by one
ulp in about two thirds of their entries, plus 16 fp64 ulps of the quantity's scale (test_gpu_smooth_dynamics.py takes
its bars the same way).  Time, the warm start (qacc of the nominal / centre row) and the warnings (rows whose
counts[4r+3] is non-zero) are exact.  A filter that fails - a factor with a pivot below 1e-15 or not finite, or a new
state or covariance that is not finite - stays bitwise untouched, and the other filters of its bank are bitwise what
they are alone.

End to end (real step launches on the linear slide and on the free / ball scene): the device is compared with the exact
fp64 filter, and its error is held to 16x the error of the restatement run on the closed-form step rounded to float32.
test_zz_report prints the largest ratio of each group to its bar.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter_scenes as FS  # noqa: E402
import joint_scenes as JS  # noqa: E402

from mujoco_mpc_b200.engine import EngineError  # noqa: E402
from mujoco_mpc_b200.estimator import CppBatchEstimator  # noqa: E402

pytestmark = pytest.mark.gpu

NEIGHBOURS = 4
UPDATED, SENSOR_FAILED, COVARIANCE_FAILED, NONFINITE = 0, 1, 2, 3
RATIOS = {}
REPORT = {}


def _ratio(group, err, bar):
    r = float(err) / float(bar) if bar > 0 else (0.0 if err == 0 else np.inf)
    RATIOS[group] = max(RATIOS.get(group, 0.0), r)
    return r <= 1.0


_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        _SCENES[name] = getattr(FS, name)()
    return _SCENES[name]


def _bank(sc, kind, B=1, alpha=1.0, epsilon=1e-3, centered=True, nsensor=None):
    return CppBatchEstimator(sc.m, kind, B, sensor_start=FS.SENSOR_START,
                             nsensor=sc.nsensor if nsensor is None else nsensor, timestep=JS.DT, alpha=alpha,
                             beta=2.0, epsilon=epsilon, centered=centered)


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32)


def _neighbour(a, k):
    """float32 array a moved by one ulp up or down in about two thirds of its non-zero finite entries (copy k)."""
    a = np.array(a, np.float32)
    rng = np.random.default_rng(1000 + k)
    pick = (rng.random(a.shape) < 2 / 3) & (a != 0) & np.isfinite(a)
    up = rng.random(a.shape) < 0.5
    out = a.copy()
    out[pick & up] = np.nextafter(a[pick & up], np.float32(np.inf))
    out[pick & ~up] = np.nextafter(a[pick & ~up], np.float32(-np.inf))
    return out


def _bars(fn, f32_inputs):
    """(restated results, bars): fn(*inputs) -> tuple of arrays; bar = 4 x spread over NEIGHBOURS + 16 ulps of scale."""
    r0 = fn(*f32_inputs)
    spread = [np.zeros(()) for _ in r0]
    for k in range(NEIGHBOURS):
        rk = fn(*[_neighbour(a, 7 * k + j) for j, a in enumerate(f32_inputs)])
        spread = [np.maximum(s, np.max(np.abs(np.asarray(a) - b))) for s, a, b in zip(spread, rk, r0)]
    bars = [4 * s + 16 * np.spacing(np.max(np.abs(r))) for s, r in zip(spread, r0)]
    return r0, bars


def _snapshot(est, b):
    x, P, t, sc = est.get(b)
    return x, P, t, int(sc[3])


def _assert_untouched(est, b, before):
    x, P, t, w = _snapshot(est, b)
    assert np.array_equal(x, before[0]) and np.array_equal(P, before[1]) and t == before[2] and w == before[3], b


def _rows(est, phase):
    qpos, qvel, warm, status = est.debug_rows(phase)
    return np.concatenate([qpos, qvel], axis=2), warm, status


def _spd(n, cond, seed):
    rng = np.random.default_rng(seed)
    Qm, _ = np.linalg.qr(rng.normal(size=(n, n)))
    ev = np.geomspace(1.0, 1.0 / cond, n) * 1e-2
    P = Qm @ np.diag(ev) @ Qm.T
    return 0.5 * (P + P.T)


# ------------------------------------------------------------------------------------------------------- rows
def _check_rows(dev, ref):
    ref32 = _f32(ref)
    err = np.abs(dev.astype(np.float64) - ref32.astype(np.float64))
    ulp = np.maximum(np.spacing(np.abs(ref32)), np.float32(1e-30)).astype(np.float64)
    assert _ratio("rows (float ulps)", np.max(err / ulp), 1.0), np.max(err / ulp)


ROW_CASES = ["well_conditioned", "cond_1e12", "pivot_at_1e-15", "pivot_below_1e-15", "rank_deficient",
             "rot_0.1", "rot_1.5", "rot_pi-1e-3", "rot_pi+0.3"]


def _row_case(case):
    if case.startswith("rot_"):
        sc = _scene("free_ball")
    else:
        sc = _scene("slide")
    m = sc.m
    n = 2 * m.nv
    x = sc.x0.copy()
    if case == "well_conditioned":
        P = _spd(n, 10.0, 1)
    elif case == "cond_1e12":
        P = _spd(n, 1e12, 2)
    elif case == "pivot_at_1e-15":
        P = np.diag([1e-2] * (n - 1) + [1e-15])
    elif case == "pivot_below_1e-15":
        P = np.diag([1e-2] * (n - 1) + [1e-15 * (1 - 2.0 ** -40)])
    elif case == "rank_deficient":
        P = _spd(n, 10.0, 3)
        P[1, :] = P[:, 1] = 0.0
    else:
        th = {"rot_0.1": 0.1, "rot_1.5": 1.5, "rot_pi-1e-3": np.pi - 1e-3, "rot_pi+0.3": np.pi + 0.3}[case]
        step = np.sqrt(n)   # alpha 1
        P = np.diag(np.full(n, 1e-6))
        P[4, 4] = (th / step) ** 2          # the free body's second rotation dof
        P[7 + 2, 7 + 2] = (th / step) ** 2  # the ball's third rotation dof
        P[3, 5] = P[5, 3] = 0.5e-6          # and a coupling within the free body's rotation
    return sc, x, P


@pytest.mark.parametrize("case", ROW_CASES)
def test_sigma_rows(case):
    sc, x, P = _row_case(case)
    m = sc.m
    est = _bank(sc, "unscented")
    est.set(0, x, P, 0.25)
    rows, _, status = _rows(est, 0)
    W = FS.UKFWeights(2 * m.nv, 1.0)
    try:
        ref = FS.sigma_points(m, x, P, W)
    except FS.FactorError:
        ref = None
    if ref is None:
        assert status[0] == COVARIANCE_FAILED, (case, status)
        assert np.array_equal(rows[0], np.tile(_f32(x), (W.R, 1))), case
        assert case in ("pivot_below_1e-15", "rank_deficient"), case
        return
    assert status[0] == UPDATED, (case, status)
    _check_rows(rows[0], ref)


@pytest.mark.parametrize("centered", [True, False])
def test_kalman_rows_on_quaternion_dofs(centered):
    sc = _scene("free_ball")
    m = sc.m
    est = _bank(sc, "kalman", epsilon=1e-3, centered=centered)
    est.set(0, sc.x0, 1e-3 * np.eye(2 * m.nv), 0.0)
    for phase in (1, 2):
        rows, _, _ = _rows(est, phase)
        _check_rows(rows[0], FS.kalman_rows(m, sc.x0, 1e-3, centered))


# ------------------------------------------------------------------------------------------------------- updates
def _map_next(m, rows, x, kind):
    """The test's step: identity, an affine map in the tangent space about x, or a fixed rotation of each quaternion;
    fp64 of the float rows, returned as float32."""
    n = 2 * m.nv
    rows = np.asarray(rows, np.float64)
    if kind == "identity":
        return _f32(rows)
    if kind == "affine":
        rng = np.random.default_rng(5)
        T = np.eye(n) + 0.05 * rng.normal(size=(n, n))
        b = 0.01 * rng.normal(size=n)
        return _f32([FS.plus(m, x, T @ FS.minus(m, r, x) + b) for r in rows])
    out = rows.copy()
    rot = FS.FD.quat_exp(np.array([0.4, -0.3, 0.2]))
    for a in FS.quat_slots(m):
        for r in out:
            r[a:a + 4] = FS.FD.quat_mul(r[a:a + 4], rot)
    return _f32(out)


def _sensors(m, rows, x, ny, seed):
    """Sensors affine in the pre-step tangent deviation: c + G (row (-) x), as float32; and (c, G)."""
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(ny, 2 * m.nv))
    c = rng.normal(size=ny)
    return _f32([c + G @ FS.minus(m, np.asarray(r, np.float64), x) for r in rows]), c, G


def _outputs(R, nv, seed):
    rng = np.random.default_rng(seed)
    qacc = _f32(rng.normal(size=(R, nv)))
    counts = np.zeros((R, 4), np.int32)
    counts[rng.random(R) < 0.3, 3] = 1
    counts[:, 0] = 7
    return qacc, counts


def _finish(est, phase, y, nxt, ys, qacc, counts):
    m = est.m
    nxt = np.asarray(nxt, np.float32)
    B = est.num_filters
    return est.debug_finish(phase, y, nxt[..., :m.nq].reshape(B, -1), nxt[..., m.nq:].reshape(B, -1), qacc, ys, counts)


def _compare(group, dev, ref, bar):
    err = np.max(np.abs(np.asarray(dev) - ref))
    assert _ratio(group, err, bar), (group, err, bar)


UKF_CASES = [("free_ball", a, k) for a in (1.0, 0.5, 2.0) for k in ("identity", "affine", "rotation")] + \
            [("slide", 1.0, "affine"), ("hinges", 1.0, "affine"), ("hinges", 0.5, "identity")]


@pytest.mark.parametrize("scene,alpha,step", UKF_CASES)
@pytest.mark.parametrize("ny1", [False, True])
def test_unscented_update(scene, alpha, step, ny1):
    if ny1 and scene != "slide":
        pytest.skip("ny = 1 on the slide")
    sc = _scene(scene)
    m = sc.m
    n = 2 * m.nv
    est = _bank(sc, "unscented", alpha=alpha, nsensor=1 if ny1 else None)
    ny = est.nsensordata
    x = sc.x0.copy()
    P = _spd(n, 1e3, 11)
    Q, Rn = np.full(n, 1e-5) * (1 + np.arange(n) / n), np.full(ny, 1e-4) * (1 + np.arange(ny) / ny)
    est.set(0, x, P, 0.5)
    est.set_noise(0, Q, Rn)
    rows, _, status = _rows(est, 0)
    assert status[0] == UPDATED
    R = rows.shape[1]
    nxt = _map_next(m, rows[0], x, step)
    ys, c, G = _sensors(m, rows[0], x, ny, 3)
    y = c + 0.01 * np.random.default_rng(4).normal(size=ny)
    qacc, counts = _outputs(R, m.nv, 6)
    w0 = _snapshot(est, 0)[3]
    status = _finish(est, 0, y[None], nxt[None], ys[None], qacc[None], counts[None])
    assert status[0] == UPDATED, status
    W = FS.UKFWeights(n, alpha)
    (xr, Pr), (bx, bP) = _bars(lambda a, b: FS.ukf_update(m, W, a, b, y, Q, Rn)[:2], [nxt, ys])
    _, _, info = FS.ukf_update(m, W, nxt, ys, y, Q, Rn)
    for a, (lam, K) in info.items():   # a distinct top eigenvalue: the mean quaternion is the eigenvector itself
        assert lam[-1] - lam[-2] > 1e-6 * abs(lam[-1]), (a, lam)
    xd, Pd, td, wd = _snapshot(est, 0)
    _compare("unscented state", xd, xr, bx)
    _compare("unscented covariance", Pd, Pr, bP)
    assert td == 0.5 + JS.DT
    assert wd == w0 + int(np.count_nonzero(counts[:, 3]))
    _, warm, _ = _rows(est, 0)
    assert np.array_equal(warm[0], np.tile(qacc[R - 1], (R, 1)))   # every row warm-starts from the nominal row's qacc


@pytest.mark.parametrize("centered", [True, False])
def test_kalman_measurement_and_prediction(centered):
    sc = _scene("free_ball")
    m = sc.m
    n, eps = 2 * m.nv, 1e-3
    est = _bank(sc, "kalman", epsilon=eps, centered=centered)
    ny = est.nsensordata
    x, P = sc.x0.copy(), _spd(n, 1e3, 21)
    Q, Rn = np.full(n, 2e-5), np.full(ny, 1e-4) * (1 + np.arange(ny) / ny)
    est.set(0, x, P, 1.0)
    est.set_noise(0, Q, Rn)
    # measurement
    rows, _, status = _rows(est, 1)
    R = rows.shape[1]
    ys, c, G = _sensors(m, rows[0], x, ny, 23)
    y = c + 0.01 * np.random.default_rng(24).normal(size=ny)
    qacc, counts = _outputs(R, m.nv, 25)
    status = _finish(est, 1, y[None], _f32(rows), ys[None], qacc[None], counts[None])
    assert status[0] == UPDATED
    (xr, Pr), (bx, bP) = _bars(lambda b: FS.kalman_measurement(m, x, P, b, y, Rn, eps, centered), [ys])
    xd, Pd, td, _ = _snapshot(est, 0)
    _compare("kalman measurement state", xd, xr, bx)
    _compare("kalman measurement covariance", Pd, Pr, bP)
    assert td == 1.0
    # prediction, with the next quaternions of every other row on the opposite hemisphere
    rows, _, _ = _rows(est, 2)
    nxt = _map_next(m, rows[0], xd, "rotation")
    for a in FS.quat_slots(m):
        nxt[1::2, a:a + 4] *= -1
    qacc, counts = _outputs(R, m.nv, 26)
    status = _finish(est, 2, None, nxt[None], np.zeros((1, R, ny), np.float32), qacc[None], counts[None])
    assert status[0] == UPDATED
    (xr, Pr), (bx, bP) = _bars(lambda a: FS.kalman_prediction(m, Pd, a, Q, eps, centered), [nxt])
    x2, P2, t2, _ = _snapshot(est, 0)
    assert np.array_equal(x2, nxt[0].astype(np.float64))
    _compare("kalman prediction covariance", P2, Pr, bP)
    assert t2 == 1.0 + JS.DT
    _, warm, _ = _rows(est, 2)
    assert np.array_equal(warm[0], np.tile(qacc[0], (R, 1)))


# ------------------------------------------------------------------------------------------------------- conditioning
def _slide_unscented_inputs(est, b, ny, dup_scale, seed):
    """Rows, identity next rows and sensors for filter b of a slide bank whose sensor 1 is sensor 0 + dup_scale x
    another direction (dup_scale 0: an exact duplicate)."""
    m = est.m
    rows, _, _ = _rows(est, 0)
    ys, c, G = _sensors(m, rows[b], est.get(b)[0], ny, seed)
    ys[:, 1] = ys[:, 0] + _f32(dup_scale * (ys[:, 2] - ys[:, 3]))
    return _f32(rows[b]), ys, c


def test_ill_conditioned_sensor_covariance():
    """cond(S) about 1e10: near-duplicate sensors at sensor noise 1e-12."""
    sc = _scene("slide")
    m = sc.m
    n = 2 * m.nv
    est = _bank(sc, "unscented")
    ny = est.nsensordata
    P = _spd(n, 10.0, 31)
    Q, Rn = np.full(n, 1e-6), np.full(ny, 1e-12)
    est.set(0, sc.x0, P, 0.0)
    est.set_noise(0, Q, Rn)
    nxt, ys, c = _slide_unscented_inputs(est, 0, ny, 1e-4, 32)
    R = nxt.shape[0]
    W = FS.UKFWeights(n, 1.0)
    wc = W.vec(W.wc0)
    dy = ys.astype(float) - W.vec(W.wm0) @ ys.astype(float)
    S = np.diag(Rn) + (dy.T * wc) @ dy
    REPORT["cond(S), near-duplicate sensors"] = float(np.linalg.cond(S))
    assert 1e8 < np.linalg.cond(S) < 1e12
    y = ys[-1].astype(float)
    qacc, counts = _outputs(R, m.nv, 33)
    status = _finish(est, 0, y[None], nxt[None], ys[None], qacc[None], counts[None])
    assert status[0] == UPDATED
    (xr, Pr), (bx, bP) = _bars(lambda a, b: FS.ukf_update(m, W, a, b, y, Q, Rn)[:2], [nxt, ys])
    xd, Pd, _, _ = _snapshot(est, 0)
    _compare("ill-conditioned S state", xd, xr, bx)
    _compare("ill-conditioned S covariance", Pd, Pr, bP)


def _batch_case(est, b, fail):
    """Inputs of filter b of an Unscented slide bank: fail None (normal), "nan_rows", "inf_sensor" or "rank_S"."""
    m = est.m
    ny = est.nsensordata
    nxt, ys, c = _slide_unscented_inputs(est, b, ny, 0.0 if fail == "rank_S" else 0.5, 40 + b)
    if fail == "nan_rows":
        nxt[3, 1] = np.nan
    elif fail == "inf_sensor":
        ys[2, 0] = np.inf
    y = ys[-1].astype(float) + 0.01
    qacc, counts = _outputs(nxt.shape[0], m.nv, 50 + b)
    return y, nxt, ys, qacc, counts


def _setup_slide_filter(est, b, seed, zero_noise=False):
    m = est.m
    n = 2 * m.nv
    est.set(b, _scene("slide").x0 + 0.01 * seed, _spd(n, 10.0, seed), 0.1 * seed)
    est.set_noise(b, np.full(n, 1e-5 * (1 + seed)), np.full(est.nsensordata, 0.0 if zero_noise else 1e-4))


def test_isolation_of_failing_filters():
    """B = 5, filters 0 (NaN next rows) and 3 (exactly rank-deficient S) fail; they stay bitwise untouched and the
    others are bitwise what they are alone."""
    sc = _scene("slide")
    fails = {0: "nan_rows", 3: "rank_S"}
    est = _bank(sc, "unscented", B=5)
    for b in range(5):
        _setup_slide_filter(est, b, b + 1, zero_noise=fails.get(b) == "rank_S")
    before = [_snapshot(est, b) for b in range(5)]
    inputs = [_batch_case(est, b, fails.get(b)) for b in range(5)]
    status = _finish(est, 0, *[np.stack([i[k] for i in inputs]) for k in range(5)])
    assert list(status) == [NONFINITE, UPDATED, UPDATED, SENSOR_FAILED, UPDATED], status
    for b in (0, 3):
        _assert_untouched(est, b, before[b])
    for b in (1, 2, 4):
        one = _bank(sc, "unscented", B=1)
        _setup_slide_filter(one, 0, b + 1)
        _rows(one, 0)
        s1 = _finish(one, 0, *[i[None] for i in inputs[b]])
        assert s1[0] == UPDATED
        xa, Pa, ta, wa = _snapshot(one, 0)
        xb, Pb, tb, wb = _snapshot(est, b)
        assert np.array_equal(xa, xb) and np.array_equal(Pa, Pb) and ta == tb and wa == wb, b


@pytest.mark.parametrize("kind,phase,fail,expect", [
    ("unscented", 0, "nan_rows", NONFINITE),
    ("unscented", 0, "inf_rows", NONFINITE),
    ("unscented", 0, "nan_sensor", SENSOR_FAILED),
    ("unscented", 0, "inf_sensor", SENSOR_FAILED),
    ("kalman", 1, "nan_sensor", SENSOR_FAILED),
    ("kalman", 1, "inf_sensor", SENSOR_FAILED),
    ("kalman", 2, "nan_rows", NONFINITE),
    ("kalman", 2, "inf_rows", NONFINITE),
])
def test_non_finite_step_outputs_fail_the_filter_untouched(kind, phase, fail, expect):
    """A NaN or inf in one filter's next rows or sensordata (a NaN pivot of S) fails that filter and leaves it, and its
    neighbour's result, as they would be."""
    sc = _scene("free_ball")
    m = sc.m
    n = 2 * m.nv
    runs = {}
    for label, bad in (("bad", True), ("clean", False)):
        est = _bank(sc, kind, B=2)
        ny = est.nsensordata
        for b in range(2):
            est.set(b, sc.x0, _spd(n, 10.0, 60 + b), 0.0)
            est.set_noise(b, np.full(n, 1e-5), np.full(ny, 1e-4))
        before = [_snapshot(est, b) for b in range(2)]
        rows, _, _ = _rows(est, phase)
        R = rows.shape[1]
        nxt = np.stack([_map_next(m, rows[b], sc.x0, "affine") for b in range(2)])
        ys = np.stack([_sensors(m, rows[b], sc.x0, ny, 70 + b)[0] for b in range(2)])
        if bad:
            v = np.nan if fail.startswith("nan") else np.inf
            if fail.endswith("rows"):
                nxt[0, 2, 1] = v
            else:
                ys[0, 1, 2] = v
        qacc = np.zeros((2, R, m.nv), np.float32)
        counts = np.zeros((2, R, 4), np.int32)
        y = ys[:, 0, :].astype(float) + 0.01
        status = _finish(est, phase, None if phase == 2 else y, nxt, ys, qacc, counts)
        runs[label] = (est, status, before)
    est, status, before = runs["bad"]
    assert status[0] == expect and status[1] == UPDATED, status
    _assert_untouched(est, 0, before[0])
    ref = runs["clean"][0]
    assert all(np.array_equal(a, b) for a, b in zip(_snapshot(est, 1)[:3], _snapshot(ref, 1)[:3]))


@pytest.mark.parametrize("kind", ["unscented", "kalman"])
def test_public_calls_refuse_non_finite_values(kind):
    sc = _scene("slide")
    m = sc.m
    n = 2 * m.nv
    est = _bank(sc, kind, B=2)
    ny = est.nsensordata
    for b in range(2):
        est.set(b, sc.x0, _spd(n, 10.0, 80 + b), 0.0)
    before = [_snapshot(est, b) for b in range(2)]
    y = np.tile(sc.h(sc.x0), (2, 1))
    y[1, 2] = np.nan
    with pytest.raises(EngineError, match="not finite"):
        est.update(np.zeros((2, m.nu)), y)
    u = np.zeros((2, m.nu))
    u[0, 0] = np.inf
    with pytest.raises(EngineError, match="not finite"):
        est.update(u, np.tile(sc.h(sc.x0), (2, 1)))
    P = np.eye(n)
    P[0, 0] = np.nan
    with pytest.raises(EngineError, match="not finite"):
        est.set(0, sc.x0, P, 0.0)
    with pytest.raises(EngineError, match="not finite"):
        est.set(0, sc.x0, None, np.inf)
    with pytest.raises(EngineError, match="not finite"):
        est.set_noise(1, np.full(n, np.nan), None)
    with pytest.raises(EngineError, match="not finite"):
        est.set_noise(1, None, np.full(ny, -np.inf))
    for b in range(2):
        _assert_untouched(est, b, before[b])
    # and the bank still updates
    assert list(est.update(np.zeros((2, m.nu)), np.tile(sc.h(sc.x0), (2, 1)))) == [0, 0]


# ------------------------------------------------------------------------------------------------------- end to end
T_STEPS = 50


def _controls(t, nu):
    return np.array([0.5 * np.sin(0.3 * t), 0.4 * np.cos(0.2 * t)])[:nu]


def _e2e_filters(sc, kind, alpha, B):
    n = 2 * sc.m.nv
    P0 = [np.diag(np.full(n, 1e-3 * (b + 1))) for b in range(B)]
    Q = [np.full(n, 1e-6 * (b + 1)) for b in range(B)]
    R = [np.full(sc.ny, 1e-4 / (b + 1)) for b in range(B)]
    return P0, Q, R


def _truth(sc, x0, T, seed, sd):
    rng = np.random.default_rng(seed)
    xs, ys = [], []
    x = x0.copy()
    for t in range(T):
        ys.append(sc.h(x) + sd * rng.normal(size=sc.ny))
        xs.append(x)
        x = sc.step(x, _controls(t, sc.m.nu))
    return np.array(xs), np.array(ys)


def _restated_run(sc, kind, alpha, eps, x0, P0, Q, R, ys, rounded):
    """The restatement's filter on the closed-form step, exact (rounded False) or with rows, steps and sensors rounded
    to float32 as the device's are."""
    m = sc.m
    r = (lambda a: _f32(a).astype(np.float64)) if rounded else (lambda a: np.asarray(a, float))
    x, P = x0.copy(), P0.copy()
    out = []
    W = FS.UKFWeights(2 * m.nv, alpha)
    for t, y in enumerate(ys):
        u = _controls(t, m.nu)
        if kind == "unscented":
            pts = r(FS.sigma_points(m, x, P, W))
            x, P, _ = FS.ukf_update(m, W, r([sc.step(p, u) for p in pts]), r([sc.h(p) for p in pts]), y, Q, R)
        else:
            rows = r(FS.kalman_rows(m, x, eps, True))
            x, P = FS.kalman_measurement(m, x, P, r([sc.h(p) for p in rows]), y, R, eps, True)
            rows = r(FS.kalman_rows(m, x, eps, True))
            x, P = FS.kalman_prediction(m, P, r([sc.step(p, u) for p in rows]), Q, eps, True)
        out.append(x)
    return np.array(out)


def _device_run(sc, kind, alpha, eps, x0s, P0, Q, R, yss):
    B = len(x0s)
    est = _bank(sc, kind, B=B, alpha=alpha, epsilon=eps)
    for b in range(B):
        est.set(b, x0s[b], P0[b], 0.0)
        est.set_noise(b, Q[b], R[b])
    out = []
    for t in range(len(yss[0])):
        st = est.update(np.tile(_controls(t, sc.m.nu), (B, 1)), np.stack([ys[t] for ys in yss]))
        assert not st.any(), (t, st)
        out.append(np.stack([est.state(b) for b in range(B)]))
    return np.array(out).transpose(1, 0, 2)


@pytest.mark.parametrize("scene,kind,alpha", [("slide", "unscented", 1.0), ("slide", "unscented", 0.5),
                                              ("slide", "kalman", 1.0), ("free_ball", "unscented", 1.0)])
def test_end_to_end_against_the_exact_filter(scene, kind, alpha):
    sc = _scene(scene)
    B = 3 if scene == "slide" else 1
    eps = 1e-3
    P0, Q, R = _e2e_filters(sc, kind, alpha, B)
    x0s = [FS.plus(sc.m, sc.x0, 0.01 * (b + 1) * np.ones(2 * sc.m.nv)) for b in range(B)]
    yss = [_truth(sc, sc.x0, T_STEPS, 90 + b, 1e-2)[1] for b in range(B)]
    dev = _device_run(sc, kind, alpha, eps, x0s, P0, Q, R, yss)
    for b in range(B):
        exact = _restated_run(sc, kind, alpha, eps, x0s[b], P0[b], Q[b], R[b], yss[b], False)
        yard = _restated_run(sc, kind, alpha, eps, x0s[b], P0[b], Q[b], R[b], yss[b], True)
        e_dev = max(np.max(np.abs(FS.minus(sc.m, d, e))) for d, e in zip(dev[b], exact))
        e_yard = max(np.max(np.abs(FS.minus(sc.m, d, e))) for d, e in zip(yard, exact))
        REPORT[f"end to end {scene} {kind} alpha {alpha} filter {b}: device / float32 yardstick error"] = \
            (float(e_dev), float(e_yard))
        assert _ratio(f"end to end {scene} {kind}", e_dev, 16 * e_yard + 1e-9), (b, e_dev, e_yard)


def test_report_kalman_error_far_from_the_origin():
    """The Kalman perturbations x +- eps are rounded to float, so far from the origin the realised step differs from the
    nominal 2 eps that C and A divide by: reported, without a bar, with the slide at 1e2 m."""
    sc = _scene("slide")
    P0, Q, R = _e2e_filters(sc, "kalman", 1.0, 1)
    x0 = sc.x0 + np.array([100.0, 0.0, 0.0, 0.0])
    ys = _truth(sc, x0, T_STEPS, 99, 1e-2)[1]
    dev = _device_run(sc, "kalman", 1.0, 1e-3, [x0], P0, Q, R, [ys])[0]
    exact = _restated_run(sc, "kalman", 1.0, 1e-3, x0, P0[0], Q[0], R[0], ys, False)
    REPORT["kalman at 1e2 m: max |device - exact| state"] = float(np.max(np.abs(dev - exact)))


def test_zz_report():
    for k, v in sorted(RATIOS.items()):
        print(f"ratio {k}: {v:.3g}")
    for k, v in REPORT.items():
        print(f"{k}: {v}")
