"""The batched Kalman and Unscented filters (mujoco_mpc_b200.estimator.CppBatchEstimator): B filters per update, the
filter arithmetic in fp64 on the device, every filter's rows in one step launch per sigma-point set / Jacobian.

Bars.  The device restates the Python mirror filters' fp64 arithmetic (mujoco_mpc_b200.estimator.Unscented / Kalman)
and its step rows are the rows the mirror steps through EngineBackend, so from the same state, covariance, time, noise
and warm start the two are held to the 1e-9 relative that test_cpp_filter_against_python_mirror holds the single C++
filters to.  Free running, every filter of the batch meets the RMS bars the existing GPU tests set for the single filter
of its kind.  A filter's rows and its CTA read only its own inputs, so its results are bitwise the same at any position
of any batch, a failed factorisation leaves its filter bitwise unchanged, and a single C++ filter, the bank of one, is
bitwise the batch's filter given the same inputs.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import OracleSigmaBackend, load_estimator_model, mocap_vector, simulate  # noqa: E402
from quadruped_filtering import SENSOR_SD, STEPS, plant, run_filter  # noqa: E402
from test_kalman_cpu import load_task_imu  # noqa: E402

from mujoco_mpc_b200.engine import Engine, EngineError  # noqa: E402
from mujoco_mpc_b200.estimator import (CppBatchEstimator, CppKalman, CppUnscented, EngineBackend,  # noqa: E402
                                       EstimatorError, Kalman, Unscented)

pytestmark = pytest.mark.gpu

KINDS = ["unscented", "kalman"]
SINGLE = {"unscented": CppUnscented, "kalman": CppKalman}
MIRROR = {"unscented": Unscented, "kalman": Kalman}
BAD_ARGUMENT, BAD_BLOB, CAPACITY, UNSUPPORTED = -1, -2, -3, -5


def _quadruped():
    from mujoco_mpc_b200 import models
    return models.load("quadruped")


def _scenario(name):
    """(model, X, Y, U, updates) of the scenarios the single filters' mirror tests use."""
    if name == "quadruped":
        m = _quadruped()
        X, Y, U = plant(m)
        return m, X, Y, U, 10
    if name == "box3drot":
        m = load_estimator_model(name)
        X, Y, U = simulate(m, m.qpos0, [1.0, -0.75, 1.25], 20)
    else:
        m = load_task_imu()
        X, Y, U = simulate(m, [0.25], [0.0], 20)
    return m, X, Y, U, 19


def _tile(a, B):
    return np.tile(np.asarray(a, float).reshape(1, -1), (B, 1))


def _relative(x, P, f):
    """Largest relative differences of state x and covariance P from filter f's."""
    return (np.max(np.abs(x - f.state)) / max(1.0, np.abs(f.state).max()),
            np.max(np.abs(P - f.covariance)) / np.abs(f.covariance).max())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", ["box3drot", "task_imu", "quadruped"])
def test_teacher_forced_against_the_python_mirror(kind, name):
    """Per update from an identical (state, covariance, time): each of 3 batched filters, fed its own state and its
    own sensor noise, agrees with a Python mirror filter of its kind on EngineBackend to 1e-9 relative in state and
    covariance; time and warnings are equal."""
    m, X, Y, U, T = _scenario(name)
    mc = mocap_vector(m)
    B = 3
    batch = CppBatchEstimator(m, kind, B)
    e = Engine(m, batch.rows, 8, device=0)
    singles = [MIRROR[kind](m, lambda s, n, ts: EngineBackend(e, s, n, ts)) for _ in range(B)]
    for b, f in enumerate(singles):
        x0 = X[0].copy()
        x0[m.nq:] += 1e-3 * b            # each filter starts from its own velocity
        f.reset(state=x0)
        batch.reset(b, state=x0)
        if name == "quadruped":
            f.set_noise(sensor=np.full(f.nsensordata, SENSOR_SD ** 2 * (1 + b)))
            batch.set_noise(b, sensor=np.full(f.nsensordata, SENSOR_SD ** 2 * (1 + b)))
    worst = 0.0
    for t in range(T):
        for b, f in enumerate(singles):
            batch.set(b, f.state, f.covariance, f.time)
        status = batch.update(_tile(U[t], B), _tile(Y[t], B), _tile(mc, B) if mc.size else None)
        assert (status == 0).all(), status
        for b, f in enumerate(singles):
            f.update(U[t], Y[t], mc)
            x, P, tb, sc = batch.get(b)
            dx, dP = _relative(x, P, f)
            worst = max(worst, dx, dP)
            assert dx <= 1e-9 and dP <= 1e-9, (t, b, dx, dP)
            assert tb == f.time and int(sc[3]) == f.warnings
            assert np.array_equal(P, P.T)
    print("%s %s: largest relative difference from the Python mirror %.3g" % (kind, name, worst))
    expected = [2 * m.nv, batch.rows, batch.nsensordata, 0, batch.timestep] + ([batch.epsilon] if kind == "kalman" else [])
    assert list(batch.get(0)[3][[0, 1, 2, 4]]) == [expected[i] for i in (0, 1, 2, 4)]
    assert batch.rows == (singles[0].nsigma if kind == "unscented" else singles[0].nstates)
    batch.close(); e.close()


@pytest.mark.parametrize("kind", KINDS)
def test_quadruped_filtering_free_running(kind):
    """The 200-step Quadruped scenario of tests/quadruped_filtering.py with B = 8 batched filters, each persisting its
    state, covariance, time and warm start on the device.  Every filter keeps its covariance symmetric and positive
    definite with no step warnings and meets the single filter's RMS bars (tests/test_gpu_estimator.py,
    tests/test_gpu_kalman.py: within 5 % of the fp32-oracle filter, for the Kalman filter widened by the fp32 / fp64
    spread).  A single C++ filter fed the same inputs equals filter 0 bitwise at every step."""
    m = _quadruped()
    X, Y, U = plant(m)
    mc = mocap_vector(m)
    if kind == "unscented":
        ref = run_filter(m, Unscented(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=32)), X, Y, U, mc)
        bar = [1.05 * ref[0], 1.05 * ref[1]]
    else:
        ref = {p: run_filter(m, Kalman(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=p)), X, Y, U, mc)
               for p in (32, 64)}
        bar = [1.05 * ref[32][k] + abs(ref[32][k] - ref[64][k]) for k in (0, 1)]
    B = 8
    batch = CppBatchEstimator(m, kind, B)
    single = SINGLE[kind](m)
    assert (batch.sensor_start, batch.nsensor, batch.timestep, batch.rows) == (9, 21, 0.005, 73)
    single.reset(state=X[0])
    single.set_noise(sensor=np.full(single.nsensordata, SENSOR_SD ** 2))
    for b in range(B):
        batch.reset(b, state=X[0])
        batch.set_noise(b, sensor=np.full(batch.nsensordata, SENSOR_SD ** 2))
    eq, ev = [[] for _ in range(B)], [[] for _ in range(B)]
    asym, mineig = 0.0, np.inf
    for t in range(STEPS):
        status = batch.update(_tile(U[t], B), _tile(Y[t], B), _tile(mc, B))
        assert (status == 0).all(), (t, status)
        single.update(U[t], Y[t], mc)
        for b in range(B):
            x, P, tb, _ = batch.get(b)
            if b == 0:
                assert np.array_equal(x, single.state) and np.array_equal(P, single.covariance), t
                assert tb == single.time and batch.warnings(0) == single.warnings, t
            eq[b].append(x[:m.nq] - X[t + 1, :m.nq]); ev[b].append(x[m.nq:] - X[t + 1, m.nq:])
            asym = max(asym, float(np.abs(P - P.T).max()))
            mineig = min(mineig, float(np.linalg.eigvalsh(0.5 * (P + P.T)).min()))
            assert tb == pytest.approx((t + 1) * 0.005, abs=1e-12)
    for b in range(B):
        rq = float(np.sqrt(np.mean(np.square(eq[b][50:]))))
        rv = float(np.sqrt(np.mean(np.square(ev[b][50:]))))
        assert rq <= bar[0] and rv <= bar[1], (b, rq, rv, bar)
        assert batch.warnings(b) == 0
    print("batched %s quadruped: RMS qpos %.4g qvel %.4g (bars %.4g %.4g)" % (kind, rq, rv, bar[0], bar[1]))
    assert asym == 0.0 and mineig > 0
    single.close(); batch.close()


@pytest.mark.parametrize("kind", KINDS)
def test_single_filter_is_the_one_filter_bank(kind):
    """A single C++ filter and a batch of one, given the same inputs, agree bitwise over 5 Quadruped updates.  The
    Kalman filter's update_measurement and update_prediction, run separately, follow the Python mirror on EngineBackend
    teacher-forced to 1e-9 relative, through a prediction straight after reset (the ctrl and mocap of the last
    measurement are then zeros and the model's) and a prediction after a failed measurement (it steps with the last
    successful measurement's ctrl and mocap)."""
    m = _quadruped()
    X, Y, U = plant(m)
    mc = mocap_vector(m)
    single, batch = SINGLE[kind](m), CppBatchEstimator(m, kind, 1)
    noise = np.full(single.nsensordata, SENSOR_SD ** 2)
    single.reset(state=X[0]); single.set_noise(sensor=noise)
    batch.reset(0, state=X[0]); batch.set_noise(0, sensor=noise)
    for t in range(5):
        assert (batch.update(U[t][None], Y[t][None], mc[None]) == 0).all()
        single.update(U[t], Y[t], mc)
        x, P, tb, sc = batch.get(0)
        assert np.array_equal(x, single.state) and np.array_equal(P, single.covariance), t
        assert tb == single.time and int(sc[3]) == single.warnings, t
    batch.close()
    if kind == "unscented":
        single.close()
        return
    e = Engine(m, single.nstates, 8, device=0)
    py = Kalman(m, lambda s, n, ts: EngineBackend(e, s, n, ts))
    for f in (py, single):
        f.reset(state=X[0]); f.set_noise(sensor=noise)
    worst = 0.0

    def step(call, *args):
        nonlocal worst
        single.set(py.state, py.covariance, py.time)
        getattr(py, call)(*args); getattr(single, call)(*args)
        dx, dP = _relative(single.state, single.covariance, py)
        worst = max(worst, dx, dP)
        assert dx <= 1e-9 and dP <= 1e-9, (call, dx, dP)
        assert single.time == py.time and single.warnings == py.warnings

    step("update_prediction")                           # straight after reset
    for t in range(3):
        step("update_measurement", U[t], Y[t], mc)
        step("update_prediction")
    for f in (py, single):                              # a measurement that fails, then a prediction
        f.set_noise(sensor=np.full(single.nsensordata, -1e9))
        before = (f.state, f.covariance, f.time)
        with pytest.raises(EstimatorError, match="sensor covariance factorisation"):
            f.update_measurement(U[3], Y[3], mc)
        assert np.array_equal(f.state, before[0]) and np.array_equal(f.covariance, before[1]) and f.time == before[2]
        f.set_noise(sensor=noise)
    step("update_prediction")
    step("update_measurement", U[4], Y[4], mc)
    print("Kalman measurement / prediction: largest relative difference from the Python mirror %.3g" % worst)
    single.close(); e.close()


def _inputs(m, X, Y, U, B, t, rng):
    """Per-filter inputs of update t for a batch of B: filter b's rows of the scenario, perturbed by filter."""
    u = np.stack([U[(t + 3 * b) % len(U)] for b in range(B)])
    y = np.stack([Y[(t + 3 * b) % len(Y)] for b in range(B)]) + 1e-4 * rng.normal(size=(B, Y.shape[1]))
    mc = _tile(mocap_vector(m), B)
    if mc.size:
        mc[:, :3] += 1e-2 * rng.normal(size=(B, 3))
    return u, y, mc


def _prepare(m, X, f, p, b):
    """Filter p of a batch: the start state and noise of scenario filter b."""
    f.reset(p, state=X[(5 * b) % len(X)], covariance_scale=1e-4 * (1 + 0.5 * b))
    f.set_noise(p, process=np.full(2 * m.nv, 1e-4 * (1 + b)), sensor=np.full(f.nsensordata, SENSOR_SD ** 2 * (1 + b)))


@pytest.mark.parametrize("kind", KINDS)
def test_filters_are_independent(kind):
    """Filter 2's results after each of 5 updates are bitwise the same whether it runs alone (B = 1) or at position
    0, 5 or 7 of a batch of 8 whose other filters have other states, noises, ctrl, sensors and mocap."""
    m = _quadruped()
    X, Y, U = plant(m)
    T, src = 5, 2

    def run(B, pos):
        f = CppBatchEstimator(m, kind, B)
        rng = np.random.default_rng(11)
        order = [b for b in range(8) if b != src][:B - 1]
        order.insert(pos, src)                       # order[p] = which scenario filter p runs
        for p, b in enumerate(order):
            _prepare(m, X, f, p, b)
        out = []
        for t in range(T):
            u, y, mc = _inputs(m, X, Y, U, 8, t, rng)
            status = f.update(u[order], y[order], mc[order])
            assert (status == 0).all()
            out.append(f.get(pos))
        f.close()
        return out

    alone = run(1, 0)
    for pos in (0, 5, 7):
        batched = run(8, pos)
        for a, c in zip(alone, batched):
            assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) and a[2] == c[2], pos
            assert np.array_equal(a[3], c[3]), pos


@pytest.mark.parametrize("kind", KINDS)
def test_failed_factorisation_is_isolated(kind):
    """Filter 3's covariance set to -I: status[3] is MJPC_B200_ERR_BAD_ARGUMENT (Unscented: the covariance factor;
    Kalman: the sensor covariance C P C' + R), filter 3 is bitwise unchanged, and every other filter is bitwise equal to
    a run where filter 3 was healthy."""
    m = _quadruped()
    X, Y, U = plant(m)
    B = 8

    def run(broken):
        f = CppBatchEstimator(m, kind, B)
        for b in range(B):
            _prepare(m, X, f, b, b)
        if broken:
            x3, _, t3, _ = f.get(3)
            f.set(3, x3, -np.eye(2 * m.nv), t3)
        before = f.get(3)
        rng = np.random.default_rng(4)
        status = None
        for t in range(3):
            status = f.update(*_inputs(m, X, Y, U, B, t, rng))
        out = [f.get(b) for b in range(B)]
        f.close()
        return before, status, out

    before, status, broken = run(True)
    _, status_ok, healthy = run(False)
    assert status[3] == BAD_ARGUMENT and (np.delete(status, 3) == 0).all(), status
    assert (status_ok == 0).all()
    assert all(np.array_equal(a, c) for a, c in zip(before[:2], broken[3][:2])) and before[2] == broken[3][2]
    assert np.array_equal(before[3], broken[3][3])
    for b in range(B):
        if b != 3:
            assert all(np.array_equal(a, c) for a, c in zip(broken[b], healthy[b])), b


def test_create_and_call_refusals():
    """create refuses what the single creates refuse, on the device as on the host: a sensor the engine does not
    evaluate (the Quadruped's user sensors), a range outside the model's sensors, a bad blob, and more step rows than
    one handle holds; calls with a filter index outside [0, B) are refused."""
    import ctypes as C
    from mujoco_mpc_b200.engine import _model_blob, load_library
    lib = load_library()
    m = _quadruped()
    _, mb = _model_blob(m)
    h = C.c_void_p()
    create = lib.mjpc_b200_batch_estimator_create
    for kind, prm in ((1, (1e-3, 1.0)), (2, (1.0, 2.0))):
        s = (C.c_double * 2)(*prm)
        assert create(C.byref(mb), kind, 2, 0, 10, C.c_double(0.005), s, 0, C.byref(h)) == UNSUPPORTED and not h.value
        assert create(C.byref(mb), kind, 2, 9, m.nsensor, C.c_double(0.005), s, 0, C.byref(h)) == BAD_ARGUMENT
        assert create(C.byref(mb), kind, 65536 // 73 + 1, 9, 21, C.c_double(0.005), s, 0, C.byref(h)) == CAPACITY
        assert not h.value
    f = CppBatchEstimator(m, "unscented", 2)
    with pytest.raises(EngineError):
        f.get(2)
    with pytest.raises(EngineError):
        f.reset(-1)
    f.close()
