"""The IMU sensors on the device (mjpc_b200_step_sensors) and the Kalman filter with its finite-difference steps on the
engine.

Bars.  gyro and velocimeter are fp32 velocity kinematics (cvel, a site offset and a rotation): against the fp64 sensor
oracle, teacher-forced at the same fp32 state, 1e-5.  The accelerometer adds the post-solve qacc, which comes from an
fp32 constraint solve when there are contacts: its bar is max(4 |fp32 - fp64|, 1e-4 |g|) with the fp32 sensor oracle as
the yardstick.  next_states / qacc / counts come from the same launch as mjpc_b200_step_batch's and must be bitwise
equal to them.  The C++ filter and its Python mirror run the same launches (both cast the same doubles to the same
fp32 kernel inputs), so they differ only by the order of double-precision sums: 1e-9 relative per update.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import OracleSigmaBackend, load_estimator_model, mocap_vector, sensor_oracle, simulate  # noqa: E402
from quadruped_filtering import plant, run_filter  # noqa: E402
from test_kalman_cpu import IMU_CHAIN_XML, IMU_FREE_XML, load_task_imu  # noqa: E402

from mujoco_mpc_b200.estimator import (CppKalman, CppUnscented, EngineBackend, EstimatorError, Kalman,  # noqa: E402
                                       Unscented)
from mujoco_mpc_b200.mjcf import SENS_ACCELEROMETER, compile_xml  # noqa: E402

pytestmark = pytest.mark.gpu

QUAD_IMU = ('<accelerometer site="torso"/><gyro site="torso"/><velocimeter site="torso"/>'
            '<accelerometer site="head"/><gyro site="head"/><velocimeter site="head"/>')


def _engine(m, n=128):
    from mujoco_mpc_b200.engine import Engine
    return Engine(m, n, 8, device=0)


def _quadruped_imu(monkeypatch):
    """The Quadruped with the three IMU sensors on its torso and head sites appended after its own sensors."""
    from mujoco_mpc_b200 import models
    xml = models.quadruped_flat_xml
    monkeypatch.setattr(models, "quadruped_flat_xml", lambda **kw: xml(**kw).replace("</sensor>", QUAD_IMU + "</sensor>"))
    m = models.load("quadruped")
    monkeypatch.setattr(models, "quadruped_flat_xml", xml)
    return m


def _states(m, rng, n=8):
    X = np.array([np.concatenate([m.qpos0 + 0.3 * rng.normal(size=m.nq), rng.normal(size=m.nv)]) for _ in range(n)])
    for j in range(m.njnt):
        if m.jnt_type[j] in (0, 1):
            a = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == 0 else 0)
            X[:, a:a + 4] /= np.linalg.norm(X[:, a:a + 4], axis=1)[:, None]
    return X


def _quadruped_states(m, T=96):
    """fp64 oracle trajectory of the A1 from the home key under a PD law plus seeded torques: contacts make and break."""
    k = m.key_names.index("home")
    rng = np.random.default_rng(1)
    o = sensor_oracle(m)
    x, w, mc = np.concatenate([m.key_qpos[k], np.zeros(m.nv)]), np.zeros(m.nv), mocap_vector(m)
    X, U, W = [], [], []
    for t in range(T):
        u = np.clip(2.0 * (m.key_qpos[k][7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:] + 0.6 * np.sin(0.2 * t + np.arange(12))
                    + 0.3 * rng.normal(size=m.nu), -1, 1)
        X.append(x); U.append(u); W.append(w)
        r = o.step(x[None, :m.nq], x[None, m.nq:], u[None], mc, [t * m.opt_timestep], m.nsensor - 6, 6,
                   warmstart=w[None])
        x, w = np.concatenate([r["next_qpos"][0], r["next_qvel"][0]]), r["qacc"][0]
    return np.array(X), np.array(U), np.array(W)


@pytest.mark.parametrize("scene,generic", [("chain", False), ("free", False), ("task_imu", False),
                                           ("quadruped", False), ("quadruped", True)])
def test_device_imu_sensors_against_the_oracle(monkeypatch, scene, generic):
    """Teacher-forced: device IMU sensors at given states against the fp64 sensor oracle, on the purpose-built scenes,
    the reference's task_imu and the Quadruped (its static instance, and the generic one with MJPC_B200_NO_STATIC=1)."""
    rng = np.random.default_rng(9)
    if scene == "quadruped":
        m = _quadruped_imu(monkeypatch)
        X, U, W = _quadruped_states(m)
        X, U, W = X[::6], U[::6], W[::6]
        start, n = m.nsensor - 6, 6
    else:
        m = load_task_imu() if scene == "task_imu" else compile_xml(IMU_CHAIN_XML if scene == "chain" else IMU_FREE_XML)
        X = _states(m, rng)
        U, W = rng.normal(size=(len(X), m.nu)), np.zeros((len(X), m.nv))
        start, n = 0, m.nsensor
    if generic:
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    e = _engine(m, n=16)
    o64, o32 = sensor_oracle(m, precision=64), sensor_oracle(m, precision=32)
    mc, g = mocap_vector(m), np.linalg.norm(m.opt_gravity)
    acc = np.array([m.sensor_type[i] == SENS_ACCELEROMETER for i in range(start, start + n) for _ in range(m.sensor_dim[i])])
    X32, W32 = X.astype(np.float32).astype(float), W.astype(np.float32).astype(float)
    worst = 0.0
    for i in range(len(X)):
        o = e.step_sensors(X32[i:i + 1], U[i], mc, 0.0, start, n, warmstart=W32[i:i + 1])
        if scene == "quadruped":
            assert e.last_kernel_static == (0 if generic else 1)
        r = e.step_batch(X32[i:i + 1, :m.nq], X32[i:i + 1, m.nq:], U[i:i + 1], mc, np.zeros(1), warmstart=W32[i:i + 1])
        assert np.array_equal(o["next_states"], np.concatenate([r["next_qpos"], r["next_qvel"]], axis=1))
        assert np.array_equal(o["qacc"], r["qacc"])
        for k in ("ncon", "nefc", "niter", "warning"):
            assert np.array_equal(o[k], r[k])
        args = (X32[i:i + 1, :m.nq], X32[i:i + 1, m.nq:], U[i:i + 1], mc, [0.0], start, n)
        y = o["sensordata"][0].astype(float)
        y64, y32 = o64.step(*args, warmstart=W32[i:i + 1])["sensordata"][0], o32.step(*args, warmstart=W32[i:i + 1])["sensordata"][0]
        assert np.max(np.abs(y[~acc] - y64[~acc])) < 1e-5, (i, np.abs(y - y64)[~acc].max())
        bar = np.maximum(4 * np.abs(y32[acc] - y64[acc]), 1e-4 * g)
        assert (np.abs(y[acc] - y64[acc]) <= bar).all(), (i, y[acc], y64[acc], y32[acc])
        worst = max(worst, float(np.abs(y[acc] - y64[acc]).max()))
    print("%s%s: max |accelerometer - fp64| %.3g" % (scene, " (generic)" if generic else "", worst))
    e.close()


def test_task_imu_accelerometer_reads_gravity_at_rest():
    m = load_task_imu()
    e = _engine(m, n=4)
    x, w = np.array([0.25, 0.0]), np.zeros((1, m.nv))
    for t in range(3000):
        o = e.step_sensors(x[None], np.zeros(m.nu), np.zeros(0), t * m.opt_timestep, 0, 2, warmstart=w)
        if t == 0:
            assert np.abs(o["sensordata"][0][1:]).max() < 1e-5    # free fall
        x, w = o["next_states"][0].astype(float), o["qacc"]
    g = np.linalg.norm(m.opt_gravity)
    assert np.abs(o["sensordata"][0][1:] - [0, 0, g]).max() < 1e-3 * g, o["sensordata"]
    e.close()


def _reference_kalman_test(m, f, T=200):
    """kalman_test.cc on filter f: the max error norms after update_measurement against the simulation's state t."""
    X, Y, U = simulate(m, [0.25], [0.0], T)
    f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
    ep = ev = 0.0
    for t in range(T):
        f.update_measurement(U[t], Y[t])
        s = f.state
        ep, ev = max(ep, np.linalg.norm(s[:m.nq] - X[t, :m.nq])), max(ev, np.linalg.norm(s[m.nq:] - X[t, m.nq:]))
        P = f.covariance
        assert np.array_equal(P, P.T)
        f.update_prediction()
    assert f.warnings == 0 and f.time == pytest.approx(T * m.opt_timestep)
    return ep, ev


def test_reference_kalman_test_on_the_engine():
    """kalman_test.cc with the Python mirror and with the C++ filter on the engine at the engine defaults, at the
    reference's 1e-4 (the fp32-oracle dry run, tests/test_kalman_cpu.py, meets it)."""
    m = load_task_imu()
    e = _engine(m, n=2 * 2 * m.nv + 1)
    for f in (Kalman(m, lambda s, n, ts: EngineBackend(e, s, n, ts)), CppKalman(m)):
        ep, ev = _reference_kalman_test(m, f)
        print("%s: max qpos error %.3g qvel error %.3g" % (type(f).__name__, ep, ev))
        assert ep <= 1e-4 and ev <= 1e-4, (ep, ev)
    e.close()


@pytest.mark.parametrize("name", ["task_imu", "box3drot", "quadruped"])
def test_cpp_kalman_against_python_mirror(name):
    """Per update from an identical (state, covariance, time): the C++ filter and the Python mirror, both on the
    engine, agree to 1e-9 relative in state and covariance."""
    if name == "quadruped":
        from mujoco_mpc_b200 import models
        m = models.load("quadruped")
        X, Y, U = plant(m)
        T = 10
    elif name == "box3drot":
        m = load_estimator_model(name)
        X, Y, U = simulate(m, m.qpos0, [1.0, -0.75, 1.25], 20)
        T = 19
    else:
        m = load_task_imu()
        X, Y, U = simulate(m, [0.25], [0.0], 20)
        T = 19
    mc = mocap_vector(m)
    e = _engine(m, n=4 * m.nv + 1)
    py = Kalman(m, lambda s, n, ts: EngineBackend(e, s, n, ts))
    cpp = CppKalman(m)
    py.reset(state=X[0]); cpp.reset(state=X[0])
    for t in range(T):
        cpp.set(py.state, py.covariance, py.time)
        py.update(U[t], Y[t], mc); cpp.update(U[t], Y[t], mc)
        xs, P = cpp.state, cpp.covariance
        assert np.max(np.abs(xs - py.state)) <= 1e-9 * max(1.0, np.abs(py.state).max()), t
        assert np.max(np.abs(P - py.covariance)) <= 1e-9 * np.abs(py.covariance).max(), t
        assert cpp.time == pytest.approx(py.time, abs=1e-15)
    cpp.close(); e.close()


def test_kalman_quadruped_filtering_against_the_oracle_plant():
    """The Quadruped scenario of tests/quadruped_filtering.py with the engine filters (Python and C++).  The covariance
    stays symmetric and positive definite with no step warnings, and the RMS qpos / qvel errors are within 5 % of the
    fp32-oracle Kalman filter's, widened by the spread between the fp32- and fp64-oracle filters (tests/test_kalman_cpu.py:
    linearised through contacts, this filter's errors move by 10-20 % with the step's rounding)."""
    from mujoco_mpc_b200 import models
    m = models.load("quadruped")
    X, Y, U = plant(m)
    mc = mocap_vector(m)
    ref = {p: run_filter(m, Kalman(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=p)), X, Y, U, mc)
           for p in (32, 64)}
    bar = [1.05 * ref[32][k] + abs(ref[32][k] - ref[64][k]) for k in (0, 1)]
    e = _engine(m, n=73)
    for f in (Kalman(m, lambda s, n, ts: EngineBackend(e, s, n, ts)), CppKalman(m)):
        assert (f.sensor_start, f.nsensor, f.timestep, f.nstates) == (9, 21, 0.005, 73)
        rq, rv, asym, mineig = run_filter(m, f, X, Y, U, mc)
        print("Kalman quadruped %s: RMS qpos %.4g qvel %.4g (fp32 oracle %.4g %.4g, fp64 oracle %.4g %.4g)"
              % (type(f).__name__, rq, rv, ref[32][0], ref[32][1], ref[64][0], ref[64][1]))
        assert asym == 0.0 and mineig > 0 and f.warnings == 0
        assert rq <= bar[0] and rv <= bar[1], (rq, rv, bar)
    e.close()


def _create_refusals(kind, cpp_filter):
    """<kind>_create itself refuses a range outside the model's sensors and one with a sensor the engine does not
    evaluate (the Python wrapper's measured_range check is bypassed to reach it); a failed sensor-covariance
    factorisation through the C++ filter leaves state, covariance and time untouched."""
    import ctypes as C
    from mujoco_mpc_b200 import models
    from mujoco_mpc_b200.engine import _model_blob, load_library
    lib = load_library()
    m = models.load("quadruped")
    _, mb = _model_blob(m)
    h = C.c_void_p()
    create = getattr(lib, "mjpc_b200_%s_create" % kind)
    settings = (C.c_double(1e-3), 1) if kind == "kalman" else (C.c_double(1.0), C.c_double(2.0))
    args = (C.c_double(0.005), *settings, 0, C.byref(h))
    assert create(C.byref(mb), 0, 10, *args) == -5 and not h.value      # user sensors
    assert create(C.byref(mb), 9, m.nsensor, *args) == -1 and not h.value
    assert create(C.byref(mb), -1, 2, *args) == -1 and not h.value
    p = load_task_imu()
    f = cpp_filter(p)
    f.reset(state=[0.25, 0.0], time=0.3)
    f.set_noise(sensor=np.full(f.nsensordata, -1.0))
    before = (f.state, f.covariance, f.time)
    with pytest.raises(EstimatorError, match="sensor covariance factorisation"):
        f.update(np.zeros(p.nu), [0.25, 0.0, 0.0, 0.0])
    assert np.array_equal(f.state, before[0]) and np.array_equal(f.covariance, before[1]) and f.time == before[2]
    f.close()


def test_kalman_create_refusals():
    _create_refusals("kalman", CppKalman)


def test_unscented_create_refusals():
    """The Unscented filter's create refuses the same inputs as the Kalman filter's: both are one-filter banks."""
    _create_refusals("unscented", CppUnscented)


def test_unscented_on_task_imu_through_the_new_sensors():
    """The Unscented filter, unchanged, measures task_imu's accelerometer on the engine in the reference's Kalman test
    scenario (state after update t against the simulation at t + 1).  Its sigma points straddle the ground at the impact,
    and with fp32 steps it cannot hold 1e-4 there: the fp32-oracle filter's errors reach about 9e-4 in qpos and 1.5e-2 in
    qvel.  The bar is the reference's 1e-4 or twice the fp32-oracle filter's error, whichever is larger."""
    m = load_task_imu()
    X, Y, U = simulate(m, [0.25], [0.0], 200)

    def errors(f):
        f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
        ep = ev = 0.0
        for t in range(199):
            f.update(U[t], Y[t])
            ep = max(ep, np.linalg.norm(f.state[:m.nq] - X[t + 1, :m.nq]))
            ev = max(ev, np.linalg.norm(f.state[m.nq:] - X[t + 1, m.nq:]))
        assert f.warnings == 0
        return ep, ev
    ref = errors(Unscented(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=32)))
    e = _engine(m, n=4 * m.nv + 1)
    ep, ev = errors(Unscented(m, lambda s, n, ts: EngineBackend(e, s, n, ts)))
    print("Unscented task_imu: max qpos error %.3g qvel %.3g (fp32 oracle %.3g %.3g)" % (ep, ev, ref[0], ref[1]))
    assert ep <= max(1e-4, 2 * ref[0]) and ev <= max(1e-4, 2 * ref[1]), (ep, ev, ref)
    e.close()
