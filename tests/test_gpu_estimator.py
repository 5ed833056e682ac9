"""Measurement sensors on the device (mjpc_b200_step_sensors) and the Unscented filter with its sigma-point steps on
the engine.

Bars.  jointpos / jointvel copy the fp32 state the kernel was given, so they must equal it exactly.  framepos is fp32
forward kinematics: every body position is a chain of at most 4 rotate-and-add steps of fp32 quaternion products, each
rounding at 2^-24 relative of operands below 1 m, so the world position of an A1 foot carries a few 1e-7 m; with the
fp32 rounding of the input quaternion this stays below 2e-6 m, and the bar is 1e-5 m against the fp64 kinematics.
Touch is checked against the fp64 sensor oracle teacher-forced, with the fp32 oracle as the yardstick: a touch reading
is a sum of constraint forces from an fp32 Newton solve, so the device may differ from fp64 by what fp32 rounding does
to the solve, bar max(4 |fp32 - fp64|, 2e-3 |fp64| + 1e-3 N) where the device and the oracle found the same contacts;
and against physics: a body at rest on flat ground presses with its weight, m |g| (bar 2e-3 relative).
The C++ filter and its Python mirror are fed the same sigma-point steps (both cast the same doubles to the same fp32
kernel inputs), so they differ only by the order of double-precision sums: 1e-9 relative per update.  next_states / qacc / counts of step_sensors come from the same kernel launch as
those of mjpc_b200_step_batch and must be bitwise equal to them.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import (FRAMES_XML, OracleSigmaBackend, TOUCH_XML, load_estimator_model, mocap_vector,  # noqa: E402
                                quat_error, sensor_oracle, sensors_fp64, settle, simulate)
from quadruped_filtering import plant, run_filter  # noqa: E402

from mujoco_mpc_b200.estimator import CppUnscented, EngineBackend, EstimatorError, Unscented  # noqa: E402
from mujoco_mpc_b200.mjcf import compile_xml  # noqa: E402

pytestmark = pytest.mark.gpu


def _engine(m, n=128):
    from mujoco_mpc_b200.engine import Engine
    return Engine(m, n, 8, device=0)


def _quadruped():
    from mujoco_mpc_b200 import models
    return models.load("quadruped")


def _quadruped_states(m, T=120, seed=0):
    """Oracle trajectory of the A1 from the home key under seeded random torques: feet make and break contact."""
    rng = np.random.default_rng(seed)
    k = m.key_names.index("home")
    q, v = m.key_qpos[k].copy(), np.zeros(m.nv)
    from oracle import pyoracle
    from mujoco_mpc_b200.blob import to_blob
    o = pyoracle.Oracle(to_blob(m), m, 64)
    mc = mocap_vector(m)
    X, U, W = [], [], []
    w = np.zeros(m.nv)
    for t in range(T):
        u = np.clip(2.0 * (m.key_qpos[k][7:] - q[7:]) - 0.1 * v[6:] + 0.6 * np.sin(0.2 * t + np.arange(12)), -1, 1)
        u = np.clip(u + 0.3 * rng.normal(size=m.nu), -1, 1)
        X.append(np.concatenate([q, v])); U.append(u); W.append(w)
        r = o.step_batch(q[None], v[None], u[None], mc, [t * m.opt_timestep], warmstart=w[None])
        q, v, w = r["next_qpos"][0], r["next_qvel"][0], r["qacc"][0]
    return np.array(X), np.array(U), np.array(W)


@pytest.mark.parametrize("generic", [False, True])
def test_step_sensors_equals_step_batch_and_fp64_kinematics(monkeypatch, generic):
    if generic:
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = _quadruped()
    e = _engine(m)
    X, U, W = _quadruped_states(m)
    s0, n = 9, 21
    o64, o32 = sensor_oracle(m, precision=64), sensor_oracle(m, precision=32)
    touched = compared = 0
    mc = mocap_vector(m)
    idx = np.arange(0, len(X), 8)
    for i in idx:
        xs = np.repeat(X[i:i + 1], 3, axis=0)
        o = e.step_sensors(xs, U[i], mc, 0.1, s0, n, warmstart=np.repeat(W[i:i + 1], 3, axis=0))
        assert e.last_kernel_static == (0 if generic else 1)
        r = e.step_batch(xs[:, :m.nq], xs[:, m.nq:], np.repeat(U[i:i + 1], 3, axis=0), mc, np.full(3, 0.1),
                         warmstart=np.repeat(W[i:i + 1], 3, axis=0))
        assert np.array_equal(o["next_states"], np.concatenate([r["next_qpos"], r["next_qvel"]], axis=1))
        assert np.array_equal(o["qacc"], r["qacc"])
        for k in ("ncon", "nefc", "niter", "warning"):
            assert np.array_equal(o[k], r[k])
        x32 = X[i].astype(np.float32).astype(float)
        ref = sensors_fp64(m, x32[:m.nq], x32[m.nq:], s0, 17, mc)
        y = o["sensordata"][0].astype(float)
        assert np.max(np.abs(y[:15] - ref[:15])) < 1e-5
        assert np.array_equal(y[15:27], ref[15:27])
        # touch against the fp64 sensor oracle, fp32 oracle as the yardstick
        args = (x32[None, :m.nq], x32[None, m.nq:], U[i:i + 1], mc, [0.1], s0, n)
        r64 = o64.step(*args, warmstart=W[i:i + 1].astype(np.float32).astype(float))
        r32 = o32.step(*args, warmstart=W[i:i + 1].astype(np.float32).astype(float))
        assert np.max(np.abs(y[:27] - r64["sensordata"][0][:27])) < 1e-5
        if o["ncon"][0] == r64["ncon"][0]:
            t64, t32, td = r64["sensordata"][0][27:], r32["sensordata"][0][27:], y[27:]
            bar = np.maximum(4 * np.abs(t32 - t64), 2e-3 * np.abs(t64) + 1e-3)
            assert (np.abs(td - t64) <= bar).all(), (td, t64, t32)
            touched += int((t64 > 0).sum()); compared += 1
    assert compared >= len(idx) // 2 and touched > 0
    e.close()


def test_touch_rest_weight_of_the_a1():
    """The A1 held at its home pose by a joint PD law settles on flat ground on its feet: the four foot touch sensors
    then read the robot's weight."""
    m = _quadruped()
    e = _engine(m)
    e.set_options(0.005)
    k = m.key_names.index("home")
    x = np.concatenate([m.key_qpos[k], np.zeros(m.nv)])
    w = np.zeros((1, m.nv))
    mc = mocap_vector(m)
    for t in range(300):
        u = np.clip(2.0 * (m.key_qpos[k][7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:], -1, 1)
        o = e.step_sensors(x[None], u, mc, t * 0.005, 26, 4, warmstart=w)
        x, w = o["next_states"][0].astype(float), o["qacc"]
    touch = o["sensordata"][0]
    weight = m.body_subtreemass[m.body_names.index("trunk")] * np.linalg.norm(m.opt_gravity)
    assert np.abs(x[m.nq:]).max() < 0.05 and (touch > 0).all()
    assert abs(touch.sum() - weight) < 2e-3 * weight, (touch, weight)
    e.close()


def _touch_scene(cone):
    return compile_xml(f"""
<mujoco model="touch scene">
  <option timestep="0.002" cone="{cone}"/>
  <worldbody>
    <geom name="floor" type="plane" size="1 1 .1"/>
    <body name="other" mocap="true" pos="0.3 0 0.3">
      <site name="other" type="sphere" size="1"/>
    </body>
    <body name="ball" pos="0 0 0.05">
      <freejoint/>
      <geom name="ball" type="sphere" size="0.05" mass="1"/>
      <site name="inside" type="sphere" size="0.08"/>
      <site name="ray" type="sphere" size="0.01"/>
      <site name="miss" type="sphere" size="0.01" pos="0.03 0 0"/>
      <site name="boxzone" type="box" size="0.01 0.01 0.01"/>
    </body>
  </worldbody>
  <sensor>
    <touch site="inside"/><touch site="ray"/><touch site="miss"/><touch site="other"/><touch site="boxzone"/>
  </sensor>
</mujoco>""")


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_touch_scenes(cone):
    """A 1 kg ball at rest on a plane: the contact point inside the zone and the ray into the ball hitting the zone
    both read m |g|; a zone beside the ray and a zone of another body (which contains the contact point) read 0."""
    from mujoco_mpc_b200.engine import EngineError
    m = _touch_scene(cone)
    e = _engine(m)
    x = np.concatenate([m.qpos0, np.zeros(m.nv)])
    w = np.zeros((1, m.nv))
    mc = mocap_vector(m)
    for t in range(500):
        o = e.step_sensors(x[None], np.zeros(0), mc, t * 0.002, 0, 4, warmstart=w)
        x, w = o["next_states"][0].astype(float), o["qacc"]
    y = o["sensordata"][0]
    g = np.linalg.norm(m.opt_gravity)
    assert o["ncon"][0] == 1
    assert abs(y[0] - g) < 2e-3 * g and abs(y[1] - g) < 2e-3 * g, y
    assert y[2] == 0 and y[3] == 0, y
    with pytest.raises(EngineError, match="-5.*touch zone"):
        e.step_sensors(x[None], np.zeros(0), mc, 0.0, 0, 5)
    e.close()


def test_step_sensors_error_paths():
    from mujoco_mpc_b200.engine import EngineError
    m = _quadruped()
    e = _engine(m, n=16)
    x = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])[None]
    mc, u = mocap_vector(m), np.zeros(m.nu)
    with pytest.raises(EngineError, match="-5.*sensor 0"):
        e.step_sensors(x, u, mc, 0.0, 0, 10)                     # user sensors (cost terms) are not evaluated
    with pytest.raises(EngineError, match="-1.*outside"):
        e.step_sensors(x, u, mc, 0.0, 9, m.nsensor)
    with pytest.raises(EngineError, match="-1.*outside"):
        e.step_sensors(x, u, mc, 0.0, -1, 2)
    with pytest.raises(EngineError, match="-3"):
        e.step_sensors(np.repeat(x, 17, axis=0), u, mc, 0.0, 9, 21)
    e.close()


CASES = [("particle1d", [0.25], [0.0], 5), ("box3drot", None, [1.0, -0.75, 1.25], 100)]


@pytest.mark.parametrize("name,q0,v0,T", CASES)
def test_reference_unscented_tests_on_the_engine(name, q0, v0, T):
    """unscented_test.cc Particle1D / Box3Drot with the sigma points stepped by the engine, the plant the fp64 oracle,
    at the reference's 1e-4."""
    m = load_estimator_model(name)
    X, Y, _ = simulate(m, m.qpos0 if q0 is None else np.array(q0), np.array(v0), T)
    e = _engine(m, n=32)
    f = Unscented(m, lambda s, n, ts: EngineBackend(e, s, n, ts))
    assert f.nsigma == 2 * 2 * m.nv + 1
    f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
    for t in range(T - 1):
        f.update(np.zeros(m.nu), Y[t])
        if name == "box3drot":
            ep = np.linalg.norm(quat_error(m, f.state[:m.nq], X[t + 1, :m.nq]))
        else:
            ep = np.linalg.norm(f.state[:m.nq] - X[t + 1, :m.nq])
        ev = np.linalg.norm(f.state[m.nq:] - X[t + 1, m.nq:])
        assert ep <= 1e-4 and ev <= 1e-4, (t, ep, ev)
        assert np.array_equal(f.covariance, f.covariance.T)
        np.linalg.cholesky(f.covariance)
    assert f.warnings == 0 and f.backend.last_kernel_ms > 0
    # a failed covariance factorisation leaves the filter as it was
    f.covariance = -np.eye(f.ndstate)
    before = (f.state.copy(), f.time)
    with pytest.raises(EstimatorError, match="covariance factorisation"):
        f.update(np.zeros(m.nu), Y[0])
    assert np.array_equal(f.state, before[0]) and f.time == before[1]
    e.close()


@pytest.mark.parametrize("scene", ["frames", "particle1d", "box3drot", "touch_pyramidal", "touch_elliptic"])
def test_device_sensors_against_the_oracle(scene):
    """Teacher-forced: device sensors at given states against the fp64 sensor oracle - every framepos object type
    (purpose-built scene), the reference's estimator models, and the settled touch scenes."""
    rng = np.random.default_rng(4)
    if scene == "frames":
        m = compile_xml(FRAMES_XML)
    elif scene.startswith("touch"):
        m = compile_xml(TOUCH_XML.format(cone=scene.split("_")[1]))
    else:
        m = load_estimator_model(scene)
    n = 4 if scene.startswith("touch") else m.nsensor
    e, o64 = _engine(m, n=16), sensor_oracle(m)
    mc = mocap_vector(m)
    if scene.startswith("touch"):
        x, w = settle(lambda x, w, t: o64.step(x[None, :m.nq], x[None, m.nq:], np.zeros((1, 0)), mc, [t], 0, n,
                                               warmstart=w), m, 500, 0.002)
        X, Wm = x[None], w
    else:
        X = np.array([np.concatenate([m.qpos0 + 0.3 * rng.normal(size=m.nq), rng.normal(size=m.nv)]) for _ in range(8)])
        for j in range(m.njnt):
            if m.jnt_type[j] == 1:
                a = m.jnt_qposadr[j]
                X[:, a:a + 4] /= np.linalg.norm(X[:, a:a + 4], axis=1)[:, None]
        Wm = None
    X32 = X.astype(np.float32).astype(float)
    u = np.zeros(m.nu)
    o = e.step_sensors(X32, u, mc, 0.0, 0, n, warmstart=Wm)
    r = o64.step(X32[:, :m.nq], X32[:, m.nq:], np.zeros((len(X), m.nu)), mc, np.zeros(len(X)), 0, n,
                 warmstart=None if Wm is None else Wm.astype(np.float32).astype(float))
    y, ref = o["sensordata"].astype(float), r["sensordata"]
    if scene.startswith("touch"):
        g = np.linalg.norm(m.opt_gravity)
        assert np.max(np.abs(y - ref)) < 2e-3 * g and ref[0, 2] == ref[0, 3] == y[0, 2] == y[0, 3] == 0, (y, ref)
    else:
        assert np.max(np.abs(y - ref)) < 1e-5, np.abs(y - ref).max()
    e.close()


@pytest.mark.parametrize("name", ["particle1d", "box3drot", "quadruped"])
def test_cpp_filter_against_python_mirror(name):
    """Per update from an identical (state, covariance, time): the C++ filter and the Python mirror, both on the
    engine, agree to 1e-9 relative in state and covariance."""
    if name == "quadruped":
        m = _quadruped()
        X, Y, U = plant(m)
        T = 10
    else:
        m = load_estimator_model(name)
        X, Y, U = simulate(m, m.qpos0 if name == "box3drot" else [0.25], [1.0, -0.75, 1.25] if name == "box3drot"
                           else [0.0], 20)
        T = 19
    mc = mocap_vector(m)
    e = _engine(m, n=4 * m.nv + 1)
    py = Unscented(m, lambda s, n, ts: EngineBackend(e, s, n, ts))
    cpp = CppUnscented(m)
    py.reset(state=X[0]); cpp.reset(state=X[0])
    for t in range(T):
        cpp.set(py.state, py.covariance, py.time)
        py.update(U[t], Y[t], mc); cpp.update(U[t], Y[t], mc)
        xs, P = cpp.state, cpp.covariance
        assert np.max(np.abs(xs - py.state)) <= 1e-9 * max(1.0, np.abs(py.state).max()), t
        assert np.max(np.abs(P - py.covariance)) <= 1e-9 * np.abs(py.covariance).max(), t
        assert cpp.time == pytest.approx(py.time, abs=1e-15)
    # a failed covariance factorisation leaves the C++ filter as it was
    cpp.set(py.state, -np.eye(cpp.ndstate), py.time)
    before = cpp.state
    with pytest.raises(EstimatorError, match="covariance factorisation"):
        cpp.update(U[0], Y[0], mc)
    assert np.array_equal(cpp.state, before) and cpp.time == py.time
    cpp.close(); e.close()


@pytest.mark.parametrize("name,q0,v0,T", CASES)
def test_reference_unscented_tests_on_the_cpp_filter(name, q0, v0, T):
    """unscented_test.cc Particle1D / Box3Drot on the C++ filter, the plant the fp64 oracle, at the reference's 1e-4."""
    m = load_estimator_model(name)
    X, Y, _ = simulate(m, m.qpos0 if q0 is None else np.array(q0), np.array(v0), T)
    f = CppUnscented(m)
    f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
    for t in range(T - 1):
        f.update(np.zeros(m.nu), Y[t])
        s = f.state
        ep = np.linalg.norm(quat_error(m, s[:m.nq], X[t + 1, :m.nq]) if name == "box3drot" else s[:m.nq] - X[t + 1, :m.nq])
        assert ep <= 1e-4 and np.linalg.norm(s[m.nq:] - X[t + 1, m.nq:]) <= 1e-4, t
    assert f.warnings == 0
    f.close()


def test_quadruped_filtering_against_the_oracle_plant():
    """The Quadruped scenario of tests/quadruped_filtering.py: the fp64 oracle is the plant, the 21 estimator sensors
    (touch included) carry seeded noise.  The Python and the C++ filter on the engine keep the covariance symmetric and
    positive definite at every step, and their RMS qpos / qvel errors are within 5 % of the filter whose sigma points
    the fp32 oracle steps (the bar test_estimator_cpu.py derives: fp32 and fp64 oracle filters agree to 1e-3)."""
    m = _quadruped()
    X, Y, U = plant(m)
    mc = mocap_vector(m)
    ref = run_filter(m, Unscented(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=32)), X, Y, U, mc)
    e = _engine(m, n=73)
    for f in (Unscented(m, lambda s, n, ts: EngineBackend(e, s, n, ts)), CppUnscented(m)):
        assert (f.sensor_start, f.nsensor, f.timestep, f.nsigma) == (9, 21, 0.005, 73)
        rq, rv, asym, mineig = run_filter(m, f, X, Y, U, mc)
        print("quadruped filter RMS qpos %.4g qvel %.4g (fp32 oracle %.4g %.4g)" % (rq, rv, ref[0], ref[1]))
        assert asym == 0.0 and mineig > 0
        assert rq <= 1.05 * ref[0] and rv <= 1.05 * ref[1], (rq, rv, ref)
        assert f.warnings == 0
    e.close()
