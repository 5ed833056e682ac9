"""GPU: the frame, subtree, ball-joint, actuator and tendon sensors of the device (mjpc_b200_step_sensors, the plant
bank, the filter banks) against the fp64 sensor oracle, and the refusals of the sensors the device does not evaluate.

Bars.  Teacher-forced, the device and the oracle start from the same fp32-rounded state; the fp32 sensor oracle is the
yardstick of what fp32 arithmetic does to each reading.  A reading is held to max(4 |fp32 - fp64|, floor), where the
device and the oracle found the same contacts.  The floor is 1e-3 (1 + |fp64|) for the readings that go through qacc,
and so through the constraint solve (accelerometer, framelinacc, frameangacc).  Every other reading, the actuator and
joint-actuator forces included, is computed from qpos, qvel and ctrl alone, and its floor is 2e-5 (1 + |fp64|).
Plant-bank sensor outputs come from the same k_sensors code as step_sensors on the same inputs, so they are bitwise
equal.  The filters follow tests/test_gpu_batch_estimator.py: 1e-9 relative from the Python mirror per update, bitwise
between a bank and single filters, and an RMS state error within 5 % (plus the fp32 / fp64 spread) of the filter whose
sigma points / Jacobians the fp32 oracle steps; for the Kalman filter with the accelerometer, of the worse of two fp32
realisations (see test_imu_filters).
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import OracleSigmaBackend, mocap_vector, sensor_oracle  # noqa: E402
from sensor_scenes import ROTATIONS, SCENES, imu_body, imu_plant, load_augmented, random_states, scene  # noqa: E402

from mujoco_mpc_b200.mjcf import compile_xml  # noqa: E402

pytestmark = pytest.mark.gpu

# readings that go through qacc (accelerometer, framelinacc, frameangacc)
ACCELERATION_TYPES = {10, 17, 18}


def _engine(m, n=32):
    from mujoco_mpc_b200.engine import Engine
    return Engine(m, n, 8, device=0)


def _bars(m, start, count, y64, y32):
    loose = np.concatenate([np.full(int(m.sensor_dim[i]), int(m.sensor_type[i]) in ACCELERATION_TYPES)
                            for i in range(start, start + count)])
    floor = np.where(loose, 1e-3, 2e-5) * (1 + np.abs(y64))
    return np.maximum(4 * np.abs(y32 - y64), floor)


def _compare(m, e, X, U, W, start, count, mc, what):
    """step_sensors at the states X (controls U, warm starts W) against the fp64 sensor oracle; returns the number of
    states compared (same contact count) and the worst reading / bar"""
    o64, o32 = sensor_oracle(m, precision=64), sensor_oracle(m, precision=32)
    X32 = X.astype(np.float32).astype(float)
    W32 = None if W is None else W.astype(np.float32).astype(float)
    U32 = U.astype(np.float32).astype(float)
    t = np.zeros(len(X))
    args = (X32[:, :m.nq], X32[:, m.nq:], U32, mc, t, start, count)
    r64, r32 = o64.step(*args, warmstart=W32), o32.step(*args, warmstart=W32)
    compared, worst = 0, 0.0
    for b in range(len(X)):
        o = e.step_sensors(X32[b:b + 1], U32[b], mc, 0.0, start, count, warmstart=None if W32 is None else W32[b:b + 1])
        if o["ncon"][0] != r64["ncon"][b]:
            continue
        y, y64, y32 = o["sensordata"][0].astype(float), r64["sensordata"][b], r32["sensordata"][b]
        bar = _bars(m, start, count, y64, y32)
        worst = max(worst, float(np.max(np.abs(y - y64) / bar)))
        bad = np.nonzero(np.abs(y - y64) > bar)[0]
        assert bad.size == 0, (what, b, bad, y[bad], y64[bad], y32[bad])
        compared += 1
    print("%s: %d states, worst |device - fp64| / bar %.3g" % (what, compared, worst))
    return compared


@pytest.mark.parametrize("name", sorted(SCENES))
@pytest.mark.parametrize("rot", range(len(ROTATIONS)))
def test_scene_sensors_against_the_oracle(name, rot):
    m = scene(name, ROTATIONS[rot])
    e = _engine(m)
    X = random_states(m, 8, seed=10 + rot)
    U = np.random.default_rng(rot).uniform(-1.2, 1.2, size=(len(X), m.nu))
    assert _compare(m, e, X, U, None, 0, m.nsensor, np.zeros(0), "%s rot %d" % (name, rot)) == len(X)
    e.close()


def _trajectory(m, x0, T, ctrl, seed=0):
    """fp64 oracle trajectory (states, controls, warm starts) from x0 under ctrl(t, x, rng)"""
    from oracle import pyoracle
    from mujoco_mpc_b200.blob import to_blob
    o = pyoracle.Oracle(to_blob(m), m, 64)
    rng = np.random.default_rng(seed)
    mc = mocap_vector(m)
    q, v, w = x0[:m.nq].copy(), x0[m.nq:].copy(), np.zeros(m.nv)
    X, U, W = [], [], []
    for t in range(T):
        u = ctrl(t, np.concatenate([q, v]), rng)
        X.append(np.concatenate([q, v])); U.append(u); W.append(w)
        r = o.step_batch(q[None], v[None], u[None], mc, [t * m.opt_timestep], warmstart=w[None])
        q, v, w = r["next_qpos"][0], r["next_qvel"][0], r["qacc"][0]
    return np.array(X), np.array(U), np.array(W)


@pytest.mark.parametrize("case", ["quadruped", "quadruped-generic", "humanoid_track", "shadow_reorient"])
def test_augmented_models_against_the_oracle(case, monkeypatch):
    """The shipped models with the new sensors added, along oracle trajectories: the A1's feet make and break contact
    (static and generic instances), the humanoid falls, the hand grasps the cube."""
    name = case.split("-")[0]
    m, start, count = load_augmented(name, monkeypatch)
    if case.endswith("generic"):
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    e = _engine(m)
    k = 0
    x0 = np.concatenate([m.key_qpos[k], np.zeros(m.nv) if name != "humanoid_track" else m.key_qvel[k]])
    if name == "quadruped":
        home = m.key_qpos[m.key_names.index("home")]
        x0 = np.concatenate([home, np.zeros(m.nv)])

        def ctrl(t, x, rng):
            return np.clip(2.0 * (home[7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:] + 0.6 * np.sin(0.2 * t + np.arange(12))
                           + 0.3 * rng.normal(size=m.nu), -1, 1)
    else:
        def ctrl(t, x, rng):
            return np.clip(0.4 * rng.normal(size=m.nu), -1, 1)
    X, U, W = _trajectory(m, x0, 96, ctrl)
    idx = np.arange(0, len(X), 8)
    mc = mocap_vector(m)
    n = _compare(m, e, X[idx], U[idx], W[idx], start, count, mc, case)
    assert n >= len(idx) // 2
    if name == "quadruped":
        assert e.last_kernel_static == (0 if case.endswith("generic") else 1)
    e.close()


def test_refusals_name_the_sensor_and_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import EngineError
    xml = SCENES["tendon_pair"](ROTATIONS[0]).replace(
        "</sensor>", '<force site="tip"/><torque site="tip"/></sensor>')
    m = compile_xml(xml)
    # a maintainer's blob with a slider-crank transmission (mjTRN_SLIDERCRANK, 2) on the motor
    mm = type(m)(m)
    tr = np.array(m.actuator_trntype, np.int32)
    tr[1] = 2
    mm["actuator_trntype"] = tr
    x = random_states(m, 1, seed=1)
    u = np.array([0.3, 0.9])
    for model, refused in ((m, (14, 15)), (mm, (2, 3))):
        e = _engine(model, n=8)
        ok = e.step_sensors(x, u, np.zeros(0), 0.0, 0, 2)
        for s in refused:
            with pytest.raises(EngineError, match="-5.*sensor %d" % s):
                e.step_sensors(x, u, np.zeros(0), 0.0, s, 1)
            again = e.step_sensors(x, u, np.zeros(0), 0.0, 0, 2)
            for f in ("sensordata", "next_states", "qacc"):
                assert np.array_equal(again[f], ok[f])
        e.close()
    with pytest.raises(EngineError, match="slide or hinge joint or a fixed tendon"):
        e = _engine(mm, n=8)
        try:
            e.step_sensors(x, u, np.zeros(0), 0.0, 2, 1)
        finally:
            e.close()


def test_plant_sensors_equal_step_sensors_with_and_without_variants():
    """Plant-bank sensor outputs of the new types are step_sensors' bitwise; a plant on a variant with a heavier hand
    reads another tip framelinacc than a plant on the base model, and equals a bank created from that variant."""
    from mujoco_mpc_b200.engine import CppPlantBank
    base = scene("ball_chain", ROTATIONS[3])
    heavy = compile_xml(SCENES["ball_chain"](ROTATIONS[3]).replace(
        '<geom name="hand" type="sphere" size="0.03" pos="0.01 0 0" mass="0.1"/>',
        '<geom name="hand" type="sphere" size="0.03" pos="0.01 0 0" mass="0.4"/>'))
    B, steps, n = 4, 20, base.nsensor
    X0 = random_states(base, B, seed=7).astype(np.float32)
    U = np.zeros((steps, B, 0), np.float32)
    tip = slice(int(base.sensor_adr[7]), int(base.sensor_adr[7]) + 3)

    def run(bank):
        for b in range(B):
            bank.reset(b, X0[b, :base.nq], X0[b, base.nq:], 0.0)
        outs = []
        for k in range(steps):
            outs.append(bank.step(U[k]))
        return outs

    bank = CppPlantBank(base, B, sensor_start=0, nsensor=n)
    plain = run(bank)
    e = _engine(base, n=8)
    q, v, w = X0[:, :base.nq].copy(), X0[:, base.nq:].copy(), np.zeros((B, base.nv), np.float32)
    for k in range(steps):
        for b in range(B):
            s = e.step_sensors(np.concatenate([q[b], v[b]])[None], np.zeros(0), np.zeros(0), k * base.opt_timestep, 0, n,
                               warmstart=w[b][None])
            assert np.array_equal(plain[k]["sensordata"][b], s["sensordata"][0]), (k, b)
            q[b], v[b], w[b] = s["next_states"][0, :base.nq], s["next_states"][0, base.nq:], s["qacc"][0]
    e.close()
    bank.set_models([base, heavy, base, heavy])
    var = run(bank)
    one = CppPlantBank(heavy, 1, sensor_start=0, nsensor=n)
    for b in (1, 3):
        one.reset(0, X0[b, :base.nq], X0[b, base.nq:], 0.0)
        for k in range(steps):
            r = one.step(U[k, b:b + 1])
            assert np.array_equal(var[k]["sensordata"][b], r["sensordata"][0]), (b, k)
    for k in range(steps):
        assert np.array_equal(var[k]["sensordata"][0], plain[k]["sensordata"][0])
    assert not np.array_equal(var[-1]["sensordata"][1][tip], plain[-1]["sensordata"][1][tip])
    bank.close(); one.close()


# --------------------------------------------------------------------------------------------- filters on the IMU body
def _filter_rms(m, f, X, Y, U, T):
    f.reset(state=X[0])
    f.set_noise(sensor=np.full(f.nsensordata, 1e-6))
    e = []
    for t in range(T):
        f.update(U[t], Y[t][:f.nsensordata], np.zeros(0))
        e.append(np.concatenate([f.state[:3] - X[t + 1, :3], f.state[m.nq:] - X[t + 1, m.nq:]]))
    return float(np.sqrt(np.mean(np.square(e[T // 4:]))))


class _Fp32Accelerometer:
    """The fp64 sensor oracle's steps with the accelerometer rows (sensordata 10:13) of the fp32 oracle's: the filter
    that sees fp32 rounding in the accelerometer alone"""

    def __init__(self, m, s, n, ts):
        self.o64, self.o32 = OracleSigmaBackend(m, s, n, ts, 64), OracleSigmaBackend(m, s, n, ts, 32)

    def step_sensors(self, states, ctrl, mocap, time, warmstart):
        nxt, y, qacc, nwarn = self.o64.step_sensors(states, ctrl, mocap, time, warmstart)
        y = y.copy()
        y[:, 10:13] = self.o32.step_sensors(states, ctrl, mocap, time, warmstart)[1][:, 10:13]
        return nxt, y, qacc, nwarn


@pytest.mark.parametrize("kind", ["unscented", "kalman"])
def test_imu_filters(kind):
    """Kalman and Unscented on the free-flying IMU body (framepos, framequat, gyro, accelerometer), driven by an fp64
    oracle plant: the C++ filter matches the Python mirror per update, a B = 4 bank matches 4 single C++ filters
    bitwise, and the RMS error is within 5 % (plus the fp32 / fp64 spread) of the fp32-oracle filter's."""
    from mujoco_mpc_b200.estimator import (CppBatchEstimator, CppKalman, CppUnscented, EngineBackend, Kalman,
                                           Unscented)
    m = imu_body(ROTATIONS[3])
    T = 60
    X, Y, U = imu_plant(m, T)
    Cpp, Mirror = (CppUnscented, Unscented) if kind == "unscented" else (CppKalman, Kalman)
    cpp = Cpp(m)
    e = _engine(m, n=64)
    mirror = Mirror(m, lambda s, n, ts: EngineBackend(e, s, n, ts))
    for f in (cpp, mirror):
        f.reset(state=X[0])
        f.set_noise(sensor=np.full(f.nsensordata, 1e-6))
    for t in range(20):
        cpp.set(mirror.state, mirror.covariance, mirror.time)
        mirror.update(U[t], Y[t], np.zeros(0))
        cpp.update(U[t], Y[t], np.zeros(0))
        dx = np.max(np.abs(cpp.state - mirror.state)) / max(1.0, np.abs(mirror.state).max())
        dP = np.max(np.abs(cpp.covariance - mirror.covariance)) / np.abs(mirror.covariance).max()
        assert dx <= 1e-9 and dP <= 1e-9, (t, dx, dP)
    # bank of 4 against 4 single C++ filters, bitwise
    B = 4
    bank = CppBatchEstimator(m, kind, B)
    singles = [Cpp(m) for _ in range(B)]
    for b in range(B):
        x0 = X[0].copy()
        x0[m.nq:] += 1e-3 * b
        bank.reset(b, state=x0); singles[b].reset(state=x0)
        bank.set_noise(b, sensor=np.full(bank.nsensordata, 1e-6)); singles[b].set_noise(sensor=np.full(bank.nsensordata, 1e-6))
    for t in range(20):
        assert (bank.update(np.tile(U[t], (B, 1)), np.tile(Y[t], (B, 1)), None) == 0).all()
        for b in range(B):
            singles[b].update(U[t], Y[t], np.zeros(0))
            x, P, _, _ = bank.get(b)
            assert np.array_equal(x, singles[b].state) and np.array_equal(P, singles[b].covariance), (t, b)
    # RMS against the filters whose sigma points / Jacobians the fp64 and fp32 oracles step
    def rms(backend, nsensor=None):
        return _filter_rms(m, Mirror(m, backend, nsensor=nsensor), X, Y, U, T)
    dev = _filter_rms(m, Cpp(m), X, Y, U, T)
    o64 = rms(lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, 64))
    o32 = rms(lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, 32))
    print("%s IMU filter RMS: device %.4g, fp32 oracle %.4g, fp64 oracle %.4g" % (kind, dev, o32, o64))
    if kind == "unscented":
        assert dev <= 1.05 * o32 + abs(o32 - o64), (dev, o32, o64)
    else:
        # In free fall the accelerometer reads the difference of two g-sized terms (the gravity offset and the
        # acceleration of the free joint), so its fp32 rounding (~1e-6) divided by the centred difference's 2e-3 puts
        # errors of ~6e-4 into Jacobian rows whose entries are at most ~0.03 (profiles/kalman_imu_jacobians.py); the
        # other rows and the transition Jacobian differ from fp64 by ~1e-5.  The filter's error then depends on which
        # rounding the accelerometer got.  Without the accelerometer fp32 and fp64 agree to 1e-5 and the device is held
        # to the Quadruped's bar; with it, to 5 % above the worse of two fp32 realisations, the fp32 oracle's and the
        # fp64 oracle's with the fp32 accelerometer alone, plus the fp32 / fp64 spread.
        d3 = _filter_rms(m, Cpp(m, nsensor=3), X, Y, U, T)
        o64_3 = rms(lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, 64), 3)
        o32_3 = rms(lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, 32), 3)
        acc32 = rms(lambda s, n, ts: _Fp32Accelerometer(m, s, n, ts))
        print("kalman without the accelerometer: device %.4g, fp32 oracle %.4g, fp64 oracle %.4g; fp64 oracle with "
              "the fp32 accelerometer %.4g" % (d3, o32_3, o64_3, acc32))
        assert d3 <= 1.05 * o32_3 + abs(o32_3 - o64_3), (d3, o32_3, o64_3)
        assert dev <= 1.05 * max(o32, acc32) + abs(o32 - o64), (dev, o32, acc32, o64)
    bank.close(); e.close()


# ------------------------------------------------------------------------------------------ closed loop on the hand
class _Recorder:
    """A filter bank that keeps each update's status and filter states"""

    def __init__(self, bank):
        self.bank, self.states, self.status = bank, [], []

    def update(self, ctrl, sensor, mocap=None):
        st = self.bank.update(ctrl, sensor, mocap)
        self.status.append(st)
        self.states.append([self.bank.state(b) for b in range(self.bank.num_filters)])
        return st

    def __getattr__(self, name):
        return getattr(self.bank, name)


def test_hand_closed_loop_through_an_unscented_bank(monkeypatch):
    """synchronous_planning_cost on the stand-in hand, the planner reading the estimate of an Unscented bank that
    measures the cube's framepos, framequat, framelinvel and frameangvel and the hand's jointpos (added to a copy of the
    model): two episodes in one batch equal two loops of one bitwise, every filter state stays finite.  The cube-pose
    error of the estimate is printed (no bar has been measured for it)."""
    from conftest import mocap_of
    from sensor_scenes import HAND_FILTER_SENSORS
    from test_gpu_plant import _episode
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    m, start, count = load_augmented("shadow_reorient", monkeypatch, extra=HAND_FILTER_SENSORS)
    B, steps, spp, seeds, N, H = 2, 30, 2, [51, 52], 16, 16
    rng = np.random.default_rng(12)
    q0 = m.key_qpos[m.key_names.index("grasp")].astype(np.float32)
    starts = [(q0, np.zeros(m.nv, np.float32)), (q0, (0.02 * rng.standard_normal(m.nv)).astype(np.float32))]
    mc = mocap_of(m)

    def bank(n):
        return _Recorder(CppBatchEstimator(m, "unscented", n, sensor_start=start, nsensor=count,
                                           timestep=m.opt_timestep))
    fb = bank(B)
    batched = _episode("sampling", m, None, starts, mc, [0.0] * B, steps, spp, seeds, estimator=fb, N=N, H=H)
    est = np.array(fb.states)                                   # [steps][B][nq + nv]
    assert np.isfinite(est).all() and (np.array(fb.status) == 0).all()
    for b in range(B):
        f1 = bank(1)
        one = _episode("sampling", m, None, starts[b:b + 1], mc, [0.0], steps, spp, seeds[b:b + 1], estimator=f1,
                       N=N, H=H)
        for f in ("costs", "states", "status"):
            assert np.array_equal(batched[f][:, b], one[f][:, 0]), (b, f)
        assert np.array_equal(np.array(f1.states)[:, 0], est[:, b]), b
        f1.close()
    assert (batched["final_status"] == 0).all()
    # the estimate after update i is of the state after step i
    a = m.jnt_qposadr[m.body_jntadr[m.body_names.index("cube")]]
    X = batched["states"].astype(float)
    dp = np.linalg.norm(est[:, :, a:a + 3] - X[:, :, a:a + 3], axis=2)
    qe, qx = est[:, :, a + 3:a + 7], X[:, :, a + 3:a + 7]
    dot = np.abs(np.sum(qe * qx, axis=2)) / (np.linalg.norm(qe, axis=2) * np.linalg.norm(qx, axis=2))
    ang = 2 * np.arccos(np.clip(dot, 0, 1))
    print("hand closed loop, Unscented bank on the cube's frame sensors: cube position error mean %.3g max %.3g m, "
          "orientation error mean %.3g max %.3g rad; average cost %s" % (dp.mean(), dp.max(), ang.mean(), ang.max(),
                                                                           batched["average_cost"]))
    fb.close()
