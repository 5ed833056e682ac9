"""GPU: the magnetometer and rangefinder of the device (mjpc_b200_step_sensors, the plant bank, the filter banks) against
the fp64 sensor oracle, the filters that they make observe a heading and a height, and the rangefinder's refusal.

Bars follow tests/test_gpu_sensors.py: teacher-forced from the same fp32-rounded state, a reading is held to
max(4 |fp32 oracle - fp64 oracle|, 2e-5 (1 + |fp64|)), where the device and the oracle found the same contacts.  A ray
that grazes a surface is ill-conditioned in fp32 (hit or miss turns on the last bit), so states whose fp64 rangefinder
readings change by more than 1e-2, or from a hit to a miss, when the pose is nudged by 1e-4 are left out; each test
asserts how many states it compared.  Plant-bank outputs come from the same k_sensors code as step_sensors, so they are
bitwise equal.  The filters are held to the bars of the fp64-oracle filters in tests/test_range_magnet_sensors_cpu.py.
"""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import mocap_vector, sensor_oracle  # noqa: E402
from test_range_magnet_sensors_cpu import (CLOSED_FORMS, NAV_BARS, NAV_T, ROOM_ASSETS, ROOM_GEOMS,  # noqa: E402
                                            ROOM_SENSORS, ROOM_SITES, down, imu_nav, nav_columns, nav_error,
                                            nav_flight, nav_start, probe_xml, room, room_states)

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.mjcf import SENS_RANGEFINDER, axisangle2quat, compile_xml, quat_mul  # noqa: E402

pytestmark = pytest.mark.gpu


def _engine(m, n=32):
    from mujoco_mpc_b200.engine import Engine
    return Engine(m, n, 8, device=0)


def _range_columns(m, start, count):
    a0 = int(m.sensor_adr[start])
    return [int(m.sensor_adr[i]) - a0 for i in range(start, start + count) if m.sensor_type[i] == SENS_RANGEFINDER]


def _well_conditioned(m, X, W, mc, start, count):
    """the states whose fp64 rangefinder readings are stable under 1e-4 nudges of every free joint's pose"""
    cols = _range_columns(m, start, count)
    o = sensor_oracle(m)
    t = np.zeros(len(X))
    U = np.zeros((len(X), m.nu))

    def ranges(Z):
        y = o.step(Z[:, :m.nq], Z[:, m.nq:], U, mc, t, start, count, warmstart=W)["sensordata"]
        return y[:, cols]
    base = ranges(X)
    ok = np.ones(len(X), bool)
    rng = np.random.default_rng(0)
    free = [int(m.jnt_qposadr[j]) for j in range(m.njnt) if m.jnt_type[j] == 0]
    for _ in range(4):
        Z = X.copy()
        for a in free:
            Z[:, a:a + 3] += 1e-4 * rng.normal(size=(len(X), 3))
            for b in range(len(X)):
                Z[b, a + 3:a + 7] = quat_mul(Z[b, a + 3:a + 7], axisangle2quat(rng.normal(size=3), 1e-4))
        Z[:, :m.nq][:, [i for i in range(m.nq) if all(not (a <= i < a + 7) for a in free)]] += \
            1e-4 * rng.normal(size=(len(X), m.nq - 7 * len(free)))
        r = ranges(Z)
        ok &= ((r < 0) == (base < 0)).all(axis=1) & (np.abs(r - base) < 1e-2).all(axis=1)
    return ok


def _compare(m, e, X, U, W, start, count, mc, what):
    """step_sensors at the well-conditioned states of X against the fp64 sensor oracle; returns the number compared"""
    o64, o32 = sensor_oracle(m, precision=64), sensor_oracle(m, precision=32)
    X32 = X.astype(np.float32).astype(float)
    W32 = None if W is None else W.astype(np.float32).astype(float)
    U32 = U.astype(np.float32).astype(float)
    t = np.zeros(len(X))
    args = (X32[:, :m.nq], X32[:, m.nq:], U32, mc, t, start, count)
    r64, r32 = o64.step(*args, warmstart=W32), o32.step(*args, warmstart=W32)
    ok = _well_conditioned(m, X32, W32, mc, start, count)
    compared, worst, hits = 0, 0.0, 0
    cols = _range_columns(m, start, count)
    for b in np.nonzero(ok)[0]:
        s = e.step_sensors(X32[b:b + 1], U32[b], mc, 0.0, start, count, warmstart=None if W32 is None else W32[b:b + 1])
        if s["ncon"][0] != r64["ncon"][b]:
            continue
        y, y64, y32 = s["sensordata"][0].astype(float), r64["sensordata"][b], r32["sensordata"][b]
        bar = np.maximum(4 * np.abs(y32 - y64), 2e-5 * (1 + np.abs(y64)))
        worst = max(worst, float(np.max(np.abs(y - y64) / bar)))
        bad = np.nonzero(np.abs(y - y64) > bar)[0]
        assert bad.size == 0, (what, b, bad, y[bad], y64[bad], y32[bad])
        compared += 1
        hits += int((y64[cols] >= 0).sum())
    print("%s: %d of %d states, %d rangefinder hits, worst |device - fp64| / bar %.3g"
          % (what, compared, len(X), hits, worst))
    return compared, hits


@pytest.mark.parametrize("generic", [False, True])
def test_room_against_the_oracle(generic, monkeypatch):
    if generic:
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = room()
    e = _engine(m)
    X = room_states(m, 32, seed=11)
    n, hits = _compare(m, e, X, np.zeros((len(X), 0)), None, 0, m.nsensor - 1, np.zeros(0), "room")
    assert n >= 24 and hits >= 48, (n, hits)
    e.close()


def test_closed_form_scenes_against_the_oracle():
    for case in sorted(CLOSED_FORMS):
        xml, pos, dist = CLOSED_FORMS[case]
        m = compile_xml(probe_xml(xml, pos=pos, quat=down()))
        e = _engine(m, n=8)
        x = np.concatenate([m.qpos0, np.zeros(m.nv)])[None]
        y = e.step_sensors(x, np.zeros(0), np.zeros(0), 0.0, 0, m.nsensor - 1)["sensordata"][0]
        assert abs(y[0] - dist) <= 2e-5 * (1 + dist), (case, y[0], dist)
        e.close()


# ------------------------------------------------------------------------------------------ the shipped models
QUADRUPED_EXTRA = """
    <rangefinder site="torso"/><magnetometer site="torso"/>
    <rangefinder site="FR"/><rangefinder site="FL"/><rangefinder site="RR"/><rangefinder site="RL"/>
"""
HUMANOID_EXTRA = """
    <rangefinder site="tracking[pelvis]"/><magnetometer site="tracking[head]"/>
    <rangefinder site="foot_right"/><rangefinder site="foot_left"/><magnetometer site="foot_left"/>
"""


def _load(name, monkeypatch):
    """models.load(name) with the sensors above appended to a copy of its MJCF, and the trunk's (pelvis') site turned to
    look down: a new orientation of an existing site, so the layout, and with it the static instance, stays the
    shipped model's"""
    fn, extra = {"quadruped": ("quadruped_flat_xml", QUADRUPED_EXTRA),
                 "humanoid_track": ("humanoid_track_xml", HUMANOID_EXTRA)}[name]
    orig = getattr(models, fn)

    def patched(*a, **k):
        x = orig(*a, **k)
        x = x.replace('<site name="torso"/>', '<site name="torso" quat="0 1 0 0"/>', 1)
        x = re.sub(r'(<site name="tracking\[pelvis\]")', r'\1 quat="0 1 0 0"', x, count=1)
        i = x.rindex("</sensor>")
        return x[:i] + extra + x[i:]
    base = models.load(name)
    monkeypatch.setattr(models, fn, patched)
    m = models.load(name)
    monkeypatch.setattr(models, fn, orig)
    return m, base.nsensor, m.nsensor - base.nsensor


def _trajectory(m, x0, T, ctrl, seed=0):
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


@pytest.mark.parametrize("case", ["quadruped", "quadruped-generic", "humanoid_track", "humanoid_track-generic"])
def test_shipped_models_against_the_oracle(case, monkeypatch):
    name = case.split("-")[0]
    m, start, count = _load(name, monkeypatch)
    assert m.sensor_type[start] in (28, 29)
    if case.endswith("generic"):
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    e = _engine(m)
    if name == "quadruped":
        home = m.key_qpos[m.key_names.index("home")]
        x0 = np.concatenate([home, np.zeros(m.nv)])

        def ctrl(t, x, rng):
            return np.clip(2.0 * (home[7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:] + 0.6 * np.sin(0.2 * t + np.arange(12))
                           + 0.3 * rng.normal(size=m.nu), -1, 1)
    else:
        x0 = np.concatenate([m.key_qpos[0], m.key_qvel[0]])

        def ctrl(t, x, rng):
            return np.clip(0.4 * rng.normal(size=m.nu), -1, 1)
    X, U, W = _trajectory(m, x0, 96, ctrl)
    idx = np.arange(0, len(X), 6)
    n, hits = _compare(m, e, X[idx], U[idx], W[idx], start, count, mocap_vector(m), case)
    assert n >= len(idx) // 2 and hits >= n, (n, hits)
    expected = 0 if case.endswith("generic") else 1
    assert e.last_kernel_static == expected
    e.close()


# ------------------------------------------------------------------------------------------------- plant bank
def test_plant_sensors_equal_step_sensors_with_variants_and_a_wrench():
    """Plant-bank readings are step_sensors' at each plant's pre-step state, bitwise (the magnetometer and rangefinder
    read positions only); a plant on a variant with a larger ball reads that ball's new surface; a held wrench moves the
    readings, which still equal step_sensors'."""
    from mujoco_mpc_b200.engine import CppPlantBank
    base = room()
    big = compile_xml(probe_xml(ROOM_GEOMS.replace('name="ball" type="sphere" pos="0.8 0.6 0.4" size="0.25"',
                                                   'name="ball" type="sphere" pos="0.8 0.6 0.4" size="0.35"'),
                                pos=(0.1, 0.05, 1.1), quat=down(0.3), assets=ROOM_ASSETS, extra_sites=ROOM_SITES,
                                extra_sensors=ROOM_SENSORS))
    B, steps, n = 4, 12, base.nsensor - 1
    X0 = room_states(base, B, seed=4).astype(np.float32)
    X0[:, 7:] *= 0.1
    X0[1, :3] = X0[3, :3] = [0.8, 0.6, 1.2]            # plants 1 and 3 hover over the ball, looking straight down
    X0[1, 3:7] = X0[3, 3:7] = down()
    U = np.zeros((steps, B, 0), np.float32)
    engines = {id(base): _engine(base, n=8), id(big): _engine(big, n=8)}

    def run(bank, models, wrench=None):
        """the bank's steps from X0, each plant's readings checked against step_sensors on its model"""
        for b in range(B):
            bank.reset(b, X0[b, :base.nq], X0[b, base.nq:], 0.0)
            bank.set_xfrc(b, wrench)
        outs = [bank.step(U[k]) for k in range(steps)]
        for k in range(steps):
            pre = X0 if k == 0 else outs[k - 1]["state"]
            for b in range(B):
                s = engines[id(models[b])].step_sensors(pre[b:b + 1], np.zeros(0), np.zeros(0), 0.0, 0, n)
                assert np.array_equal(outs[k]["sensordata"][b], s["sensordata"][0]), (k, b)
        return outs

    bank = CppPlantBank(base, B, sensor_start=0, nsensor=n)
    plain = run(bank, [base] * B)
    bank.set_models([base, big, base, big])
    var = run(bank, [base, big, base, big])
    for k in range(steps):
        assert np.array_equal(var[k]["sensordata"][0], plain[k]["sensordata"][0])
        # the ball's top is at 0.4 + r below an eye at the plant's height
        for b in (1, 3):
            pre = (X0 if k == 0 else plain[k - 1]["state"])[b][2], (X0 if k == 0 else var[k - 1]["state"])[b][2]
            assert abs(plain[k]["sensordata"][b][0] - (pre[0] - 0.65)) < 1e-4
            assert abs(var[k]["sensordata"][b][0] - (pre[1] - 0.75)) < 1e-4
    bank.set_models(None)
    wrench = np.zeros((base.nbody, 6))
    wrench[base.body_names.index("probe")] = [0, 0, -80.0, 0.3, -0.2, 0.1]
    pushed = run(bank, [base] * B, wrench)
    assert not np.array_equal(pushed[-1]["sensordata"], plain[-1]["sensordata"])
    bank.close()
    for e in engines.values():
        e.close()


# ------------------------------------------------------------------------------------------------ the filters
@pytest.mark.parametrize("kind", ["kalman", "unscented"])
@pytest.mark.parametrize("what", ["heading", "height"])
def test_filter_banks_observe_heading_and_height(kind, what):
    """A bank of two filters on the IMU body, started with a 0.5 rad yaw error or a 0.3 m height error: with the
    magnetometer (the rangefinder) among its sensors the error falls below the fp64-oracle filters' bar; a bank without
    it keeps the error."""
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    m = imu_nav()
    T = NAV_T
    X, Y, U = nav_flight(m, T)
    for measured in (True, False):
        s, n, a, e = nav_columns(m, what, measured)
        bank = CppBatchEstimator(m, kind, 2, sensor_start=s, nsensor=n)
        x0, P0 = nav_start(m, X[0], what)
        for b in range(2):
            bank.set(b, x0, P0, 0.0)
            bank.set_noise(b, process=np.full(2 * m.nv, 1e-8), sensor=np.full(e - a, 1e-6))
        for t in range(T):
            assert (bank.update(np.tile(U[t], (2, 1)), np.tile(Y[t][a:e], (2, 1)), None) == 0).all()
        errs = [nav_error(m, bank.state(b), X[T], what) for b in range(2)]
        print("%s bank, %s %s: final errors %s" % (kind, what, "measured" if measured else "not measured", errs))
        for err in errs:
            assert err < NAV_BARS[what][0] if measured else err > NAV_BARS[what][1], (measured, err)
        assert np.array_equal(bank.state(0), bank.state(1))
        bank.close()


# ---------------------------------------------------------------------------------------------------- refusals
def test_rangefinder_refused_over_a_hfield():
    from mujoco_mpc_b200.engine import EngineError
    m = compile_xml(probe_xml('<geom type="hfield" size="1 1 0.1"/><geom type="plane" size="0 0 1"/>', quat=down()))
    e = _engine(m, n=8)
    x = np.concatenate([m.qpos0, np.zeros(m.nv)])[None]
    ok = e.step_sensors(x, np.zeros(0), np.zeros(0), 0.0, 1, 1)
    with pytest.raises(EngineError, match="-5.*sensor 0.*geom 0"):
        e.step_sensors(x, np.zeros(0), np.zeros(0), 0.0, 0, 1)
    again = e.step_sensors(x, np.zeros(0), np.zeros(0), 0.0, 1, 1)
    for f in ("sensordata", "next_states", "qacc"):
        assert np.array_equal(again[f], ok[f])
    e.close()
