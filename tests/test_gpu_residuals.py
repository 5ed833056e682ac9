"""GPU: the device task residuals (csrc/dev_task.cuh k_residual, k_residual_quadruped, ground_height) against the fp64
oracle on the purpose-built cases of tests/residual_scenes.py.

Device and oracle get the same inputs, rounded to fp32 and upcast, so that the comparison measures kernel arithmetic.
Per case every residual row, the step's cost and the warning flag are compared, through three kernel instances:
Engine.step_batch on the static step instance, step_batch on the generic instance (MJPC_B200_NO_STATIC=1), and the
static rollout kernel (one batched launch, a different task snapshot per problem), whose recorded residual rows are
evaluated by the oracle at the device's own recorded states, controls and times.

Bars: the oracle's fp32 instantiation is the yardstick.  A row's bar is 4 x |fp32 oracle - fp64 oracle| plus a floor of
2e-6 x the scene's length scale (1 m, or the trunk's distance from the origin); the cost's is 4 x the fp32 oracle's
error plus 5e-6, relative to the cost.  A rollout step's residual reads the fp32 running time, which drifts up to
3e-7 s from the recorded time (DESIGN.md): its bar adds 4e-7 s x the row's clock rate, measured on the fp64 oracle.  A
case flagged discontinuous passes a row when the device equals fp64 at the case or at one of its sides.  A case moved
to clock time t0 (1e2, 1e4, 1e6 s) must meet its t0 = 0 bar.  test_zz_report prints the largest error / bar per row group.
"""
import numpy as np
import pytest

import residual_scenes as RS

pytestmark = pytest.mark.gpu

REPORT = {}     # (instance, row group) -> largest error / bar


@pytest.fixture(scope="module")
def rig(oracle_lib):
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    build.build()
    cache = {}

    def get(name):
        if name not in cache:
            m = RS.model(name)
            cache[name] = (oracle_lib.Oracle(to_blob(m), m, 64), oracle_lib.Oracle(to_blob(m), m, 32), Engine(m, 64, 16))
        return cache[name]
    yield get
    for _, _, e in cache.values():
        e.close()


def _groups(c):
    if c.model_name.startswith("quadruped"):
        return RS.QUAD_GROUPS
    return {c.model_name: (0, c.m.task_num_residual)}


def _oracle_step(o, c):
    o.set_task(parameters=c.parameters, task_state=c.task_state)
    r = o.step_batch(c.qpos[None], c.qvel[None], c.ctrl[None], c.mocap, np.array([c.time]))
    return r["residual"][0, : c.m.task_num_residual], float(r["cost"][0]), int(r["warning"][0])


def _device_step(e, c):
    e.set_task(parameters=c.parameters, task_state=c.task_state)
    r = e.step_batch(c.qpos[None], c.qvel[None], c.ctrl[None], c.mocap, np.array([c.time]), time0=c.t0)
    return r["residual"][0, : c.m.task_num_residual].astype(float), float(r["cost"][0]), int(r["warning"][0])


def _floor(c):
    L = max(1.0, float(np.abs(c.qpos[:3]).max())) if c.model_name.startswith("quadruped") else 1.0
    return 2e-6 * L


def _bars(rig, c):
    """(row bar, relative cost bar) of case c (at clock time 0) from the fp32 oracle's error.  At a discontinuity the
    fp32 oracle may fall on the other side of the threshold at the case itself, which would make its error the jump:
    each row takes the smallest fp32 error over the case and its sides."""
    o64, o32, _ = rig(c.model_name)
    rb, cb = np.inf, np.inf
    for v in [c] + c.side_cases():
        r64, c64, _ = _oracle_step(o64, v)
        r32, c32, _ = _oracle_step(o32, v)
        rb, cb = np.minimum(rb, 4 * np.abs(r32 - r64)), min(cb, (4 * abs(c32 - c64) + 1e-9) / abs(c64))
    return rb + _floor(c), cb + 5e-6


def _check(rig, c, bars, instance, static):
    """Compare the device's step_batch with fp64 on case c (rounded inputs) against bars; record error / bar."""
    o64, _, e = rig(c.model_name)
    dev, dcost, dwarn = _device_step(e, c)
    if static is not None:
        assert e.last_kernel_static == static, (c.name, instance)
    r64, c64, w64 = _oracle_step(o64, c)
    rb, cb = bars[0], bars[1] * abs(c64)
    err, cerr = np.abs(dev - r64), abs(dcost - c64)
    for s in c.side_cases():
        sr, sc, _ = _oracle_step(o64, s)
        err, cerr = np.minimum(err, np.abs(dev - sr)), min(cerr, abs(dcost - sc))
    assert dwarn == w64 == int("warning" in c.flags), (c.name, instance, dwarn, w64)
    ratio = err / rb
    for g, (a, b) in _groups(c).items():
        key = (instance, g)
        REPORT[key] = max(REPORT.get(key, 0.0), float(ratio[a:b].max()))
    REPORT[(instance, "cost")] = max(REPORT.get((instance, "cost"), 0.0), cerr / cb)
    bad = np.nonzero(ratio > 1)[0]
    assert not len(bad), (c.name, instance, [(int(i), float(dev[i]), float(r64[i]), float(rb[i])) for i in bad[:6]])
    assert cerr <= cb, (c.name, instance, dcost, c64, cb)


ALL_CASES = RS.quadruped_cases() + RS.other_cases()


@pytest.mark.parametrize("generic", [False, True], ids=["static", "generic"])
def test_step_residuals_against_fp64(rig, generic, monkeypatch):
    if generic:
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    for c in ALL_CASES:
        c = c.rounded()
        static = 0 if generic else (1 if c.model_name == "quadruped" else None)
        _check(rig, c, _bars(rig, c), "step_batch " + ("generic" if generic else "static"), static)


@pytest.mark.parametrize("t0", RS.CLOCK_SHIFTS[1:])
def test_clock_shift_meets_the_t0_bar(rig, t0):
    """The same Quadruped case at absolute clock time t0 meets its t0 = 0 bar: the gait phase, which grows at
    2 pi cadence per second, must reach the device as a phase relative to the launch, not as an absolute one."""
    for c in RS.quadruped_cases():
        bars = _bars(rig, c.rounded())
        _check(rig, RS.shifted(c, t0).rounded(), bars, f"step_batch static t0={t0:g}",
               1 if c.model_name == "quadruped" else None)


def test_rollout_residual_rows_against_fp64(rig):
    """One batched launch of the static rollout kernel, each problem with its own task snapshot (every mode); the
    recorded residual rows, step costs and failure flags against the oracle's steps at the recorded states, controls
    and times."""
    names = ("quadruped", "biped_type0", "biped_type1", "walk_straight", "walk_turning", "scramble", "flip_dir0",
             "flip_dir1", "flip_crouch_before", "flip_land_after", "gait1_t1", "gait3_t2", "gait4_t0", "ramp", "hill_top",
             "box_moved_rotated")
    cases = [c.rounded() for c in RS.quadruped_cases() if c.name in names]
    assert len(cases) == len(names)
    o64, o32, e = rig("quadruped")
    m = RS.model("quadruped")
    B, N, H, P = len(cases), 2, 16, 3
    rng = np.random.default_rng(3)
    states = np.array([np.concatenate([c.qpos, c.qvel]) for c in cases])
    times = np.array([c.time for c in cases])
    mocaps = np.array([c.mocap for c in cases])
    knots = np.clip(0.3 * rng.standard_normal((B, N, P, m.nu)), -1, 1).astype(np.float32)
    kt = times[:, None] + np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    _, fail, _ = e.rollout_spline_batched(states, times, mocaps, knots, kt, 2, H,
                                          parameters=np.array([c.parameters for c in cases]),
                                          task_states=np.array([c.task_state for c in cases]))
    assert e.last_kernel_static
    tr = e.fetch_all()
    nq, nr = m.nq, m.task_num_residual
    for b, c in enumerate(cases):
        sl = slice(b * N, (b + 1) * N)
        S = tr["states"][sl, : H - 1].reshape(-1, nq + m.nv).astype(float)
        U = tr["actions"][sl, : H - 1].reshape(-1, m.nu).astype(float)
        T = tr["times"][sl, : H - 1].reshape(-1)
        dev = tr["residual"][sl, : H - 1].reshape(-1, nr).astype(float)
        dcost = tr["costs"][sl, : H - 1].reshape(-1).astype(float)
        out = {}
        for name, o in (("64", o64), ("32", o32)):
            o.set_task(parameters=c.parameters, task_state=c.task_state)
            for k, dt in (("", 0.0), ("+", 1e-5), ("-", -1e-5)):
                if name == "32" and k:
                    continue
                out[name + k] = o.step_batch(S[:, :nq], S[:, nq:], U, c.mocap, T + dt)
        res = {k: v["residual"][:, :nr] for k, v in out.items()}
        rate = np.abs(res["64+"] - res["64-"]) / 2e-5
        bar = 4 * np.abs(res["32"] - res["64"]) + _floor(c) + 4e-7 * rate
        ratio = np.abs(dev - res["64"]) / bar
        c64 = out["64"]["cost"]
        crate = np.abs(out["64+"]["cost"] - out["64-"]["cost"]) / 2e-5
        cbar = 4 * np.abs(out["32"]["cost"] - c64) + 5e-6 * np.abs(c64) + 4e-7 * crate + 1e-9
        cratio = np.abs(dcost - c64) / cbar
        for g, (a, bb) in RS.QUAD_GROUPS.items():
            key = ("rollout static", g)
            REPORT[key] = max(REPORT.get(key, 0.0), float(ratio[:, a:bb].max()))
        REPORT[("rollout static", "cost")] = max(REPORT.get(("rollout static", "cost"), 0.0), float(cratio.max()))
        assert ratio.max() <= 1, (c.name, np.unravel_index(ratio.argmax(), ratio.shape), ratio.max())
        assert cratio.max() <= 1, (c.name, int(cratio.argmax()), cratio.max())
        # a candidate fails when one of its steps warns; the oracle's steps at the recorded states warn the same
        warned = out["64"]["warning"].reshape(N, H - 1).any(1)
        np.testing.assert_array_equal(fail[b].astype(bool), warned, err_msg=c.name)
        assert not warned.any(), c.name


def test_plant_steps_at_a_late_clock(rig):
    """A closed-loop plant stepping at t ~ 1e5 s, 3.3 s into its episode, has the cost the fp64 oracle gives, to the
    accuracy of the same plant at t ~ 0."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.engine import CppPlantBank
    o64, _, _ = rig("quadruped")
    base = next(c for c in RS.quadruped_cases() if c.name == "gait1_t1").rounded()
    rel = {}
    for t0 in (0.0, 1e5):
        c = RS.shifted(base, t0)
        ts = c.task_state.copy()
        for i in (T.QS_MODE_START_TIME, T.QS_PHASE_START_TIME, T.QS_PHASE_START):
            ts[i] -= 3.3                                        # the episode started 3.3 s earlier
        c = c.replace(task_state=ts)
        bank = CppPlantBank(c.m, 1)
        try:
            bank.reset(0, c.qpos, c.qvel, c.time, c.mocap)
            bank.set_task(0, parameters=c.parameters, task_state=c.task_state)
            o = bank.step(c.ctrl[None])
            assert o["status"][0] == 0 and bank.last_kernel_static() == 1
        finally:
            bank.close()
        _, c64, _ = _oracle_step(o64, c)
        rel[t0] = abs(float(o["cost"][0]) - c64) / abs(c64)
    print("plant cost relative error vs fp64: t ~ 0: %.2e, t ~ 1e5 s: %.2e" % (rel[0.0], rel[1e5]))
    assert rel[1e5] <= max(4 * rel[0.0], 5e-6), rel


def test_zz_report():
    for (inst, g), v in sorted(REPORT.items()):
        print("%-32s %-9s max error / bar %.3f" % (inst, g, v))
