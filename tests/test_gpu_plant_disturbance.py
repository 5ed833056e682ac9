"""GPU: the plants' disturbances (mjpc_b200_plant_set_disturbance / _set_xfrc / _get_disturbance / _last_ctrl,
CppPlantBank.set_disturbance / set_xfrc / disturbance).

A plant without disturbances must step bitwise as before.  Control noise must be exactly extra control, its noise the
numpy restatement (tests/plant_noise.py).  A held wrench and the force noise must match the fp64 oracle fed the same
xfrc_applied, within the teacher-forced bars of tests/test_gpu_teacher_forced.py (3x the fp32 oracle's error)."""
import ctypes as C

import numpy as np
import pytest

import plant_noise as PN
from conftest import get_model, mocap_of
from test_gpu_model_variants import _variants
from test_gpu_plant import QUAD_SENSORS, _bank, _ctrl, _eq, _mocap, _run, _start

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, UNSUPPORTED = -1, -5
TRUNK = 3                                               # the Quadruped's trunk body
WRENCH = np.array([15.0, -10.0, 5.0, 0.5, -0.3, 0.2])   # force (N), torque (N m), world frame


def _trunk_xfrc(m, w=WRENCH):
    x = np.zeros((m.nbody, 6))
    x[TRUNK] = w
    return x


# ------------------------------------------------------------------------------------------ 1. bitwise unchanged
@pytest.mark.parametrize("case", ["quadruped", "quadruped-generic", "humanoid_track"])
def test_undisturbed_plants_step_bitwise_as_before(case, monkeypatch):
    name = case.split("-")[0]
    if case.endswith("generic"):
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model(name)
    B, steps = 4, 30
    sensors = QUAD_SENSORS if name == "quadruped" else (None, 0)
    mc, starts, U = _mocap(m), _start(m, B), _ctrl(m, B, steps, seed=7)
    plain, zeros, cleared = _bank(m, B, sensors), _bank(m, B, sensors), _bank(m, B, sensors)
    for b in range(B):
        zeros.set_disturbance(b, 0.0, 1.0, 0.0, 1.0, seed=100 + b)
        zeros.set_xfrc(b, np.zeros((m.nbody, 6)))
        cleared.set_xfrc(b, np.ones((m.nbody, 6)))
        cleared.set_xfrc(b, None)
    ref = _run(plain, starts, mc, U)
    for bank, what in ((zeros, "all-zero disturbance"), (cleared, "cleared wrench")):
        got = _run(bank, starts, mc, U)
        assert bank.last_kernel_static() == (0 if case.endswith("generic") else 1)
        for k in range(steps):
            for f in ("state", "cost", "time", "status", "sensordata", "ctrl"):
                _eq(got[k][f], ref[k][f], f"{case} {what} step {k} {f}")
            _eq(got[k]["ctrl"], U[k], f"{case} {what} step {k}: the applied ctrl is the commanded ctrl")
        for b in range(B):
            d = bank.disturbance(b)
            assert not d["ctrl_noise"].any() and not d["xfrc_noise"].any()
            g, r = bank.get(b), plain.get(b)
            for f in g:
                _eq(g[f], r[f], f"{case} {what} plant {b} {f}")
        bank.close()
    plain.close()


# ------------------------------------------------------------------------------------------ 2. control noise
def test_control_noise_is_exactly_extra_control():
    m = get_model("quadruped")
    B, steps, std, rate = 2, 200, 0.3, 0.05
    seeds = [17, 18]
    mc, starts = mocap_of(m), _start(m, B)
    t = np.arange(steps)[:, None, None] * m.opt_timestep
    U = (0.3 * np.sin(2 * np.pi * (t + np.arange(m.nu) / m.nu))).repeat(B, 1).astype(np.float32)
    U[:, :, 0] = 1.2            # past ctrlrange [-1, 1]: actuation clamps the noisy ctrl
    U[:, :, 5] = -0.95          # at the edge: the noise crosses the limit both ways
    noisy, clean = _bank(m, B), _bank(m, B)
    for b in range(B):
        noisy.set_disturbance(b, ctrl_std=std, ctrl_rate=rate, seed=seeds[b])
    for b, (q, v) in enumerate(starts):
        noisy.reset(b, q, v, 0.0, mc)
        clean.reset(b, q, v, 0.0, mc)
    applied = np.zeros((steps, B, m.nu), np.float32)
    for k in range(steps):
        o = noisy.step(U[k])
        r = clean.step(o["ctrl"])
        assert (o["status"] == 0).all()
        for f in ("state", "cost", "time"):
            _eq(o[f], r[f], f"step {k} {f}: a noisy plant is a clean plant stepped from the applied ctrl")
        applied[k] = o["ctrl"]
    for b in range(B):
        ref = PN.ou_states(seeds[b], steps, m.nu, std, rate, m.opt_timestep, PN.TAG_CTRL)
        err = np.abs((applied[:, b].astype(float) - U[:, b]) - ref)
        print("plant %d: |applied - u - OU| max %.2e, noise rms %.3f" % (b, err.max(), np.sqrt((ref ** 2).mean())))
        assert err.max() < 2e-6 * 8      # rounding of u + n (|u + n| < 2) and the fp32 stream
        np.testing.assert_allclose(noisy.disturbance(b)["ctrl_noise"], ref[-1], atol=2e-6)
    assert (applied[:, :, 0] > 1).any() and (applied[:, :, 5] < -1).any()     # the clamp was exercised
    assert (applied[:, :, 5] > -1).any()
    noisy.close(); clean.close()


# ------------------------------------------------------------------------------------------ 3. held wrench
def test_particle_force_equals_control():
    """On the particle (two slide joints on one body, unit-gear motors on them) a force on the body is a control."""
    m = get_model("particle")
    body = int(m.jnt_bodyid[0])
    steps = 40
    pushed, driven = _bank(m, 1), _bank(m, 1)
    q0, v0 = np.array([0.05, -0.02], np.float32), np.array([0.1, 0.0], np.float32)
    f = np.array([0.3, -0.2])
    x = np.zeros((m.nbody, 6))
    x[body, :2] = f
    x[body, 3:] = [0.7, -0.4, 0.1]     # a torque has no dof to act on
    pushed.set_xfrc(0, x)
    for bank in (pushed, driven):
        bank.reset(0, q0, v0, 0.0, mocap_of(m))
    for k in range(steps):
        a = pushed.step(np.zeros((1, m.nu), np.float32))
        r = driven.step(f[None].astype(np.float32))
        np.testing.assert_allclose(a["state"], r["state"], atol=2e-6, err_msg=f"step {k}")
    assert abs(a["state"][0, 0] - q0[0]) > 1e-3
    pushed.close(); driven.close()


def _oracles(m):
    import sensor_oracle as so
    from mujoco_mpc_b200.blob import to_blob
    so.build()
    return so.SensorOracle(to_blob(m), m, 64), so.SensorOracle(to_blob(m), m, 32)


def _teacher_forced(bank, m, mc, U, xfrc_of):
    """Step the bank through U; before every step give the fp64 and fp32 oracles each plant's state, warm start, ctrl
    and xfrc_of(k, b).  Returns the device's and the fp32 oracle's per-step qvel errors against fp64, and the qpos
    error."""
    o64, o32 = _oracles(m)
    B, nq = bank.num_plants, m.nq
    ev, ev32, eq = [], [], []
    for k in range(len(U)):
        pre = [bank.get(b) for b in range(B)]
        S = np.array([p["state"] for p in pre], float); W = np.array([p["warmstart"] for p in pre], float)
        T = np.array([p["time"] for p in pre])
        X = np.array([xfrc_of(k, b) for b in range(B)])
        o = bank.step(U[k])
        assert (o["status"] == 0).all(), k
        args = (S[:, :nq], S[:, nq:], o["ctrl"].astype(float), mc, T, 0, 0)
        r64 = o64.step(*args, warmstart=W, xfrc=X)
        r32 = o32.step(*args, warmstart=W, xfrc=X)
        ev.append(np.abs(o["state"][:, nq:] - r64["next_qvel"]).max(1))
        ev32.append(np.abs(r32["next_qvel"] - r64["next_qvel"]).max(1))
        eq.append(np.abs(o["state"][:, :nq] - r64["next_qpos"]).max(1))
    return np.concatenate(ev), np.concatenate(ev32), np.concatenate(eq)


def _assert_teacher_forced_bars(ev, ev32, eq, what):
    p = lambda e: (float(np.median(e)), float(np.percentile(e, 99)), float(e.max()))   # noqa: E731
    (p50, p99, mx), (q50, q99, qmx) = p(ev), p(ev32)
    print("%s: device qvel err median %.2e p99 %.2e max %.2e | fp32 oracle %.2e %.2e %.2e" % (
        what, p50, p99, mx, q50, q99, qmx))
    assert p50 <= 2e-5 and p99 <= 6e-4 and mx <= 5e-3
    assert p50 <= 3 * max(q50, 1e-6) and p99 <= 3 * max(q99, 1e-5) and mx <= 3 * max(qmx, 1e-3)
    assert eq.max() <= 1e-5 + 0.01 * mx * 1.01 + 2e-6


def test_trunk_wrench_against_fp64():
    m = get_model("quadruped")
    B, steps = 8, 40
    mc, starts, U = mocap_of(m), _start(m, B, seed=4), _ctrl(m, B, steps, seed=8)
    X = [_trunk_xfrc(m, WRENCH * (1 + 0.25 * b)) for b in range(B)]
    bank = _bank(m, B)
    for b, (q, v) in enumerate(starts):
        bank.reset(b, q, v, 0.0, mc)
        bank.set_xfrc(b, X[b])
    ev, ev32, eq = _teacher_forced(bank, m, mc, U, lambda k, b: X[b])
    _assert_teacher_forced_bars(ev, ev32, eq, "trunk wrench")
    # the wrench is visible: the same controls without it end elsewhere
    free = _bank(m, B)
    ref = _run(free, starts, mc, U)
    assert np.abs(bank.get(0)["state"] - ref[-1]["state"][0]).max() > 1e-2
    bank.close(); free.close()


# ------------------------------------------------------------------------------------------ 4. force noise
def test_force_noise_states_and_steps_against_fp64():
    m = get_model("quadruped")
    B, steps, std, rate = 4, 100, 2.0, 0.1
    seeds = [5, 6, 7, 8]
    mc, starts, U = mocap_of(m), _start(m, B, seed=5), _ctrl(m, B, steps, seed=9)
    held = _trunk_xfrc(m, WRENCH * 0.5)
    bank = _bank(m, B)
    for b, (q, v) in enumerate(starts):
        bank.reset(b, q, v, 0.0, mc)
        bank.set_disturbance(b, xfrc_std=std, xfrc_rate=rate, seed=seeds[b])
    bank.set_xfrc(1, held)          # held + noise on plant 1
    nx = 6 * m.nbody
    ref = [PN.ou_states(seeds[b], steps, nx, std, rate, m.opt_timestep, PN.TAG_XFRC) for b in range(B)]

    def xfrc_of(k, b):
        return ref[b][k].reshape(m.nbody, 6) + (held if b == 1 else 0)
    ev, ev32, eq = _teacher_forced(bank, m, mc, U, xfrc_of)
    _assert_teacher_forced_bars(ev, ev32, eq, "force noise")
    for b in range(B):
        d = bank.disturbance(b)
        np.testing.assert_allclose(d["xfrc_noise"].reshape(-1), ref[b][-1], atol=1e-5 * std)
        assert bank.get(b)["steps"] == steps and not d["ctrl_noise"].any()
    bank.close()


# ------------------------------------------------------------------------------------------ 5. independence, variants
def _disturb(bank, b, cfg):
    cs, cr, xs, xr, seed, w = cfg
    bank.set_disturbance(b, cs, cr, xs, xr, seed)
    bank.set_xfrc(b, w)


def test_a_disturbed_plant_is_independent_of_its_position_and_the_others():
    m = get_model("quadruped")
    steps, B = 30, 4
    mc = mocap_of(m)
    me = _start(m, 1, seed=9)[0]
    mine = _ctrl(m, 1, steps, seed=2)
    my_cfg = (0.2, 0.05, 1.5, 0.1, 99, _trunk_xfrc(m))
    alone = _bank(m, 1)
    _disturb(alone, 0, my_cfg)
    ref = _run(alone, [me], mc, mine)
    alone.close()
    bank = _bank(m, B)
    for j in range(B):
        starts, U = _start(m, B, seed=10 + j), _ctrl(m, B, steps, seed=20 + j)
        starts[j] = me
        U[:, j] = mine[:, 0]
        for b in range(B):
            _disturb(bank, b, my_cfg if b == j else (0.1 * b, 0.02 * (b + 1), 0.5 * b, 0.05, 99 if b % 2 else b,
                                                     _trunk_xfrc(m, -WRENCH * b) if b % 2 else None))
        got = _run(bank, starts, mc, U)
        for k in range(steps):
            for f in ("state", "cost", "ctrl"):
                _eq(got[k][f][j], ref[k][f][0], f"position {j} step {k} {f}")
    bank.close()


def test_variant_plants_are_disturbed_on_their_variant():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, steps = 4, 30
    mc, starts, U = mocap_of(base), _start(base, B), _ctrl(base, B, steps, seed=1)
    cfg = [(0.1 + 0.05 * b, 0.05, 1.0 + b, 0.1, 40 + b, _trunk_xfrc(base, WRENCH * (b - 1.5))) for b in range(B)]
    bank = _bank(base, B, QUAD_SENSORS)
    bank.set_models(V)
    for b in range(B):
        _disturb(bank, b, cfg[b])
    got = _run(bank, starts, mc, U)
    for b in range(B):
        one = _bank(V[b], 1, QUAD_SENSORS)
        _disturb(one, 0, cfg[b])
        ref = _run(one, starts[b:b + 1], mc, U[:, b:b + 1])
        for k in range(steps):
            for f in ("state", "cost", "time", "sensordata", "ctrl"):
                _eq(got[k][f][b], ref[k][f][0], f"variant {b} step {k} {f}")
        one.close()
    bank.close()


# ------------------------------------------------------------------------------------------ 6. reset, divergence, refusals
def test_reset_replays_and_a_diverged_step_keeps_the_noise():
    from mujoco_mpc_b200.engine import PLANT_DIVERGED
    m = get_model("quadruped")
    B, steps = 2, 20
    mc, starts, U = mocap_of(m), _start(m, B), _ctrl(m, B, steps, seed=3)
    bank = _bank(m, B)
    for b in range(B):
        _disturb(bank, b, (0.2, 0.05, 1.0, 0.1, 7 + b, _trunk_xfrc(m)))
    first = _run(bank, starts, mc, U)
    second = _run(bank, starts, mc, U)       # reset keeps the settings and the wrench and replays the noise
    for k in range(steps):
        for f in ("state", "cost", "ctrl"):
            _eq(second[k][f], first[k][f], f"replay step {k} {f}")
    # a step that diverges (a 1e30 N push) commits nothing, the noise states included
    before = [bank.disturbance(b) for b in range(B)]
    bank.set_xfrc(0, _trunk_xfrc(m, np.array([1e30, 0, 0, 0, 0, 0])))
    o = bank.step(U[0])
    assert o["status"].tolist() == [PLANT_DIVERGED, 0]
    after = bank.disturbance(0)
    for f in ("ctrl_noise", "xfrc_noise"):
        _eq(after[f], before[0][f], f"diverged plant's {f}")
    assert bank.get(0)["steps"] == steps
    assert not np.array_equal(bank.disturbance(1)["xfrc_noise"], before[1]["xfrc_noise"])
    bank.close()


def test_refusals_leave_the_bank_unchanged():
    from mujoco_mpc_b200.engine import EngineError, _model_blobs
    m = get_model("quadruped")
    B, steps = 3, 6
    mc, starts, U = mocap_of(m), _start(m, B), _ctrl(m, B, 2 * steps, seed=6)
    bank, control = _bank(m, B), _bank(m, B)
    for bk in (bank, control):
        for b in range(B):
            _disturb(bk, b, (0.2, 0.05, 1.0, 0.1, 3 + b, _trunk_xfrc(m)))
        _run(bk, starts, mc, U[:steps])
    snap = [(bank.get(b), bank.disturbance(b)) for b in range(B)]
    lib, d, u32 = bank.lib, C.c_double, C.c_uint32
    nan, inf = float("nan"), float("inf")
    for cs, cr, xs, xr in ((-0.1, 1, 0, 1), (nan, 1, 0, 1), (inf, 1, 0, 1), (0, 1, -1, 1), (0, 1, nan, 1),
                           (0.1, 0, 0, 1), (0.1, -1, 0, 1), (0.1, nan, 0, 1), (0.1, inf, 0, 1), (0, 1, 1, 0),
                           (0, 1, 1, nan), (1e39, 1, 0, 1)):
        assert lib.mjpc_b200_plant_set_disturbance(bank.h, 0, d(cs), d(cr), d(xs), d(xr), u32(1)) == BAD_ARGUMENT, \
            (cs, cr, xs, xr)
    bad = np.zeros(6 * m.nbody, np.float32); bad[7] = np.nan
    assert lib.mjpc_b200_plant_set_xfrc(bank.h, 0, bad.ctypes.data_as(C.POINTER(C.c_float))) == BAD_ARGUMENT
    bad[7] = np.inf
    assert lib.mjpc_b200_plant_set_xfrc(bank.h, 0, bad.ctypes.data_as(C.POINTER(C.c_float))) == BAD_ARGUMENT
    for p in (B, -1):
        with pytest.raises(EngineError, match="outside"):
            bank.set_disturbance(p, 0.1)
        with pytest.raises(EngineError, match="outside"):
            bank.set_xfrc(p, None)
        with pytest.raises(EngineError, match="outside"):
            bank.disturbance(p)
    assert lib.mjpc_b200_plant_last_ctrl(bank.h, None) == BAD_ARGUMENT
    for b in range(B):
        g, dist = bank.get(b), bank.disturbance(b)
        for f in snap[b][0]:
            _eq(g[f], snap[b][0][f], f"plant {b} {f} after refusals")
        for f in dist:
            _eq(dist[f], snap[b][1][f], f"plant {b} {f} after refusals")
    for k in range(steps, 2 * steps):
        a, r = bank.step(U[k]), control.step(U[k])
        for f in ("state", "ctrl"):
            _eq(a[f], r[f], f"step {k} {f} after refusals")
    # every new call is refused while a model ensemble is set
    bufs, arr, n = _model_blobs([m, m])
    assert lib.mjpc_b200_set_model_ensemble(bank.h, arr, n, n) == 0
    out = np.zeros((B, m.nu), np.float32)
    fp = C.POINTER(C.c_float)
    assert lib.mjpc_b200_plant_set_disturbance(bank.h, 0, d(0.1), d(1), d(0), d(1), u32(0)) == UNSUPPORTED
    assert lib.mjpc_b200_plant_set_xfrc(bank.h, 0, None) == UNSUPPORTED
    assert lib.mjpc_b200_plant_get_disturbance(bank.h, 0, None, None) == UNSUPPORTED
    assert lib.mjpc_b200_plant_last_ctrl(bank.h, out.ctypes.data_as(fp)) == UNSUPPORTED
    assert lib.mjpc_b200_set_model_ensemble(bank.h, None, 0, 0) == 0
    for b in range(B):
        _eq(bank.disturbance(b)["xfrc_noise"], control.disturbance(b)["xfrc_noise"], f"plant {b} after the ensemble")
    bank.close(); control.close()


# ------------------------------------------------------------------------------------------ 7. estimator in the loop
def test_estimator_receives_the_applied_ctrl():
    from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
    from mujoco_mpc_b200.engine import CppBatchSamplingPlanner
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    m = get_model("quadruped")
    B, steps, N, H = 2, 30, 32, 16
    mc, starts = mocap_of(m), _start(m, B)

    def setup():
        pl = CppBatchSamplingPlanner(m, B, N, H, seeds=[51, 52])
        est = CppBatchEstimator(m, "unscented", B, timestep=m.opt_timestep)
        bank = _bank(m, B, (est.sensor_start, est.nsensor))
        for b, (q, v) in enumerate(starts):
            pl.reset(b)
            bank.reset(b, q, v, 0.0, mc)
            bank.set_disturbance(b, ctrl_std=0.3, ctrl_rate=0.05, seed=60 + b)
            est.reset(b, state=np.concatenate([q, v]).astype(float), time=0.0)
        return pl, bank, est

    pl, bank, est = setup()
    out = synchronous_planning_cost(pl, bank, steps, 1, estimator=est)
    loop_est = np.array([est.state(b) for b in range(B)])
    pl.close(); bank.close(); est.close()
    # the same loop written out, the applied ctrl passed by hand (and, as a control, the commanded one)
    for passed in ("applied", "commanded"):
        pl, bank, est = setup()
        t = np.zeros(B)
        states = []
        for i in range(steps):
            ctrl = np.zeros((B, m.nu), np.float32)
            for b in range(B):
                pl.set_state(b, np.asarray(est.state(b), float), t[b], np.asarray(bank.mocap[b], float))
                ctrl[b] = pl.action_from_policy(b, t[b])
            o = bank.step(ctrl)
            t = o["time"].copy()
            states.append(o["state"])
            est.update(o["ctrl"] if passed == "applied" else ctrl, o["sensordata"].astype(float),
                       bank.mocap if m.nmocap else None)
            pl.optimize_policy()
        hand = np.array([est.state(b) for b in range(B)])
        if passed == "applied":
            _eq(np.array(states), out["states"], "states of the loop and the hand loop")
            _eq(hand, loop_est, "estimates of the loop and the hand loop")
        else:
            assert not np.array_equal(hand, loop_est)
        pl.close(); bank.close(); est.close()
