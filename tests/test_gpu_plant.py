"""GPU: closed-loop plants (mjpc_b200_plant_*, engine.CppPlantBank) and the batched closed loop
(closed_loop.synchronous_planning_cost).

A plant step runs the device functions of mjpc_b200_step_batch, so its reference is step_batch with the plant's time,
task rows and warm start: every output must be BITWISE equal.  Model variants, positions in the bank and the other
plants' inputs must not change a plant's trajectory.  The batched loop must be bitwise B loops of one; against the
fp64 oracle plant it must hold the bars tests/test_closed_loop.py holds a device planner to."""
import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_model_variants import _variants

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, UNSUPPORTED = -1, -5
QUAD_SENSORS = (9, 21)   # the Quadruped's measured sensors: 5 framepos, 12 jointpos, 4 touch


def _eq(a, b, what):
    assert np.array_equal(np.asarray(a), np.asarray(b)), what


def _bank(m, B, sensors=(None, 0)):
    from mujoco_mpc_b200.engine import CppPlantBank
    return CppPlantBank(m, B, sensor_start=sensors[0], nsensor=sensors[1])


def _track_mocap(m, k=0):
    mpos = np.asarray(m.key_mpos[k]).reshape(m.nmocap, 3)
    return np.concatenate([mpos, np.tile([1.0, 0, 0, 0], (m.nmocap, 1))], 1).reshape(-1)


def _start(m, B, seed=3):
    """B bench-like start states: the home (Quadruped) or first reference keyframe, with perturbed velocities."""
    rng = np.random.default_rng(seed)
    q0 = m.key_qpos[0]
    v0 = np.zeros(m.nv) if m.nmocap != 16 else m.key_qvel[0]
    return [(np.asarray(q0, np.float32), np.asarray(v0 + 0.05 * b * rng.standard_normal(m.nv), np.float32))
            for b in range(B)]


def _mocap(m):
    return _track_mocap(m) if m.nmocap == 16 else mocap_of(m)


def _ctrl(m, B, steps, seed=0):
    return np.clip(0.4 * np.random.default_rng(seed).standard_normal((steps, B, m.nu)), -1, 1).astype(np.float32)


# ------------------------------------------------------------------------------------------ 1. a step is step_batch's
@pytest.mark.parametrize("case", ["quadruped", "quadruped-generic", "humanoid_track"])
def test_plant_step_equals_step_batch(case, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    name = case.split("-")[0]
    if case.endswith("generic"):
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model(name)
    B, steps, t0 = 8, 30, 0.37
    sensors = QUAD_SENSORS if name == "quadruped" else (None, 0)
    bank, e = _bank(m, B, sensors), Engine(m, B, 4)
    mc = _mocap(m)
    start = _start(m, B)
    for b, (q, v) in enumerate(start):
        bank.reset(b, q, v, t0, mc)
    q = np.array([s[0] for s in start]); v = np.array([s[1] for s in start])
    warm = np.zeros((B, m.nv), np.float32)
    t, warnings = t0, np.zeros(B, int)
    U = _ctrl(m, B, steps)
    for k in range(steps):
        o = bank.step(U[k])
        assert bank.last_kernel_static() == (0 if case.endswith("generic") or name == "particle" else 1)
        r = e.step_batch(q, v, U[k], mc, np.full(B, t), time0=t, warmstart=warm)
        assert (o["status"] == 0).all()
        _eq(o["state"], np.concatenate([r["next_qpos"], r["next_qvel"]], 1), f"{case} step {k} state")
        _eq(o["cost"], r["cost"], f"{case} step {k} cost")
        if sensors[1]:
            for b in range(B):
                s = e.step_sensors(np.concatenate([q[b], v[b]])[None], U[k, b], mc, t, *sensors, warmstart=warm[b][None])
                _eq(o["sensordata"][b], s["sensordata"][0], f"{case} step {k} plant {b} sensors")
        warnings += r["warning"]
        t += m.opt_timestep
        _eq(o["time"], np.full(B, t), f"{case} step {k} time")
        q, v, warm = r["next_qpos"], r["next_qvel"], r["qacc"]
    for b in range(B):
        g = bank.get(b)
        _eq(g["warmstart"], warm[b], f"{case} plant {b} warm start")
        assert g["steps"] == steps and g["warnings"] == warnings[b] and g["status"] == 0
    e.close(); bank.close()


# ------------------------------------------------------------------------------------------ 2. variants
def _run(bank, starts, mc, U, t0=0.0):
    for b, (q, v) in enumerate(starts):
        bank.reset(b, q, v, t0, mc)
    return [bank.step(u) for u in U]


def test_variant_plants_equal_a_bank_per_variant():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, steps = 4, 30
    mc, starts, U = mocap_of(base), _start(base, B), _ctrl(base, B, steps, seed=1)
    bank = _bank(base, B, QUAD_SENSORS)
    bank.set_models(V)
    got = _run(bank, starts, mc, U)
    for b in range(B):
        one = _bank(V[b], 1, QUAD_SENSORS)
        ref = _run(one, starts[b:b + 1], mc, U[:, b:b + 1])
        for k in range(steps):
            for f in ("state", "cost", "time", "sensordata", "status"):
                _eq(got[k][f][b], ref[k][f][0], f"variant {b} step {k} {f}")
        one.close()
    assert len({float(got[-1]["state"][b, 2]) for b in range(B)}) == B    # the variants step differently
    bank.set_models(None)
    fresh = _bank(base, B, QUAD_SENSORS)
    a, r = _run(bank, starts, mc, U), _run(fresh, starts, mc, U)
    for k in range(steps):
        for f in ("state", "cost", "sensordata"):
            _eq(a[k][f], r[k][f], f"cleared step {k} {f}")
    bank.close(); fresh.close()


# ------------------------------------------------------------------------------------------ 3. independence
def test_a_plant_is_independent_of_its_position_and_the_others():
    m = get_model("quadruped")
    steps, B = 30, 8
    mc = mocap_of(m)
    me = _start(m, 1, seed=9)[0]
    mine = _ctrl(m, 1, steps, seed=2)
    alone = _bank(m, 1)
    ref = _run(alone, [me], mc, mine)
    alone.close()
    bank = _bank(m, B)
    for j in range(B):
        starts = _start(m, B, seed=10 + j)
        starts[j] = me
        U = _ctrl(m, B, steps, seed=20 + j)
        U[:, j] = mine[:, 0]
        got = _run(bank, starts, mc, U)
        for k in range(steps):
            _eq(got[k]["state"][j], ref[k]["state"][0], f"position {j} step {k}")
            _eq(got[k]["cost"][j], ref[k]["cost"][0], f"position {j} step {k} cost")
    bank.close()


# ------------------------------------------------------------------------------------------ 4. per-plant task rows
def test_humanoid_track_plants_read_their_own_task_rows():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("humanoid_track")
    B, steps, t0 = 4, 10, 0.2
    bank, e = _bank(m, B), Engine(m, 1, 4)
    mc = _track_mocap(m, 3)
    starts = _start(m, B)
    ts = [np.array([0.0, t0 - 0.05 * b]) for b in range(B)]      # (mode, reference time): each plant its own clip clock
    for b, (q, v) in enumerate(starts):
        bank.reset(b, q, v, t0, mc)
        bank.set_task(b, task_state=ts[b])
    U = _ctrl(m, B, steps, seed=4)
    q = [s[0] for s in starts]; v = [s[1] for s in starts]; warm = [np.zeros(m.nv, np.float32)] * B
    t = t0
    for k in range(steps):
        o = bank.step(U[k])
        for b in range(B):
            e.set_task(task_state=ts[b])
            r = e.step_batch(q[b][None], v[b][None], U[k, b][None], mc, [t], time0=t, warmstart=warm[b][None])
            _eq(o["state"][b], np.concatenate([r["next_qpos"][0], r["next_qvel"][0]]), f"plant {b} step {k}")
            _eq(o["cost"][b], r["cost"][0], f"plant {b} step {k} cost")
            q[b], v[b], warm[b] = r["next_qpos"][0], r["next_qvel"][0], r["qacc"][0]
        t += m.opt_timestep
    assert len({float(o["cost"][b]) for b in range(B)}) == B
    e.close(); bank.close()


# ------------------------------------------------------------------------------------------ 5. divergence
def test_a_diverged_plant_is_held_and_the_others_step_on():
    from mujoco_mpc_b200.engine import PLANT_DIVERGED
    m = get_model("quadruped")
    B, steps = 4, 5
    mc, starts, U = mocap_of(m), _start(m, B), _ctrl(m, B, steps, seed=5)
    ctrl_bank = _bank(m, B)
    ref = _run(ctrl_bank, starts, mc, U)
    bank = _bank(m, B)
    bad_v = starts[2][1].copy(); bad_v[3] = np.nan
    for b, (q, v) in enumerate(starts):
        bank.reset(b, q, bad_v if b == 2 else v, 0.0, mc)
    before = bank.get(2)
    for k in range(steps):
        o = bank.step(U[k])
        assert o["status"].tolist() == [0, 0, PLANT_DIVERGED, 0]
        assert o["cost"][2] == 0 and o["time"][2] == 0.0
        for b in (0, 1, 3):
            _eq(o["state"][b], ref[k]["state"][b], f"step {k} plant {b}")
    after = bank.get(2)
    assert after["status"] == PLANT_DIVERGED and after["steps"] == 0 and after["cost_sum"] == 0 and after["time"] == 0
    assert np.array_equal(after["state"], before["state"], equal_nan=True), "diverged plant's state"
    bank.reset(2, *starts[2], 0.0, mc)
    o = bank.step(U[0])
    assert o["status"][2] == 0
    _eq(o["state"][2], ref[0]["state"][2], "reset plant runs again")
    bank.close(); ctrl_bank.close()


# ------------------------------------------------------------------------------------------ 6. refusals
def test_refusals_leave_the_bank_usable_and_unchanged():
    import ctypes as C
    from mujoco_mpc_b200.engine import Engine, EngineError
    base, V = get_model("quadruped"), _variants("quadruped")
    B, steps = 8, 4
    mc, starts, U = mocap_of(base), _start(base, B), _ctrl(base, B, 2 * steps, seed=6)
    bank, control = _bank(base, B), _bank(base, B)
    a, r = _run(bank, starts, mc, U[:steps]), _run(control, starts, mc, U[:steps])
    snap = [bank.get(b) for b in range(B)]
    bank.set_models(V[:4])                                          # 4 variants for 8 plants
    with pytest.raises(EngineError, match="plant step"):
        bank.step(U[steps])
    bank.set_models(None)
    for bad in (B, -1):
        with pytest.raises(EngineError, match="outside"):
            bank.reset(bad, *starts[0], 0.0, mc)
        with pytest.raises(EngineError, match="outside"):
            bank.get(bad)
    lib = bank.lib
    assert lib.mjpc_b200_plant_init(bank.h, B, 0, 1) == UNSUPPORTED              # a residual (user) sensor
    assert lib.mjpc_b200_plant_init(bank.h, B, base.nsensor - 1, 2) == BAD_ARGUMENT
    assert lib.mjpc_b200_plant_init(bank.h, 10 ** 6, 0, 0) == -3                 # above max_candidates
    for b in range(B):
        g = bank.get(b)
        for f in snap[b]:
            _eq(g[f], snap[b][f], f"plant {b} {f} after refusals")
    for k in range(steps, 2 * steps):
        _eq(bank.step(U[k])["state"], control.step(U[k])["state"], f"step {k} after refusals")
    e = Engine(base, 4, 4)                                          # a handle without plants
    u = np.zeros((4, base.nu), np.float32)
    assert lib.mjpc_b200_plant_step(e.h, u.ctypes.data_as(C.POINTER(C.c_float)), None, None, None, None, None) == BAD_ARGUMENT
    assert b"plant_init" in lib.mjpc_b200_last_error()
    e.close(); bank.close(); control.close()


# ------------------------------------------------------------------------------------------ 7. batched loop = loops of one
def _planner(kind, m, B, seeds, N=32, H=16):
    from mujoco_mpc_b200 import engine as E
    if kind == "sampling":
        return E.CppBatchSamplingPlanner(m, B, N, H, seeds=seeds)
    if kind == "ce":
        return E.CppBatchCrossEntropyPlanner(m, B, N, H, seeds=seeds)
    return E.CppBatchILQGPlanner(m, B, H, num_rollouts=4)


def _episode(kind, m, plant_models, starts, mc, t0s, steps, spp, seeds, transitions=None, estimator=None, N=32, H=16):
    """One synchronous_planning_cost run: a batch planner on model m (its problems on plant_models when they differ
    from m), a bank on plant_models."""
    from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
    B = len(starts)
    pl = _planner(kind, m, B, seeds, N, H)
    bank = _bank(m, B, (estimator.sensor_start, estimator.nsensor) if estimator else (None, 0))
    if plant_models is not None:
        bank.set_models(plant_models)
        pl.set_models(plant_models)
    for b, (q, v) in enumerate(starts):
        pl.reset(b)
        bank.reset(b, q, v, t0s[b], mc)
        if estimator is not None:
            estimator.reset(b, state=np.concatenate([q, v]).astype(float), time=t0s[b])
    out = synchronous_planning_cost(pl, bank, steps, spp, transitions=transitions, estimator=estimator)
    pl.close(); bank.close()
    return out


def _assert_loops_equal(batched, singles, what):
    for b, one in enumerate(singles):
        for f in ("costs", "states", "status"):
            _eq(batched[f][:, b], one[f][:, 0], f"{what} episode {b} {f}")
        _eq(batched["average_cost"][b], one["average_cost"][0], f"{what} episode {b} average")


@pytest.mark.parametrize("kind", ["sampling", "ce", "ilqg"])
def test_batched_loop_equals_single_loops_quadruped(kind):
    base, V = get_model("quadruped"), _variants("quadruped")[:3]
    B, steps, spp, seeds = 3, 60, 4, [11, 12, 13]
    mc, starts = mocap_of(base), _start(base, B)
    batched = _episode(kind, base, V, starts, mc, [0.0] * B, steps, spp, seeds)
    singles = [_episode(kind, V[b], None, starts[b:b + 1], mc, [0.0], steps, spp, seeds[b:b + 1]) for b in range(B)]
    _assert_loops_equal(batched, singles, kind)
    assert (batched["final_status"] == 0).all()
    print(f"{kind}: average cost per plant {batched['average_cost']}, x-realtime {batched['x_realtime']:.2f}")


def test_batched_loop_equals_single_loops_humanoid_track():
    from mujoco_mpc_b200.transition import HumanoidTrackTransition
    base, V = get_model("humanoid_track"), _variants("humanoid_track")[:3]
    B, steps, spp, seeds = 3, 40, 4, [21, 22, 23]
    t0s = [0.0, 0.1, 0.25]
    mc, starts = _track_mocap(base), _start(base, B)
    batched = _episode("sampling", base, V, starts, mc, t0s, steps, spp, seeds,
                       transitions=[HumanoidTrackTransition(base) for _ in range(B)], H=41)
    singles = [_episode("sampling", V[b], None, starts[b:b + 1], mc, t0s[b:b + 1], steps, spp, seeds[b:b + 1],
                        transitions=[HumanoidTrackTransition(V[b])], H=41) for b in range(B)]
    _assert_loops_equal(batched, singles, "humanoid track")
    assert (batched["final_status"] == 0).all()
    print("humanoid track: average cost per plant", batched["average_cost"])


# ------------------------------------------------------------------------------------------ 8. against the fp64 plant
def test_device_plant_loop_against_the_fp64_plant(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import CppBatchSamplingPlanner
    m = get_model("quadruped")
    steps, N, H, seed = 60, 64, 32, 0x5EED
    q0, v0 = m.key_qpos[0].astype(np.float32), np.zeros(m.nv, np.float32)
    mc = mocap_of(m)
    dev = _episode("sampling", m, None, [(q0, v0)], mc, [0.0], steps, 1, [seed], N=N, H=H)
    # the same loop order on the fp64 oracle plant
    plant = oracle_lib.Oracle(to_blob(m), m, 64)
    pl = CppBatchSamplingPlanner(m, 1, N, H, seeds=[seed])
    pl.reset(0)
    q, v, t, warm, costs, heights = q0.astype(float), v0.astype(float), 0.0, None, [], []
    for i in range(steps):
        pl.set_state(0, np.concatenate([q, v]), t, mc)
        u = pl.action_from_policy(0, t)
        r = plant.forward_debug(q, v, u, mc, time=t, warmstart=warm)
        costs.append(plant.cost_value(r["residual"][: m.task_num_residual]))
        warm, q, v = r["qacc"], r["next_qpos"], r["next_qvel"]
        t += m.opt_timestep
        heights.append(q[2])
        pl.optimize_policy()
    pl.close()
    costs = np.array(costs)
    c_dev = dev["costs"][:, 0].astype(float)
    print("device plant vs fp64 plant: first costs %s / %s; average %.4f / %.4f; min trunk height %.3f / %.3f" % (
        c_dev[:5], costs[:5], dev["average_cost"][0], costs.mean(), dev["states"][:, 0, 2].min(), min(heights)))
    np.testing.assert_allclose(c_dev[:5], costs[:5], rtol=2e-3)
    assert abs(dev["average_cost"][0] - costs.mean()) < 0.1 * costs.mean()
    assert (dev["states"][:, 0, 2] > 0.15).all() and min(heights) > 0.15


# ------------------------------------------------------------------------------------------ 9. nominal planning, variant plants
def test_planning_on_the_nominal_model_keeps_every_variant_plant_up():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, steps = 4, 60
    mc, starts = mocap_of(base), _start(base, B)
    # planning every step, as the fp64-plant comparison above (at 4 steps per plan the nominal plant's trunk sinks to
    # about 0.147 m by the 60th step)
    from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
    pl = _planner("sampling", base, B, [31, 32, 33, 34], N=64, H=32)
    bank = _bank(base, B)
    bank.set_models(V)                                               # the planner keeps the nominal model
    for b, (q, v) in enumerate(starts):
        pl.reset(b); bank.reset(b, q, v, 0.0, mc)
    out = synchronous_planning_cost(pl, bank, steps, 1)
    zero = _run(bank, starts, mc, np.zeros((steps, B, base.nu), np.float32))
    zero_avg = np.array([bank.get(b)["cost_sum"] / steps for b in range(B)])
    print("nominal planning on variants: average cost %s, zero control %s, min trunk height %s" % (
        out["average_cost"], zero_avg, out["states"][:, :, 2].min(0)))
    assert (out["final_status"] == 0).all() and (out["states"][:, :, 2] > 0.15).all()
    assert (out["average_cost"] < zero_avg).all()
    pl.close(); bank.close()


# ------------------------------------------------------------------------------------------ 10. estimator in the loop
def test_estimator_in_the_loop():
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    base, V = get_model("quadruped"), _variants("quadruped")[:3]
    B, steps, spp, seeds, N, H = 3, 60, 1, [41, 42, 43], 64, 32
    mc, starts = mocap_of(base), _start(base, B)

    def estimator(models):
        f = CppBatchEstimator(base if len(models) > 1 else models[0], "unscented", len(models),
                              timestep=base.opt_timestep)
        if len(models) > 1:
            f.set_models(models)
        return f
    fb = estimator(V)
    batched = _episode("sampling", base, V, starts, mc, [0.0] * B, steps, spp, seeds, estimator=fb, N=N, H=H)
    est = np.array([fb.state(b) for b in range(B)])
    for b in range(B):
        f1 = estimator([V[b]])
        one = _episode("sampling", V[b], None, starts[b:b + 1], mc, [0.0], steps, spp, seeds[b:b + 1], estimator=f1,
                       N=N, H=H)
        for f in ("costs", "states", "status"):
            _eq(batched[f][:, b], one[f][:, 0], f"estimator episode {b} {f}")
        _eq(f1.state(0), est[b], f"estimate {b}")
        f1.close()
    err = est - batched["states"][-1].astype(float)
    print("estimator in the loop: RMS qpos error %.3e, qvel error %.3e; min trunk height %s" % (
        np.sqrt(np.mean(err[:, :base.nq] ** 2)), np.sqrt(np.mean(err[:, base.nq:] ** 2)),
        batched["states"][:, :, 2].min(0)))
    assert (batched["final_status"] == 0).all() and (batched["states"][:, :, 2] > 0.15).all()
    fb.close()
