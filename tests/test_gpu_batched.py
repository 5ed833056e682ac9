"""GPU: several independent planning problems in one rollout launch (mjpc_b200_rollout_spline_batched) and the batched
Predictive Sampling planner.  The reference for a batch is each problem run alone: every output must be BITWISE equal."""
import numpy as np
import pytest

from conftest import get_model, mocap_of, quadruped_inputs

pytestmark = pytest.mark.gpu

TIMES = np.array([0.0, 0.13, 0.5, 1.7])
ARRAYS = ("states", "actions", "times", "residual", "costs", "trace")


def _track_mocap(m):
    return np.concatenate([m.key_mpos[0].reshape(-1, 3), np.tile([1.0, 0, 0, 0], (m.nmocap, 1))], 1).reshape(-1)


def _problems(m, N, H, B=4):
    """B distinct problems: start state, absolute start time, mocap goal, task snapshot and knots all differ."""
    from mujoco_mpc_b200 import task as T
    rng = np.random.default_rng(11)
    times = TIMES[:B]
    track = m.nmocap == 16                                  # Humanoid Track (else the Quadruped)
    if track:
        P = 8
        base_state = np.concatenate([m.key_qpos[0], m.key_qvel[0]])
        base_mocap = _track_mocap(m)
        kt = np.arange(P) * (H - 1) * 0.005 / (P - 1)
        knots = [np.clip(0.05 * rng.standard_normal((N, P, m.nu)), -1, 1) for _ in range(B)]
    else:
        base_state, base_mocap, _, kt = quadruped_inputs(m, N=N, H=H)
        knots = [quadruped_inputs(m, N=N, H=H, seed=b)[2] for b in range(B)]
    states, mocaps, weights, params, tstates = [], [], [], [], []
    for b in range(B):
        s = np.asarray(base_state, float).copy()
        s[m.nq:] += 0.05 * b * rng.standard_normal(m.nv)
        mc = np.asarray(base_mocap, float).copy().reshape(-1, 7)
        mc[:, :3] += 0.02 * b * rng.standard_normal((len(mc), 3))
        w = np.asarray(m.task_weight, float) * (1.0 + 0.3 * b)
        p = np.asarray(m.task_parameters, float).copy()
        ts = np.asarray(m.task_state, float).copy()
        if track:                                           # reference time (absolute)
            ts[1] = times[b] - 0.01 * b
        else:                                               # Quadruped: gait / mode clocks (absolute), walk speed
            p[m.task_parameter_names.index("residual_Amplitude")] += 0.02 * b
            ts[T.QS_MODE_START_TIME] = times[b] - 0.05 * b
            ts[T.QS_PHASE_START_TIME] = times[b] - 0.03 * b
        states.append(s); mocaps.append(mc.reshape(-1)); weights.append(w); params.append(p); tstates.append(ts)
    kabs = np.stack([kt + t for t in times])
    return dict(states=np.stack(states), times=times, mocaps=np.stack(mocaps), knots=np.stack(knots), knot_times=kabs,
                weights=np.stack(weights), parameters=np.stack(params), task_states=np.stack(tstates))


def _batched(e, pr, H, **over):
    a = dict(pr, **over)
    ret, fail, order = e.rollout_spline_batched(a["states"], a["times"], a["mocaps"], a["knots"], a["knot_times"], 2, H,
                                                weights=a["weights"], parameters=a["parameters"], task_states=a["task_states"])
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _single(e, pr, b, H):
    """Problem b alone, through set_task + rollout_spline."""
    e.set_task(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])
    ret, fail, order = e.rollout_spline(pr["states"][b], pr["times"][b], pr["mocaps"][b], pr["knots"][b], pr["knot_times"][b], 2, H)
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _assert_problem_equal(batch, single, b, N):
    for k in ("returns", "failure", "order"):
        np.testing.assert_array_equal(batch[k][b], single[k], err_msg=f"problem {b}: {k}")
    for k in ARRAYS:
        np.testing.assert_array_equal(batch[k][b * N:(b + 1) * N], single[k], err_msg=f"problem {b}: {k}")


@pytest.mark.parametrize("name,shape", [("quadruped", "wide"), ("quadruped", "plain"), ("quadruped", "generic"),
                                        ("humanoid_track", "wide")])
def test_batched_launch_equals_separate_launches(name, shape, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    m = get_model(name)
    if shape == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    if shape == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    N, H = (12, 32) if name == "quadruped" else (8, 24)
    pr = _problems(m, N, H)
    e = Engine(m, 4 * N, H)
    batch = _batched(e, pr, H)
    assert e.last_kernel_shape == {"wide": 1, "plain": 2, "generic": 0}[shape]
    assert batch["returns"].shape == (4, N) and not batch["failure"].any()
    assert np.abs(batch["returns"][0] - batch["returns"][1]).max() > 1e-4     # the problems do differ
    for b in range(4):
        _assert_problem_equal(batch, _single(e, pr, b, H), b, N)
    e.close()


def test_single_problem_batch_and_handle_task_values():
    """B = 1 is rollout_spline; NULL task arrays mean the handle's set_task values in every problem."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 12, 24
    pr = _problems(m, N, H, B=3)
    e = Engine(m, 3 * N, H)
    one = {k: v[:1] for k, v in pr.items()}
    batch = _batched(e, one, H, weights=None, parameters=None, task_states=None)
    ret, fail, order = e.rollout_spline(pr["states"][0], pr["times"][0], pr["mocaps"][0], pr["knots"][0], pr["knot_times"][0], 2, H)
    single = dict(e.fetch_all(), returns=ret, failure=fail, order=order)
    _assert_problem_equal(batch, single, 0, N)
    # NULL arrays vs the same snapshot given explicitly for every problem
    w, p, ts = pr["weights"][2], pr["parameters"][2], pr["task_states"][2]
    e.set_task(weight=w, parameters=p, task_state=ts)
    implicit = _batched(e, pr, H, weights=None, parameters=None, task_states=None)
    explicit = _batched(e, pr, H, weights=np.tile(w, (3, 1)), parameters=np.tile(p, (3, 1)), task_states=np.tile(ts, (3, 1)))
    for k in implicit:
        np.testing.assert_array_equal(implicit[k], explicit[k], err_msg=k)
    e.close()


def test_problems_are_independent():
    """Changing every input of one problem leaves the outputs of the others bitwise unchanged."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 12, 24
    pr = _problems(m, N, H)
    e = Engine(m, 4 * N, H)
    before = _batched(e, pr, H)
    ch = {k: np.array(v, copy=True) for k, v in pr.items()}
    ch["states"][2, m.nq:] += 0.3
    ch["mocaps"][2, :3] += 0.1
    ch["knots"][2] = np.clip(ch["knots"][2][::-1] + 0.05, -1, 1)
    ch["weights"][2] *= 2.0
    ch["parameters"][2, m.task_parameter_names.index("residual_Walk speed")] += 0.2
    ch["task_states"][2, 1] -= 0.2
    after = _batched(e, ch, H)
    assert np.abs(after["returns"][2] - before["returns"][2]).max() > 1e-4
    for b in (0, 1, 3):
        _assert_problem_equal(after, {k: (v[b] if k in ("returns", "failure", "order") else v[b * N:(b + 1) * N])
                                      for k, v in before.items()}, b, N)
    e.close()


def test_pair_synchronisation_stays_timing_only_on_a_batch(monkeypatch):
    """4 x 60 candidates lie in (#SMs, 2 #SMs]: the co-resident pair synchronisation is on by default."""
    import torch
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    B, N, H = 4, 60, 12
    assert nsm < B * N <= 2 * nsm
    pr = _problems(m, N, H, B=B)
    e = Engine(m, B * N, H)
    out = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("MJPC_B200_PAIR_SYNC", mode)
        out[mode] = _batched(e, pr, H)
    assert not out["0"]["failure"].any()
    for k in out["0"]:
        np.testing.assert_array_equal(out["0"][k], out["1"][k], err_msg=k)
    e.close()


def test_per_problem_task_snapshots_take_effect():
    """Zero weights give zero returns (ties: candidate 0 ranks first); another quadruped mode and gait give exactly
    what a single launch with that task gives."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 12, 16
    pr = _problems(m, N, H, B=2)
    pr["weights"][0] = 0.0
    ts = pr["task_states"][1]
    ts[T.QS_MODE] = 1; ts[T.QS_HEADING] = 1.0; ts[T.QS_SPEED] = 0.5; ts[T.QS_ORIENTATION] = 1.0
    pr["parameters"][1, m.task_parameter_names.index("residual_Cadence")] *= 1.5
    pr["parameters"][1, m.task_parameter_names.index("residual_Duty ratio")] = 0.3
    e = Engine(m, 2 * N, H)
    batch = _batched(e, pr, H)
    assert not batch["failure"].any()
    np.testing.assert_array_equal(batch["returns"][0], np.zeros(N, np.float32))
    np.testing.assert_array_equal(batch["order"][0], np.arange(N))
    assert (batch["returns"][1] > 0).all()
    _assert_problem_equal(batch, _single(e, pr, 1, H), 1, N)
    e.close()


def test_batched_argument_errors_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import Engine, EngineError
    m = get_model("quadruped")
    N, H = 8, 16
    pr = _problems(m, N, H)
    e = Engine(m, 4 * N, H)
    ref = _batched(e, pr, H)
    cut = lambda B, n: {k: (v[:B, :n] if k == "knots" else v[:B]) for k, v in pr.items()}
    with pytest.raises(EngineError, match="error -3"):             # B * N > max_candidates
        big = dict(pr, knots=np.concatenate([pr["knots"], pr["knots"][:, :1]], 1))
        _batched(e, big, H)
    with pytest.raises(EngineError):                               # B = 0
        _batched(e, cut(0, N), H)
    with pytest.raises(EngineError):                               # N = 0
        _batched(e, cut(4, 0), H)
    with pytest.raises(EngineError):                               # P > 64
        _batched(e, pr, H, knots=np.zeros((4, N, 65, m.nu)), knot_times=np.tile(np.linspace(0, 0.1, 65), (4, 1)))
    with pytest.raises(EngineError):                               # H > max_horizon
        _batched(e, pr, H + 1)
    again = _batched(e, pr, H)
    for k in ref:
        np.testing.assert_array_equal(ref[k], again[k], err_msg=k)
    e.close()


def test_batch_planner_equals_independent_planners():
    """CppBatchSamplingPlanner (one launch per iteration) vs one CppSamplingPlanner per problem (one launch each)."""
    from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, CppSamplingPlanner
    m = get_model("quadruped")
    B, N, H = 3, 16, 24
    seeds = [0x5EED, 7, 123456]
    pr = _problems(m, N, H, B=B)
    batch = CppBatchSamplingPlanner(m, B, N, H, seeds=seeds)
    singles = [CppSamplingPlanner(m, N, H, seed=s) for s in seeds]
    for b in range(B):
        batch.reset(b); singles[b].reset()
    for it in range(5):
        for b in range(B):
            t = pr["times"][b] + 0.01 * it
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
            singles[b].set_state(pr["states"][b], t, pr["mocaps"][b])
        res = batch.optimize_policy()
        for b in range(B):
            r = singles[b].optimize_policy()
            for k in ("returns", "knots", "knot_times"):
                np.testing.assert_array_equal(res[b][k], r[k], err_msg=f"iteration {it} problem {b}: {k}")
            assert res[b]["winner"] == r["winner"] and res[b]["improvement"] == r["improvement"]
            t = pr["times"][b] + 0.01 * it + 0.05
            for prev in (False, True):
                np.testing.assert_array_equal(batch.action_from_policy(b, t, prev), singles[b].action_from_policy(t, prev))
    assert len({float(res[b]["returns"][0]) for b in range(B)}) == B
    with pytest.raises(Exception):
        batch.set_state(B, pr["states"][0], 0.0, pr["mocaps"][0])
    batch.close()
    for s in singles:
        s.close()


def test_batch_planner_particles_reach_their_goals():
    """sampling_planner_test's bar on a batch: four particles with different goals, planned together, each reach their own."""
    from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, Engine
    m = get_model("particle")
    H, B = 11, 4
    goals = [(0.25, 0.0), (-0.25, 0.0), (0.0, 0.25), (0.0, -0.25)]
    mocaps = []
    for g in goals:
        mc = mocap_of(m).copy(); mc[:2] = g
        mocaps.append(mc)
    pl = CppBatchSamplingPlanner(m, B, 16, H)
    for b in range(B):
        pl.reset(b); pl.set_state(b, np.zeros(4), 0.0, mocaps[b])
    for _ in range(150):
        res = pl.optimize_policy()
        assert all(r["improvement"] >= 0 for r in res)
    e = Engine(m, 1, H)
    for b in range(B):
        e.rollout_spline(np.zeros(4), 0.0, mocaps[b], res[b]["knots"][None], res[b]["knot_times"],
                         int(m.numeric.get("sampling_representation", [2])[0]), H)
        tr = e.fetch_trajectory(0)
        assert np.abs(tr["states"][-1, :2] - np.asarray(goals[b])).max() < 0.1, b
        assert (np.abs(tr["actions"]) <= 1 + 1e-6).all()
    pl.close(); e.close()
