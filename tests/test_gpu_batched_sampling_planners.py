"""GPU: per-problem force-noise keys in a batched rollout launch (mjpc_b200_set_xfrc_noise_batched) and the batched
Cross-Entropy, Robust and Sample Gradient planners.  The reference for a batch is each problem run alone - a single
launch after set_xfrc_noise with that problem's key, or a single planner of the same kind on its own handle with its
own set_task - and every output must be BITWISE equal."""
import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_batched import _assert_problem_equal, _batched, _problems, _single

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, UNSUPPORTED = -1, -5
SEEDS = [0x5EED, 7, 123456]
STD, RATE = 2.0, 0.1


@pytest.mark.parametrize("name,shape", [("quadruped", "wide"), ("quadruped", "plain"), ("quadruped", "generic"),
                                        ("humanoid_track", "wide")])
def test_per_problem_noise_equals_separate_launches(name, shape, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    m = get_model(name)
    if shape == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    if shape == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    N, H = (12, 32) if name == "quadruped" else (8, 24)
    pr = _problems(m, N, H, B=3)
    e = Engine(m, 3 * N, H)
    clean = _batched(e, pr, H)
    e.set_xfrc_noise_batched(STD, RATE, SEEDS)
    batch = _batched(e, pr, H)
    assert e.last_kernel_shape == {"wide": 1, "plain": 2, "generic": 0}[shape]
    assert not batch["failure"].any()
    assert np.abs(batch["returns"] - clean["returns"]).max() > 1e-5          # the noise does act
    for b in range(3):
        e.set_xfrc_noise(STD, RATE, SEEDS[b])
        _assert_problem_equal(batch, _single(e, pr, b, H), b, N)
    e.close()


def test_per_problem_seeds_are_cleared_by_set_xfrc_noise():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 12, 24
    pr = _problems(m, N, H, B=3)
    e = Engine(m, 3 * N, H)
    e.set_xfrc_noise(STD, RATE, 99)
    before = _batched(e, pr, H)
    e.set_xfrc_noise_batched(STD, RATE, SEEDS)
    keyed = _batched(e, pr, H)
    e.set_xfrc_noise(STD, RATE, 99)
    after = _batched(e, pr, H)
    assert np.abs(keyed["returns"] - before["returns"]).max() > 1e-5
    for k in before:
        np.testing.assert_array_equal(before[k], after[k], err_msg=k)
    e.close()


def test_noise_key_argument_errors_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import Engine, EngineError
    m = get_model("quadruped")
    N, H = 8, 16
    pr = _problems(m, N, H, B=3)
    e = Engine(m, 3 * N, H)
    e.set_xfrc_noise_batched(STD, RATE, SEEDS)
    ref = _batched(e, pr, H)
    with pytest.raises(EngineError, match=f"error {BAD_ARGUMENT}"):          # two problems, three keys
        _batched(e, {k: v[:2] for k, v in pr.items()}, H)
    with pytest.raises(EngineError, match=f"error {UNSUPPORTED}"):           # sharded launches take one key
        e.rollout_spline_sharded(pr["states"][0], pr["times"][0], pr["mocaps"][0], pr["knots"][0], pr["knot_times"][0], 2, H)
    again = _batched(e, pr, H)
    for k in ref:
        np.testing.assert_array_equal(ref[k], again[k], err_msg=k)
    e.close()


# ---------------------------------------------------------------------------------------------- batched planners
def _planner_problems(m, name, B):
    """B distinct problems for a planner: start state, start time, mocap and task snapshot all differ."""
    if name == "quadruped":
        pr = _problems(m, 4, 24, B=B)
        return {k: pr[k] for k in ("states", "times", "mocaps", "weights", "parameters", "task_states")}
    rng = np.random.default_rng(5)
    states, mocaps = [], []
    for b in range(B):
        s = np.concatenate([m.key_qpos[0], 0.05 * b * rng.standard_normal(m.nv)])
        mc = mocap_of(m).reshape(-1, 7).copy()
        mc[:, :3] += 0.02 * b
        states.append(s); mocaps.append(mc.reshape(-1))
    weights = np.stack([np.asarray(m.task_weight, float) * (1.0 + 0.3 * b) for b in range(B)])
    return dict(states=np.stack(states), times=np.array([0.0, 0.13, 0.5])[:B], mocaps=np.stack(mocaps), weights=weights,
                parameters=np.tile(np.asarray(m.task_parameters, float), (B, 1)),
                task_states=np.tile(np.asarray(m.task_state, float), (B, 1)))


def _make(kind, m, B, N, H, seeds):
    from mujoco_mpc_b200 import engine as E
    if kind == "ce":
        return E.CppBatchCrossEntropyPlanner(m, B, N, H, seeds=seeds), [E.CppCrossEntropyPlanner(m, N, H, seed=s) for s in seeds]
    if kind == "robust":
        kw = dict(ncandidates=3, nrepetitions=4, xfrc_std=1.0, xfrc_rate=0.1)
        return (E.CppBatchRobustPlanner(m, B, N, H, seeds=seeds, **kw),
                [E.CppRobustPlanner(m, N, H, seed=s, **kw) for s in seeds])
    return (E.CppBatchSampleGradientPlanner(m, B, N, H, num_gradient=4, gradient_filter=0.6, seeds=seeds),
            [E.CppSampleGradientPlanner(m, N, H, num_gradient=4, gradient_filter=0.6, seed=s) for s in seeds])


def _set_task(pl, pr, b, problem=None):
    task = dict(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])
    if problem is None:
        pl.set_task(**task)
    else:
        pl.set_task(problem, **task)


def _assert_result_equal(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=f"{what}: {k}")


@pytest.mark.parametrize("kind,name,B,iters", [("ce", "quadruped", 3, 5), ("ce", "shadow_reorient", 3, 5),
                                               ("robust", "quadruped", 3, 5), ("sg", "quadruped", 3, 5),
                                               ("ce", "quadruped", 1, 3), ("robust", "quadruped", 1, 3),
                                               ("sg", "quadruped", 1, 3)])
def test_batch_equals_independent_planners(kind, name, B, iters):
    m = get_model(name)
    N, H = 16, 24
    seeds = SEEDS[:B]
    pr = _planner_problems(m, name, B)
    batch, singles = _make(kind, m, B, N, H, seeds)
    for b in range(B):
        batch.reset(b, np.zeros(m.nu)); singles[b].reset(np.zeros(m.nu))
        _set_task(batch, pr, b, b); _set_task(singles[b], pr, b)
    for it in range(iters):
        for b in range(B):
            t = pr["times"][b] + 0.01 * it
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
            singles[b].set_state(pr["states"][b], t, pr["mocaps"][b])
        res = batch.optimize_policy()
        for b in range(B):
            _assert_result_equal(res[b], singles[b].optimize_policy(), f"iteration {it} problem {b}")
            for dt in (0.0, 0.013, 0.05, 0.2):
                t = pr["times"][b] + 0.01 * it + dt
                for prev in (False, True):
                    np.testing.assert_array_equal(batch.action_from_policy(b, t, prev), singles[b].action_from_policy(t, prev))
    if B > 1:
        assert len({float(res[b]["returns"][0]) for b in range(B)}) == B     # the problems do differ
    if kind == "robust":
        assert all(len(r["scores"]) == 3 for r in res)
    batch.close()
    for s in singles:
        s.close()


@pytest.mark.parametrize("kind", ["ce", "robust", "sg"])
def test_problems_are_independent(kind):
    """Another state and task for problem 1 leave problems 0 and 2 bitwise as they were."""
    m = get_model("quadruped")
    N, H = 16, 24
    pr = _planner_problems(m, "quadruped", 3)
    ch = {k: np.array(v, copy=True) for k, v in pr.items()}
    ch["states"][1, m.nq:] += 0.3
    ch["weights"][1] *= 2.0
    ch["parameters"][1, m.task_parameter_names.index("residual_Walk speed")] += 0.2
    out = []
    for inputs in (pr, ch):
        batch, singles = _make(kind, m, 3, N, H, SEEDS)
        for s in singles:
            s.close()
        for b in range(3):
            batch.reset(b, np.zeros(m.nu)); _set_task(batch, inputs, b, b)
        for it in range(2):
            for b in range(3):
                batch.set_state(b, inputs["states"][b], inputs["times"][b] + 0.01 * it, inputs["mocaps"][b])
            res = batch.optimize_policy()
        out.append(res)
        batch.close()
    assert np.abs(out[0][1]["returns"] - out[1][1]["returns"]).max() > 1e-5
    for b in (0, 2):
        _assert_result_equal(out[0][b], out[1][b], f"problem {b}")


def test_sampling_family_kind_checks():
    """The generic batch entry points drive every kind; a kind-specific get_result refuses another kind and a problem
    outside the batch."""
    from mujoco_mpc_b200 import engine as E
    m = get_model("particle")
    H = 11
    batches = {"sampling": E.CppBatchSamplingPlanner(m, 2, 8, H), "ce": E.CppBatchCrossEntropyPlanner(m, 2, 8, H),
               "robust": E.CppBatchRobustPlanner(m, 2, 10, H), "sg": E.CppBatchSampleGradientPlanner(m, 2, 8, H, num_gradient=2)}
    getters = {"sampling": "mjpc_b200_batch_sampling_planner_get_result", "ce": "mjpc_b200_batch_ce_planner_get_result",
               "robust": "mjpc_b200_batch_robust_planner_get_result", "sg": "mjpc_b200_batch_sg_planner_get_result"}
    for kind, bp in batches.items():
        for b in range(2):
            bp.reset(b); bp.set_state(b, np.zeros(4), 0.0, mocap_of(m))
        res = bp.optimize_policy()
        assert len(res) == 2 and bp.action_from_policy(1, 0.02).shape == (m.nu,)
        lib = bp.lib
        for other, getter in getters.items():
            rc = getattr(lib, getter)(bp.h, 0, *([None] * 9))
            assert (rc == BAD_ARGUMENT) == (other != kind), (kind, other)
        assert getattr(lib, getters[kind])(bp.h, 2, *([None] * 9)) == BAD_ARGUMENT
        assert lib.mjpc_b200_batch_planner_reset(bp.h, -1, H, None) == BAD_ARGUMENT
    for bp in batches.values():
        bp.close()


def test_batch_ce_particles_reach_their_goals():
    """The Predictive Sampling batch's bar for Cross-Entropy: four particles with different goals, planned together,
    each reach their own."""
    from mujoco_mpc_b200.engine import CppBatchCrossEntropyPlanner, Engine
    m = get_model("particle")
    H, B = 11, 4
    goals = [(0.25, 0.0), (-0.25, 0.0), (0.0, 0.25), (0.0, -0.25)]
    mocaps = []
    for g in goals:
        mc = mocap_of(m).copy(); mc[:2] = g
        mocaps.append(mc)
    pl = CppBatchCrossEntropyPlanner(m, B, 16, H)
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
