"""GPU: model ensembles (mjpc_b200_set_model_ensemble and the planners' set_ensemble).

Each member's rollouts must be BITWISE those of a handle with model variants set and the member's variant selected for
every problem; each candidate's score must be bitwise the host definition (mjpc_b200_host_ensemble_score) over the
member returns, and its order a stable argsort of the scores.  A one-member ensemble of the handle's own model changes
nothing, clearing gives a fresh handle, and the planners plan on the scores exactly as their batches do."""
import ctypes as C

import numpy as np
import pytest

from conftest import get_model
from test_gpu_batched import _problems
from test_gpu_model_variants import (SEEDS, _assert_equal, _engine, _refusal_variants, _set_shape, _spline,
                                     _spline_handle_task, _sub, _variant, _variants)

pytestmark = pytest.mark.gpu

BAD_ARGUMENT = -1


def _problems_of(pr, B):
    return {k: v[:B] for k, v in pr.items()}


def _on_variant(name, base, V, pr, N, H, k, B):
    """every problem of pr on variant k of V: set_model_variants + select_model_variants on a fresh handle"""
    ref = _engine(base, B * N, H)
    ref.set_model_variants(V)
    idx = np.full(B, k, np.int32)
    assert ref.lib.mjpc_b200_select_model_variants(ref.h, idx.ctypes.data_as(C.POINTER(C.c_int)), B) == 0
    got = _spline(ref, pr, H)
    ref.close()
    return got


def _scores(mr, mf, worst):
    from mujoco_mpc_b200.engine import host_ensemble_score
    B, K, N = mr.shape
    s, f = np.zeros((B, N), np.float32), np.zeros((B, N), np.uint8)
    for b in range(B):
        for i in range(N):
            s[b, i], f[b, i] = host_ensemble_score(mr[b, :, i], mf[b, :, i], worst)
    return s, f


def _check_scores(got, mr, mf, worst):
    s, f = _scores(mr, mf, worst)
    assert got["returns"].tobytes() == s.tobytes()
    np.testing.assert_array_equal(got["failure"], f)
    np.testing.assert_array_equal(got["order"], np.argsort(s, axis=1, kind="stable"))


# ------------------------------------------------------------------------------------------ 1. members are variants
@pytest.mark.parametrize("name,shape,K,B", [("quadruped", "wide", 4, 1), ("quadruped", "wide", 4, 3),
                                            ("quadruped", "plain", 4, 3), ("quadruped", "generic", 4, 3),
                                            ("humanoid_track", "wide", 2, 3)])
def test_members_are_bitwise_variants(name, shape, K, B, monkeypatch):
    _set_shape(shape, monkeypatch)
    base, V = get_model(name), _variants(name)[:K]
    N, H = 4, 12
    pr = _problems_of(_problems(base, N, H, B=3), B)
    e = _engine(base, B * N, H)
    e.set_model_ensemble(V, worst=K)
    got = _spline(e, pr, H)
    mr, mf = e.fetch_ensemble()
    assert mr.shape == (B, K, N)
    for k in range(K):
        ref = _on_variant(name, base, V, pr, N, H, k, B)
        np.testing.assert_array_equal(mr[:, k], ref["returns"], err_msg=f"member {k} returns")
        np.testing.assert_array_equal(mf[:, k], ref["failure"], err_msg=f"member {k} failure")
        for c in range(B * N):
            member = e.fetch_trajectory_member(c, k)
            _assert_equal(member, {f: ref[f][c] for f in member}, f"{name} {shape} member {k} candidate {c}")
            if k == 0:
                _assert_equal({f: got[f][c] for f in member}, member, f"fetch_all = member 0, candidate {c}")
                _assert_equal(e.fetch_trajectory(c), member, f"fetch_trajectory = member 0, candidate {c}")
    _check_scores(got, mr, mf, K)
    assert len({float(mr[0, k, 0]) for k in range(K)}) == K   # the members do differ
    e.close()


# ------------------------------------------------------------------------------------------ 2. score and order
def _diverging_variant():
    """the Quadruped with an actuator gain so large that any non-zero control diverges within the horizon"""
    return _variant("quadruped", lambda x: _sub(x, 'gainprm="40"', 'gainprm="4e9"'))


@pytest.mark.parametrize("worst", [1, 2, 4])
def test_scores_and_order_are_the_host_definition(worst):
    base = get_model("quadruped")
    V = _variants("quadruped")[:3] + [_diverging_variant()]
    B, N, H = 3, 5, 12
    pr = _problems(base, N, H, B=B)
    e = _engine(base, B * N, H)
    e.set_model_ensemble(V, worst=worst)
    got = _spline(e, pr, H)
    mr, mf = e.fetch_ensemble()
    _check_scores(got, mr, mf, worst)
    # the diverging member fails the noisy candidates but not the nominal (zero knots), and only its failures fail
    assert mf[:, 3].any() and not mf[:, 3].all(), mf[:, 3]
    np.testing.assert_array_equal(got["failure"], mf.any(axis=1).astype(np.uint8))
    assert (got["returns"][got["failure"] == 1] == np.float32(1.0e6)).all()
    e.close()


def test_resident_launch_scores_as_the_batched_call():
    base, V = get_model("quadruped"), _variants("quadruped")
    N, H = 6, 12
    pr = _problems(base, N, H, B=1)
    e = _engine(base, N, H)
    e.set_model_ensemble(V, worst=2)
    ret, fail, order = e.rollout_spline(pr["states"][0], pr["times"][0], pr["mocaps"][0], pr["knots"][0],
                                        pr["knot_times"][0], 2, H)
    e.upload_spline_inputs(pr["states"][0], pr["times"][0], pr["mocaps"][0], pr["knots"][0], pr["knot_times"][0], 2, H)
    e.launch_resident()
    e.sync()
    r2, f2, o2 = e.read_returns()
    assert ret.tobytes() == r2.tobytes()
    np.testing.assert_array_equal(fail, f2); np.testing.assert_array_equal(order, o2)
    mr, mf = e.fetch_ensemble()
    _check_scores(dict(returns=ret[None], failure=fail[None], order=order[None]), mr, mf, 2)
    assert e.fetch_stats().shape == (4 * N, 12)
    e.close()


# ------------------------------------------------------------------------------------------ 3. no-op and clearing
def test_one_own_member_changes_nothing_and_clearing_gives_a_fresh_handle():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 3, 4, 12
    pr = _problems(base, N, H, B=B)
    fresh = _engine(base, B * N, H)
    want = _spline(fresh, pr, H)
    e = _engine(base, B * N, H)
    e.set_model_ensemble([base], worst=1)
    _assert_equal(_spline(e, pr, H), want, "K = 1, the handle's own model")
    e.set_model_ensemble(V, worst=3)
    _spline(e, pr, H)
    e.set_model_ensemble(None)
    _assert_equal(_spline(e, pr, H), want, "cleared")
    with pytest.raises(Exception, match="not a model-ensemble launch"):
        e.fetch_ensemble()
    fresh.close(); e.close()


def test_set_task_moves_every_member():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 2, 4, 12
    pr = _problems(base, N, H, B=B)
    w = np.asarray(base.task_weight, float) * 1.7
    e = _engine(base, B * N, H)
    e.set_model_ensemble(V, worst=4)
    e.set_task(weight=w)
    _spline_handle_task(e, pr, H)
    mr, _ = e.fetch_ensemble()
    for k in range(4):
        s = _engine(V[k], B * N, H)
        s.set_task(weight=w)
        np.testing.assert_array_equal(mr[:, k], _spline_handle_task(s, pr, H)["returns"], err_msg=f"member {k}")
        s.close()
    e.close()


def test_a_launch_at_full_capacity_is_accepted():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 4, 8, 16
    pr = _problems(base, N, H, B=B)
    e = _engine(base, B * N, H)                 # max_candidates = B N: the ensemble launches 4 B N trajectories
    want = _spline(e, pr, H)
    e.set_model_ensemble(V, worst=4)
    got = _spline(e, pr, H)
    mr, mf = e.fetch_ensemble()
    _check_scores(got, mr, mf, 4)
    e.set_model_ensemble(None)
    _assert_equal(_spline(e, pr, H), want, "after the ensemble, at capacity")
    e.close()


# ------------------------------------------------------------------------------------------ 4. refusals
def test_refusals_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import EngineError
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 2, 4, 12
    pr = _problems(base, N, H, B=B)
    e, ref = _engine(base, B * N, H), _engine(base, B * N, H)
    ref.set_model_ensemble(V, worst=2)
    want = _spline(ref, pr, H)
    plain = _spline(e, pr, H)
    for K, worst in ((-1, 1), (33, 1), (4, 0), (4, 5)):
        models = (V * 9)[:max(K, 0)] if K > 0 else V
        rc = e.lib.mjpc_b200_set_model_ensemble(e.h, None if K < 0 else _blobs(models)[1], K, worst)
        assert rc == BAD_ARGUMENT, (K, worst)
        _assert_equal(_spline(e, pr, H), plain, f"after K = {K}, worst = {worst}")
    for what, v in _refusal_variants().items():
        with pytest.raises(EngineError, match=r"set_model_ensemble: member 2: .* differs from the handle's model"):
            e.set_model_ensemble(V[:2] + [v] + V[3:], worst=2)
        _assert_equal(_spline(e, pr, H), plain, f"after refusing {what}")
    e.set_model_variants(V[:B])
    with pytest.raises(EngineError, match="error -5: set_model_ensemble: not available while model variants are set"):
        e.set_model_ensemble(V, worst=2)
    e.set_model_variants(None)
    e.set_model_ensemble(V, worst=2)
    with pytest.raises(EngineError, match="error -5: set_model_variants: not available while a model ensemble is set"):
        e.set_model_variants(V[:B])
    x = np.tile(pr["states"][0], (H, 1)).astype(np.float32)
    u = np.zeros((H, base.nu), np.float32)
    t = np.arange(H) * 0.01
    mc = pr["mocaps"][0]
    fb = (x[None].repeat(B, 0), u[None].repeat(B, 0), t[None].repeat(B, 0))
    calls = {
        "rollout_feedback": lambda: e.rollout_feedback(pr["states"][0], 0.0, mc, u, x, t, np.zeros((H, base.nu, 2 * base.nv)),
                                                       None, np.ones(2), 1),
        "rollout_feedback_batched": lambda: e.rollout_feedback_batched(
            pr["states"], pr["times"], pr["mocaps"], fb[1], fb[0], fb[2], np.zeros((B, H, base.nu, 2 * base.nv)), None,
            np.ones((B, 2)), 1),
        "model_derivatives": lambda: e.model_derivatives(x, u, t, mc, 3e-4),
        "model_derivatives_batched": lambda: e.model_derivatives_batched(fb[0], fb[1], fb[2], pr["mocaps"], 3e-4, 0, 1),
        "gradient_batched": lambda: e.gradient_batched(fb[0], fb[1], fb[2], pr["mocaps"],
                                                       np.zeros((B, H, e.nr), np.float32),
                                                       3e-4, 0, 1),
        "rollout_spline_sharded": lambda: e.rollout_spline_sharded(pr["states"][0], 0.0, mc, pr["knots"][0],
                                                                   pr["knot_times"][0], 2, H),
        "step_debug": lambda: e.step_debug(x[0, :base.nq], x[0, base.nq:], u[0], mc),
        "step_batch": lambda: e.step_batch(x[:2, :base.nq], x[:2, base.nq:], u[:2], mc, np.zeros(2)),
        "step_sensors": lambda: e.step_sensors(x[:2], u[0], mc, 0.0, 0, 1),
        "plant_init": lambda: e._check(e.lib.mjpc_b200_plant_init(e.h, 2, 0, 0)),
    }
    for name, call in calls.items():
        with pytest.raises(EngineError, match=f"error -5: {name}: not available while a model ensemble is set"):
            call()
        _assert_equal(_spline(e, pr, H), want, f"after refusing {name}")
    e.set_xfrc_noise(0.5, 0.1, 3)
    with pytest.raises(EngineError, match="error -5: rollout_spline: force noise"):
        _spline(e, pr, H)
    e.set_xfrc_noise(0.0)
    _assert_equal(_spline(e, pr, H), want, "after the noise refusal")
    e.close(); ref.close()


def _blobs(models):
    from mujoco_mpc_b200.engine import _model_blobs
    bufs, arr, n = _model_blobs(models)
    _blobs.keep = bufs
    return n, arr


# ------------------------------------------------------------------------------------------ 5. planners
def _planners(kind, m, N, H, seed, B=None, seeds=None):
    from mujoco_mpc_b200 import engine as E
    kw = dict(num_gradient=4, gradient_filter=0.6) if kind == "sg" else {}
    if B is None:
        cls = {"sampling": E.CppSamplingPlanner, "ce": E.CppCrossEntropyPlanner, "sg": E.CppSampleGradientPlanner}[kind]
        return cls(m, N, H, seed=seed, **kw)
    cls = {"sampling": E.CppBatchSamplingPlanner, "ce": E.CppBatchCrossEntropyPlanner,
           "sg": E.CppBatchSampleGradientPlanner}[kind]
    return cls(m, B, N, H, seeds=seeds, **kw)


def _drive(singles, pr, it, batch=None):
    B = len(singles)
    out = []
    for b in range(B):
        t = pr["times"][b] + 0.01 * it
        singles[b].set_state(pr["states"][b], t, pr["mocaps"][b])
        if batch is not None:
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
    return out


@pytest.mark.parametrize("kind", ["sampling", "ce", "sg"])
def test_one_own_member_planner_is_the_plain_planner(kind):
    base = get_model("quadruped")
    N, H = 8, 16
    pr = _problems(base, 4, H, B=1)
    a, b = _planners(kind, base, N, H, SEEDS[0]), _planners(kind, base, N, H, SEEDS[0])
    a.set_ensemble([base], worst=1)
    for p in (a, b):
        p.reset()
    for it in range(5):
        _drive([a], pr, it); _drive([b], pr, it)
        _assert_equal(a.optimize_policy(), b.optimize_policy(), f"{kind} iteration {it}")
        for dt in (0.0, 0.013, 0.05):
            t = pr["times"][0] + 0.01 * it + dt
            np.testing.assert_array_equal(a.action_from_policy(t), b.action_from_policy(t))
    a.close(); b.close()


@pytest.mark.parametrize("kind", ["sampling", "ce", "sg"])
def test_batch_with_an_ensemble_is_single_planners_with_it(kind):
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H, iters = 3, 8, 16, 3
    pr = _problems(base, 4, H, B=B)
    seeds = SEEDS[:B]
    batch = _planners(kind, base, N, H, None, B=B, seeds=seeds)
    singles = [_planners(kind, base, N, H, seeds[b]) for b in range(B)]
    batch.set_ensemble(V, worst=2)
    for s in singles:
        s.set_ensemble(V, worst=2)
    for b in range(B):
        batch.reset(b); singles[b].reset()
        task = dict(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])
        batch.set_task(b, **task); singles[b].set_task(**task)
    plain = _planners(kind, base, N, H, seeds[0])   # the same problem 0 without the ensemble plans differently
    plain.reset()
    plain.set_task(weight=pr["weights"][0], parameters=pr["parameters"][0], task_state=pr["task_states"][0])
    differs = False
    for it in range(iters):
        _drive(singles, pr, it, batch)
        _drive([plain], pr, it)
        got = batch.optimize_policy()
        for b in range(B):
            ref = singles[b].optimize_policy()
            _assert_equal(got[b], ref, f"{kind} iteration {it} problem {b}")
            for dt in (0.0, 0.013, 0.05):
                t = pr["times"][b] + 0.01 * it + dt
                np.testing.assert_array_equal(batch.action_from_policy(b, t), singles[b].action_from_policy(t))
        differs |= not np.array_equal(plain.optimize_policy()["returns"], got[0]["returns"])
    assert differs
    batch.close(); plain.close()
    for s in singles:
        s.close()


def test_the_other_kinds_refuse_an_ensemble():
    from mujoco_mpc_b200 import engine as E
    base, V = get_model("quadruped"), _variants("quadruped")[:2]
    H = 16
    singles = [E.CppRobustPlanner(base, 10, H, ncandidates=2, nrepetitions=2), E.CppGradientPlanner(base, H),
               E.CppILQGPlanner(base, H, num_rollouts=4), E.CppILQSPlanner(base, H)]
    batches = [E.CppBatchRobustPlanner(base, 2, 10, H, ncandidates=2, nrepetitions=2), E.CppBatchGradientPlanner(base, 2, H),
               E.CppBatchILQGPlanner(base, 2, H, num_rollouts=4), E.CppBatchILQSPlanner(base, 2, H)]
    for p in singles + batches:
        with pytest.raises(E.EngineError, match=r"\(-5\)"):
            p.set_ensemble(V, worst=1)
        p.close()
