"""GPU: initial-state ensembles (mjpc_b200_rollout_spline_belief_batched and the planners' set_state_ensemble).

The device's member states must be the host twin (mjpc_b200_host_state_member) rounded to float; each member's
trajectory must be BITWISE a plain rollout_spline_batched launch from that member's state, and each candidate's score
bitwise the host definition of the ensemble score over the member returns.  A zero covariance gives the plain launch's
returns, a problem does not depend on the others, member rows follow their problem's variant, and every refusal leaves
the handle usable.  The planners with a state ensemble are bitwise their batches, and a closed loop with a Kalman bank,
measurement noise and a state-ensemble batch planner is bitwise loops of one."""
import ctypes as C

import numpy as np
import pytest

from conftest import get_model
from test_gpu_batched import _problems
from test_gpu_model_ensemble import _check_scores, _planners
from test_gpu_model_variants import SEEDS, _assert_equal, _engine, _spline, _variants

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, CAPACITY, UNSUPPORTED = -1, -3, -5


def _covs(m, B, scale=1e-3, seed=0):
    """B symmetric positive definite covariances [B][2 nv][2 nv], correlated, different per problem"""
    rng = np.random.default_rng(seed)
    n = 2 * m.nv
    out = []
    for b in range(B):
        A = rng.standard_normal((n, n))
        out.append(scale * (1 + b) * (A @ A.T / n + 0.2 * np.eye(n)))
    return np.stack(out)


def _belief(e, pr, covs, H, K, worst, seed=9, iteration=3, sl=slice(None)):
    a = {k: v[sl] for k, v in pr.items()}
    ret, fail, order = e.rollout_spline_belief_batched(a["states"], covs[sl], a["times"], a["mocaps"], a["knots"],
                                                       a["knot_times"], 2, H, K, worst, seed, iteration,
                                                       weights=a["weights"], parameters=a["parameters"],
                                                       task_states=a["task_states"])
    return dict(returns=ret, failure=fail, order=order)


def _member_states(e, B, K, N):
    """[B][K][nq + nv]: row 0 of each member's trajectory of candidate 0, the state the member started from"""
    return np.array([[e.fetch_trajectory_member(b * N, k)["states"][0] for k in range(K)] for b in range(B)])


def _replicated(pr, K, states):
    """pr with problem b repeated K times, row b K + k starting from states[b][k]"""
    out = {k: np.repeat(np.asarray(v), K, axis=0) for k, v in pr.items()}
    out["states"] = states.reshape(-1, states.shape[-1])
    return out


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


# ------------------------------------------------------------------------------------------ 1. members
@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_members_are_the_host_twin_and_roll_out_as_plain_launches(name):
    from mujoco_mpc_b200.engine import host_state_member
    m = get_model(name)
    B, K, N, H, worst = 3, 4, 4, 16, 2
    pr = _problems(m, N, H, B=B)
    covs = _covs(m, B)
    e = _engine(m, B * K * N, H)
    got = _belief(e, pr, covs, H, K, worst)
    dev = _member_states(e, B, K, N)
    worst_ulps = 0
    for b in range(B):
        mean = np.asarray(pr["states"][b], np.float32)
        assert dev[b, 0].tobytes() == mean.tobytes(), f"{name}: member 0 of problem {b} is the mean"
        for k in range(1, K):
            host = host_state_member(m, mean.astype(float), covs[b], 9, 3, b, k)
            u = _ulps(dev[b, k], host.astype(np.float32))
            worst_ulps = max(worst_ulps, int(u.max()))
            assert not np.array_equal(dev[b, k], mean)
    print(f"{name}: largest difference of a device member state from the host twin: {worst_ulps} ulp")
    assert worst_ulps <= 1
    mr, mf = e.fetch_ensemble()
    _check_scores(got, mr, mf, worst)
    # each member's trajectories: a plain launch of B K problems from the member states
    members = {k: [e.fetch_trajectory_member(c, k) for c in range(B * N)] for k in range(K)}
    ref = _engine(m, B * K * N, H)
    plain = _spline(ref, _replicated(pr, K, dev), H)
    np.testing.assert_array_equal(mr.reshape(B * K, N), plain["returns"])
    for b in range(B):
        for k in range(K):
            for i in range(N):
                row = (b * K + k) * N + i
                for f in ("states", "actions", "times", "residual", "costs", "trace"):
                    np.testing.assert_array_equal(members[k][b * N + i][f], plain[f][row],
                                                  err_msg=f"{name} problem {b} member {k} candidate {i} {f}")
    e.close(); ref.close()


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_zero_covariance_gives_the_plain_launch(name):
    m = get_model(name)
    B, K, N, H = 2, 4, 8, 16
    pr = _problems(m, N, H, B=B)
    e = _engine(m, B * K * N, H)
    for worst in (1, K):
        got = _belief(e, pr, np.zeros((B, 2 * m.nv, 2 * m.nv)), H, K, worst)
        ref = _spline(e, pr, H)
        assert got["returns"].tobytes() == ref["returns"].tobytes()
        np.testing.assert_array_equal(got["failure"], ref["failure"])
        np.testing.assert_array_equal(got["order"], ref["order"])
    e.close()


def test_a_problem_does_not_depend_on_the_others():
    m = get_model("quadruped")
    B, K, N, H = 3, 4, 4, 16
    pr = _problems(m, N, H, B=B)
    covs = _covs(m, B)
    e = _engine(m, B * K * N, H)
    full = _belief(e, pr, covs, H, K, 2, seed=20)
    mr, _ = e.fetch_ensemble()
    # problem 1 alone draws with key seed + 1
    alone = _belief(e, pr, covs, H, K, 2, seed=21, sl=slice(1, 2))
    ar, _ = e.fetch_ensemble()
    assert alone["returns"].tobytes() == full["returns"][1:2].tobytes()
    assert ar.tobytes() == mr[1:2].tobytes()
    # other problems changed: problems 1 and 2 are the same
    pr2 = {k: np.array(v, copy=True) for k, v in pr.items()}
    pr2["states"][0, m.nq:] += 0.3
    covs2 = covs.copy()
    covs2[0] *= 4.0
    other = _belief(e, pr2, covs2, H, K, 2, seed=20)
    r2, _ = e.fetch_ensemble()
    assert other["returns"][1:].tobytes() == full["returns"][1:].tobytes()
    assert r2[1:].tobytes() == mr[1:].tobytes()
    assert other["returns"][0].tobytes() != full["returns"][0].tobytes()
    e.close()


def test_member_rows_follow_their_problems_variant():
    base, V = get_model("quadruped"), _variants("quadruped")
    B, K, N, H = 3, 2, 4, 16
    pr = _problems(base, N, H, B=B)
    covs = _covs(base, B)
    e = _engine(base, B * K * N, H)
    e.set_model_variants(V[:B])
    got = _belief(e, pr, covs, H, K, K)
    mr, mf = e.fetch_ensemble()
    _check_scores(got, mr, mf, K)
    dev = _member_states(e, B, K, N)
    ref = _engine(base, B * K * N, H)
    ref.set_model_variants(V[:B])
    idx = np.repeat(np.arange(B, dtype=np.int32), K)
    assert ref.lib.mjpc_b200_select_model_variants(ref.h, idx.ctypes.data_as(C.POINTER(C.c_int)), B * K) == 0
    plain = _spline(ref, _replicated(pr, K, dev), H)
    np.testing.assert_array_equal(mr.reshape(B * K, N), plain["returns"])
    # and not the base model's
    other = _engine(base, B * K * N, H)
    assert not np.array_equal(_spline(other, _replicated(pr, K, dev), H)["returns"], plain["returns"])
    e.close(); ref.close(); other.close()


# ------------------------------------------------------------------------------------------ 2. refusals
def test_refusals_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import EngineError
    m, V = get_model("quadruped"), _variants("quadruped")
    B, K, N, H = 2, 4, 4, 16
    pr = _problems(m, N, H, B=B)
    covs = _covs(m, B)
    e = _engine(m, B * K * N, H)
    fresh = _engine(m, B * K * N, H)
    want = _belief(fresh, pr, covs, H, K, 2)
    want_plain = _spline(fresh, pr, H)

    def usable(what):
        np.testing.assert_array_equal(_spline(e, pr, H)["returns"], want_plain["returns"], err_msg=what)
        assert _belief(e, pr, covs, H, K, 2)["returns"].tobytes() == want["returns"].tobytes(), what

    def refused(code, match, **kw):
        a = dict(K=K, worst=2, covs=covs)
        a.update(kw)
        with pytest.raises(EngineError, match=match) as ex:
            _belief(e, pr, a["covs"], H, a["K"], a["worst"])
        assert f"error {code}" in str(ex.value), str(ex.value)
        usable(match)

    usable("before")
    refused(BAD_ARGUMENT, "K must be", K=0)
    refused(BAD_ARGUMENT, "K must be", K=33)
    refused(BAD_ARGUMENT, "worst must be", worst=0)
    refused(BAD_ARGUMENT, "worst must be", worst=K + 1)
    small = _engine(m, B * N - 1, H)
    with pytest.raises(EngineError, match="B\\*N/H/P above capacity") as ex:
        _belief(small, pr, covs, H, K, 2)
    assert f"error {CAPACITY}" in str(ex.value)
    np.testing.assert_array_equal(_spline(small, pr, H, sl=slice(0, 1))["returns"], want_plain["returns"][:1])
    small.close()
    bad = covs.copy()
    bad[1, 3, 2] = np.inf
    refused(BAD_ARGUMENT, "problem 1: non-finite", covs=bad)
    notpsd = covs.copy()
    notpsd[1, 5, 5] = -1.0
    refused(BAD_ARGUMENT, "problem 1: the covariance is not positive semi-definite", covs=notpsd)
    e.set_model_ensemble(V[:2])
    with pytest.raises(EngineError, match="rollout_spline_belief_batched: not available while a model ensemble"):
        _belief(e, pr, covs, H, K, 2)
    e.set_model_ensemble(None)
    usable("after the model ensemble")
    e.set_xfrc_noise(0.5, 0.1, 3)
    with pytest.raises(EngineError, match="force noise") as ex:
        _belief(e, pr, covs, H, K, 2)
    assert f"error {UNSUPPORTED}" in str(ex.value)
    e.set_xfrc_noise(0.0, 1.0, 0)
    usable("after force noise")
    e.close(); fresh.close()


# ------------------------------------------------------------------------------------------ 3. planners
def _drive(ps, pr, it, covs=None, batch=None):
    for b, p in enumerate(ps):
        t = pr["times"][b] + 0.01 * it
        p.set_state(pr["states"][b], t, pr["mocaps"][b])
        if covs is not None:
            p.set_state_covariance(covs[b])
        if batch is not None:
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
            if covs is not None:
                batch.set_state_covariance(b, covs[b])


@pytest.mark.parametrize("kind", ["sampling", "ce", "sg"])
def test_a_planner_without_a_covariance_is_the_plain_planner(kind):
    base = get_model("quadruped")
    N, H = 8, 16
    pr = _problems(base, N, H, B=1)
    a, b = _planners(kind, base, N, H, SEEDS[0]), _planners(kind, base, N, H, SEEDS[0])
    a.set_state_ensemble(4, worst=1, seed=5)
    for p in (a, b):
        p.reset()
    for it in range(4):
        _drive([a], pr, it); _drive([b], pr, it)
        _assert_equal(a.optimize_policy(), b.optimize_policy(), f"{kind} iteration {it}")
        t = pr["times"][0] + 0.01 * it + 0.013
        np.testing.assert_array_equal(a.action_from_policy(t), b.action_from_policy(t))
    a.close(); b.close()


@pytest.mark.parametrize("kind", ["sampling", "ce", "sg"])
def test_batch_with_a_state_ensemble_is_single_planners_with_it(kind):
    base = get_model("quadruped")
    B, N, H, iters, K = 3, 8, 16, 3, 4
    pr = _problems(base, N, H, B=B)
    covs = _covs(base, B, scale=3e-3)
    seeds = SEEDS[:B]
    batch = _planners(kind, base, N, H, None, B=B, seeds=seeds)
    singles = [_planners(kind, base, N, H, seeds[b]) for b in range(B)]
    batch.set_state_ensemble(K, worst=2, seed=40)
    for b, s in enumerate(singles):
        s.set_state_ensemble(K, worst=2, seed=40 + b)   # problem b of the batch draws with key seed + b
    for b in range(B):
        batch.reset(b); singles[b].reset()
        task = dict(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])
        batch.set_task(b, **task); singles[b].set_task(**task)
    plain = _planners(kind, base, N, H, seeds[0])
    plain.reset()
    plain.set_task(weight=pr["weights"][0], parameters=pr["parameters"][0], task_state=pr["task_states"][0])
    differs = False
    for it in range(iters):
        _drive(singles, pr, it, covs, batch)
        _drive([plain], pr, it)
        got = batch.optimize_policy()
        for b in range(B):
            _assert_equal(got[b], singles[b].optimize_policy(), f"{kind} iteration {it} problem {b}")
            t = pr["times"][b] + 0.01 * it + 0.013
            np.testing.assert_array_equal(batch.action_from_policy(b, t), singles[b].action_from_policy(t))
        differs |= not np.array_equal(plain.optimize_policy()["returns"], got[0]["returns"])
    assert differs
    batch.close(); plain.close()
    for s in singles:
        s.close()


def test_state_and_model_ensembles_exclude_each_other_and_the_other_kinds_refuse():
    from mujoco_mpc_b200 import engine as E
    base, V = get_model("quadruped"), _variants("quadruped")[:2]
    H = 16
    for p in (_planners("sampling", base, 8, H, 1), _planners("ce", base, 8, H, None, B=2, seeds=[1, 2])):
        p.set_state_ensemble(2, worst=1)
        with pytest.raises(E.EngineError, match=r"\(-5\)"):
            p.set_ensemble(V, worst=1)
        p.set_state_ensemble(0)
        p.set_ensemble(V, worst=1)
        with pytest.raises(E.EngineError, match=r"\(-5\)"):
            p.set_state_ensemble(2, worst=1)
        for K, worst in ((33, 1), (2, 3), (2, 0)):
            with pytest.raises(E.EngineError, match=r"\((-1|-5)\)"):
                p.set_state_ensemble(K, worst=worst)
        p.close()
    singles = [E.CppRobustPlanner(base, 10, H, ncandidates=2, nrepetitions=2), E.CppGradientPlanner(base, H),
               E.CppILQGPlanner(base, H, num_rollouts=4), E.CppILQSPlanner(base, H)]
    batches = [E.CppBatchRobustPlanner(base, 2, 10, H, ncandidates=2, nrepetitions=2), E.CppBatchGradientPlanner(base, 2, H),
               E.CppBatchILQGPlanner(base, 2, H, num_rollouts=4), E.CppBatchILQSPlanner(base, 2, H)]
    for p in singles + batches:
        with pytest.raises(E.EngineError, match=r"\(-5\)"):
            p.set_state_ensemble(2, worst=1)
        with pytest.raises(E.EngineError, match=r"\(-5\)"):
            if p in singles:
                p.set_state_covariance(np.eye(2 * base.nv))
            else:
                p.set_state_covariance(0, np.eye(2 * base.nv))
        p.close()


# ------------------------------------------------------------------------------------------ 4. the closed loop
def test_closed_loop_with_measurement_noise_and_a_state_ensemble_is_loops_of_one():
    from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
    from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, CppPlantBank
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    from test_gpu_plant import _mocap, _start
    m = get_model("quadruped")
    B, steps, N, H, K = 2, 24, 16, 16, 4
    starts, mc = _start(m, B), _mocap(m)

    def run(plants):
        n = len(plants)
        pl = CppBatchSamplingPlanner(m, n, N, H, seeds=[70 + b for b in plants])
        pl.set_state_ensemble(K, worst=K, seed=90 + plants[0])
        est = CppBatchEstimator(m, "kalman", n, timestep=m.opt_timestep)
        bank = CppPlantBank(m, n, sensor_start=est.sensor_start, nsensor=est.nsensor)
        for j, b in enumerate(plants):
            q, v = starts[b]
            pl.reset(j)
            bank.reset(j, q, v, 0.0, mc)
            bank.set_disturbance(j, seed=60 + b)
            bank.set_sensor_noise(j, 0.01)
            est.reset(j, state=np.concatenate([q, v]).astype(float), time=0.0)
        out = synchronous_planning_cost(pl, bank, steps, 2, estimator=est)
        est_states = np.array([est.state(j) for j in range(n)])
        pl.close(); bank.close(); est.close()
        return out, est_states

    both, both_est = run([0, 1])
    for b in range(B):
        one, one_est = run([b])
        np.testing.assert_array_equal(both["states"][:, b], one["states"][:, 0], err_msg=f"plant {b} states")
        np.testing.assert_array_equal(both["costs"][:, b], one["costs"][:, 0], err_msg=f"plant {b} costs")
        np.testing.assert_array_equal(both_est[b], one_est[0], err_msg=f"plant {b} estimate")
    assert np.all(both["final_status"] == 0)
