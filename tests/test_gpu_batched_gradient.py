"""GPU: the device gradient sweep (mjpc_b200_gradient_batched) and the batched Gradient and iLQS planners.  The sweep's
reference is the host GradientSweep (mjpc_b200_host_gradient_sweep) on the A, B, cx and cu the two existing batched
derivative calls return for the same inputs; a batch's reference is one single planner of its kind per problem.  All
must be BITWISE equal."""
import ctypes as C

import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_batched_ilqg import _problems

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, CAPACITY, UNSUPPORTED = -1, -3, -5


def _task(pr, B):
    return dict(weights=pr["weights"][:B], parameters=pr["parameters"][:B], task_states=pr["task_states"][:B])


def _inputs(pr, B):
    return pr["x"][:B], pr["u"][:B], pr["t"][:B], pr["mocaps"][:B], pr["residual"][:B]


@pytest.mark.parametrize("name,shape", [("quadruped", "helper"), ("quadruped", "plain"), ("quadruped", "generic"),
                                        ("humanoid", "helper")])
@pytest.mark.parametrize("B", [3, 1])
@pytest.mark.parametrize("mode,skip", [(0, 0), (1, 0), (0, 2), (1, 2)])
def test_gradient_batched_equals_host_sweep(name, shape, B, mode, skip, monkeypatch):
    from mujoco_mpc_b200.engine import Engine, host_gradient_sweep
    if shape == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    elif shape == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model(name)
    H = 16
    pr = _problems(m, H, B=3)
    x, u, t, mc, res = _inputs(pr, B)
    e = Engine(m, 8, H)
    A, Bm, Cm, D = e.model_derivatives_batched(x, u, t, mc, 1e-3, skip=skip, mode=mode, **_task(pr, B))
    cx, cu, _, _, _ = e.cost_derivatives_batched(res, Cm, D, weights=pr["weights"][:B])
    n0 = e.launch_count
    k, dV0 = e.gradient_batched(x, u, t, mc, res, 1e-3, skip=skip, mode=mode, **_task(pr, B))
    assert e.launch_count - n0 == (2 if skip == 0 else 3) + 2      # fd_center, fd_column[, fd_interp], cost, sweep
    assert e.last_kernel_ms > 0
    for b in range(B):
        k_ref, dV0_ref = host_gradient_sweep(A[b], Bm[b], cx[b], cu[b])
        np.testing.assert_array_equal(k[b], k_ref, err_msg=f"problem {b}")
        assert dV0[b] == dV0_ref, (b, dV0[b], dV0_ref)
        assert np.abs(k[b]).max() > 0
    if B > 1:
        assert np.abs(k[0] - k[1]).max() > 0                          # the problems do differ
    e.close()


def test_gradient_batched_argument_errors_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import Engine, EngineError
    m = get_model("quadruped")
    H = 16
    pr = _problems(m, H, B=3)
    x, u, t, mc, res = _inputs(pr, 3)
    e = Engine(m, 8, H)
    ref = e.gradient_batched(x, u, t, mc, res, 1e-3, **_task(pr, 3))
    bad = [
        dict(args=(x[:0], u[:0], t[:0], mc[:0], res[:0], 1e-3)),                     # B = 0
        dict(args=(x[:, :1], u[:, :1], t[:, :1], mc, res[:, :1], 1e-3)),            # H = 1
        dict(args=(x, u, t, mc, None, 1e-3)),                                          # NULL residual
        dict(args=(x, u, t, mc, res, 0.0)),                                            # tol
        dict(args=(x, u, t, mc, res, 1e-3), mode=2),
        dict(args=(x, u, t, mc, res, 1e-3), skip=-1),
    ]
    assert m.nmocap > 0
    bad.append(dict(args=(x, u, t, None, res, 1e-3)))                                # missing mocaps
    for case in bad:
        kw = {k: v for k, v in case.items() if k != "args"}
        with pytest.raises(EngineError, match=f"error {BAD_ARGUMENT}"):
            e.gradient_batched(*case["args"], **kw)
    long = [np.concatenate([a, a[:, -1:]], 1) for a in (x, u, res)]
    tl = np.concatenate([t, t[:, -1:] + 0.01], 1)
    with pytest.raises(EngineError, match=f"error {CAPACITY}"):                       # H > max_horizon
        e.gradient_batched(long[0], long[1], tl, mc, long[2], 1e-3)
    again = e.gradient_batched(x, u, t, mc, res, 1e-3, **_task(pr, 3))
    for a, b in zip(ref, again):
        np.testing.assert_array_equal(a, b)
    e.close()


KW = dict(num_trajectory=8, num_spline_points=5, representation=1, fd_tolerance=1e-3, fd_mode=1)


def _batch(m, B, H, pr):
    from mujoco_mpc_b200.engine import CppBatchGradientPlanner
    batch = CppBatchGradientPlanner(m, B, H, **KW)
    for b in range(B):
        batch.reset(b)
        batch.set_task(b, pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    return batch


def _state(pr, b, it):
    return pr["states"][b], pr["times"][b] + 0.01 * it, pr["mocaps"][b]


@pytest.mark.parametrize("B", [3, 1])
def test_batch_gradient_planner_equals_independent_planners(B):
    m = get_model("quadruped")
    H = 32
    pr = _problems(m, H, B=3)
    from mujoco_mpc_b200.engine import CppGradientPlanner
    batch = _batch(m, B, H, pr)
    singles = [CppGradientPlanner(m, H, **KW) for _ in range(B)]
    for b in range(B):
        singles[b].reset()
        singles[b].set_task(pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    improved = 0
    for it in range(6):
        for b in range(B):
            batch.set_state(b, *_state(pr, b, it)); singles[b].set_state(*_state(pr, b, it))
        codes = batch.optimize_policy()
        for b in range(B):
            ok = singles[b].optimize_policy()
            assert codes[b] == ok, (it, b)
            improved += ok
            r, s = batch.result(b), singles[b].result()
            for key in s:
                np.testing.assert_array_equal(r[key], s[key], err_msg=f"iteration {it} problem {b}: {key}")
            t0 = pr["times"][b] + 0.01 * it
            for dt in (0.0, 0.013, 0.1, 0.29):
                for prev in (False, True):
                    np.testing.assert_array_equal(batch.action_from_policy(b, t0 + dt, prev),
                                                  singles[b].action_from_policy(t0 + dt, prev))
    assert improved > 0
    batch.close()
    for s in singles:
        s.close()


def test_batch_gradient_problems_are_independent():
    m = get_model("quadruped")
    H = 32
    pr = _problems(m, H, B=3)
    ch = {k: np.array(v, copy=True) for k, v in pr.items()}
    ch["states"][1, m.nq:] += 0.2
    ch["times"][1] += 0.07
    ch["weights"][1] *= 2.0
    ch["task_states"][1, 1] -= 0.2

    def run(p):
        batch = _batch(m, 3, H, p)
        out = []
        for it in range(3):
            for b in range(3):
                batch.set_state(b, *_state(p, b, it))
            out.append((batch.optimize_policy(), [batch.result(b) for b in range(3)]))
        batch.close()
        return out

    before, after = run(pr), run(ch)
    assert any(a[1][1]["total_return"] != b[1][1]["total_return"] for a, b in zip(after, before))
    for (ca, ra), (cb, rb) in zip(after, before):
        for b in (0, 2):
            assert ca[b] == cb[b]
            for key in rb[b]:
                np.testing.assert_array_equal(ra[b][key], rb[b][key], err_msg=key)


def test_gradient_ilqs_batch_kind_checks():
    """A Gradient or iLQS batch's own calls refuse a batch of another kind and a problem outside the batch; set_fd
    reaches the derivative-based kinds only."""
    from mujoco_mpc_b200.engine import CppBatchGradientPlanner, CppBatchILQSPlanner, CppBatchSamplingPlanner, load_library
    lib = load_library()
    m = get_model("particle")
    g = CppBatchGradientPlanner(m, 2, 16)
    s = CppBatchSamplingPlanner(m, 2, 8, 16)
    sc, v = (C.c_double * 6)(), (C.c_double * 64)()
    assert lib.mjpc_b200_batch_gradient_planner_get_result(s.h, 0, sc, v, v) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ce_planner_get_result(g.h, 0, *([None] * 6)) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_sampling_planner_get_result(g.h, 0, *([None] * 5)) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ilqg_planner_nominal_trajectory(g.h, 16) == BAD_ARGUMENT
    for p in (-1, 2):
        assert lib.mjpc_b200_batch_gradient_planner_get_result(g.h, p, sc, v, v) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_fd(s.h, C.c_double(1e-3), 0, 0) == UNSUPPORTED
    assert lib.mjpc_b200_batch_planner_set_fd(g.h, C.c_double(1e-3), 0, 0) == 0
    assert lib.mjpc_b200_batch_gradient_planner_get_result(g.h, 1, sc, v, v) == 5   # P
    q = CppBatchILQSPlanner(m, 2, 16)
    a = (C.c_double * 8)()
    for other in (g.h, s.h):
        assert lib.mjpc_b200_batch_ilqs_planner_get_result(other, 0, sc) == BAD_ARGUMENT
        assert lib.mjpc_b200_batch_ilqs_planner_set_exploration(other, C.c_double(0.1)) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_gradient_planner_get_result(q.h, 0, sc, v, v) == BAD_ARGUMENT
    for p in (-1, 2):
        assert lib.mjpc_b200_batch_ilqs_planner_get_result(q.h, p, sc) == BAD_ARGUMENT
        assert lib.mjpc_b200_batch_planner_action_from_policy(q.h, p, a, None, C.c_double(0.0), 0) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_fd(q.h, C.c_double(1e-3), 0, 0) == 0
    assert lib.mjpc_b200_batch_ilqs_planner_get_result(q.h, 1, sc) == 0       # the active policy: sampling
    g.close(); s.close(); q.close()


def test_ilqg_batch_generic_calls_and_kind_checks():
    """The iLQG batch's own calls refuse another kind's handle and leave it whole, the generic calls drive an iLQG
    batch as the Python class does (codes, results and actions with a state), and the sampling batch's get_result
    refuses it."""
    from mujoco_mpc_b200.engine import CppBatchILQGPlanner, CppBatchSamplingPlanner, load_library
    lib = load_library()
    m = get_model("particle")
    H = 16
    dp = C.POINTER(C.c_double)
    x, mc = np.zeros(4), np.ascontiguousarray(mocap_of(m), np.float64)
    xp, mcp = x.ctypes.data_as(dp), mc.ctypes.data_as(dp)
    s = CppBatchSamplingPlanner(m, 2, 8, H)
    sc = (C.c_double * 6)()
    t0 = C.c_double(0.0)
    assert lib.mjpc_b200_batch_ilqg_planner_nominal_trajectory(s.h, H) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ilqg_planner_get_result(s.h, 0, sc, None, None, None) == BAD_ARGUMENT
    for b in range(2):                                                     # the sampling batch is still whole
        s.reset(b); s.set_state(b, x, 0.0, mc)
    assert len(s.optimize_policy()) == 2
    s.close()

    # the same two problems through the C calls (q) and the Python class (ref)
    q = CppBatchILQGPlanner(m, 2, H)
    ref = CppBatchILQGPlanner(m, 2, H, fd_tolerance=1e-3, fd_mode=0, derivative_skip=0)
    assert lib.mjpc_b200_batch_planner_set_fd(q.h, C.c_double(1e-3), 0, 0) == 0
    for b in range(2):
        mb = mc.copy(); mb[:2] = (0.1 * (b + 1), -0.05)
        assert lib.mjpc_b200_batch_planner_reset(q.h, b, H, None) == 0
        assert lib.mjpc_b200_batch_planner_set_state(q.h, b, xp, t0, mb.ctypes.data_as(dp)) == 0
        w = np.asarray(m.task_weight, float) * (1.0 + b)
        assert lib.mjpc_b200_batch_planner_set_task(q.h, b, w.ctypes.data_as(dp), None, None) == 0
        ref.reset(b); ref.set_state(b, x, 0.0, mb); ref.set_task(b, w)
    codes = (C.c_int * 2)()
    for _ in range(3):
        assert lib.mjpc_b200_batch_planner_optimize_policy(q.h, H, codes) == 0
        np.testing.assert_array_equal(np.array(codes), ref.optimize_policy())
    state = np.array([0.05, -0.02, 0.1, 0.0])
    for b in range(2):
        got = (C.c_double * 6)()
        assert lib.mjpc_b200_batch_ilqg_planner_get_result(q.h, b, got, None, None, None) == H
        np.testing.assert_array_equal(np.array(got), np.array([ref.result(b)[k] for k in (
            "total_return", "regularization", "improvement", "expected", "surprise", "winner")]))
        a = np.zeros(m.nu)
        assert lib.mjpc_b200_batch_planner_action_from_policy(q.h, b, a.ctypes.data_as(dp), state.ctypes.data_as(dp),
                                                              C.c_double(0.05), 0) == 0
        np.testing.assert_array_equal(a, ref.action_from_policy(b, 0.05, state))
    assert lib.mjpc_b200_batch_sampling_planner_get_result(q.h, 0, *([None] * 5)) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_state(q.h, 2, xp, t0, mcp) == BAD_ARGUMENT
    lib.mjpc_b200_batch_planner_destroy(q.h)
    q.h = None
    ref.close()


def test_batch_gradient_particles_descend():
    """The criterion of the single planner's particle test on a batch: four particles with different goals, planned
    together, each descend monotonically to below 0.9 of their first return."""
    from mujoco_mpc_b200.engine import CppBatchGradientPlanner
    m = get_model("particle")
    H, B = 26, 4
    goals = [(0.1, 0.1), (-0.1, 0.05), (0.05, -0.1), (-0.08, -0.08)]
    pl = CppBatchGradientPlanner(m, B, H, num_trajectory=16, num_spline_points=6, representation=1, fd_tolerance=1e-3)
    for b, goal in enumerate(goals):
        mc = mocap_of(m).copy(); mc[:2] = goal
        pl.reset(b); pl.set_state(b, np.zeros(4), 0.0, mc)
    rets = []
    for _ in range(40):
        pl.optimize_policy()
        rets.append([pl.result(b)["total_return"] for b in range(B)])
    rets = np.array(rets)
    for b in range(B):
        assert rets[-1, b] < 0.9 * rets[0, b], (b, rets[:, b])
        assert all(y <= x + 1e-7 for x, y in zip(rets[:, b], rets[1:, b]))
    pl.close()


# ------------------------------------------------------------------------------------------ iLQS
IKW = dict(num_trajectory=8, num_rollouts=6, fd_tolerance=1e-3, fd_mode=0)
SIGMA = [0.1, 0.1, 0.0, 0.0, 0.0, 0.0, 0.0, 0.1, 0.1, 0.1]   # exploration 0: sampling cannot improve, iLQG runs


def _ilqs_batch(m, B, H, pr, seeds):
    from mujoco_mpc_b200.engine import CppBatchILQSPlanner
    batch = CppBatchILQSPlanner(m, B, H, seeds=seeds, **IKW)
    for b in range(B):
        batch.reset(b)
        batch.set_task(b, pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    return batch


@pytest.mark.parametrize("B", [3, 1])
def test_batch_ilqs_planner_equals_independent_planners(B):
    """Both active policies and the iLQG -> spline conversion (an iteration that starts from an active iLQG policy)
    must occur."""
    from mujoco_mpc_b200.engine import CppILQSPlanner
    m = get_model("particle")
    H = 26
    pr = _problems(m, H, B=3)
    seeds = [0x5EED + 7 * b for b in range(B)]
    batch = _ilqs_batch(m, B, H, pr, seeds)
    singles = [CppILQSPlanner(m, H, seed=seeds[b], **IKW) for b in range(B)]
    for b in range(B):
        singles[b].reset()
        singles[b].set_task(pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    active = [[] for _ in range(B)]
    for it, sigma in enumerate(SIGMA):
        batch.set_exploration(sigma)
        for b in range(B):
            singles[b].set_exploration(sigma)
            batch.set_state(b, *_state(pr, b, it)); singles[b].set_state(*_state(pr, b, it))
        codes = batch.optimize_policy()
        for b in range(B):
            ok = singles[b].optimize_policy()
            assert codes[b] == ok, (it, b)
            r, s = batch.result(b), singles[b].result()
            active[b].append(s["active_policy"])
            for key in s:
                np.testing.assert_array_equal(r[key], s[key], err_msg=f"iteration {it} problem {b}: {key}")
            t0 = pr["times"][b] + 0.01 * it
            for dt in (0.0, 0.013, 0.1, 0.2):
                for prev in (False, True):
                    np.testing.assert_array_equal(batch.action_from_policy(b, t0 + dt, pr["states"][b], prev),
                                                  singles[b].action_from_policy(t0 + dt, pr["states"][b], prev))
    seen = sum(active, [])
    assert 0 in seen and 1 in seen, active
    assert any(1 in a[:-1] for a in active), active     # a later iteration converts the iLQG policy to a spline
    batch.close()
    for s in singles:
        s.close()


def test_batch_ilqs_problems_are_independent():
    m = get_model("particle")
    H = 26
    pr = _problems(m, H, B=3)
    ch = {k: np.array(v, copy=True) for k, v in pr.items()}
    ch["states"][1, m.nq:] += 0.2
    ch["times"][1] += 0.07
    ch["weights"][1] *= 2.0
    seeds = [1, 2, 3]

    def run(p):
        batch = _ilqs_batch(m, 3, H, p, seeds)
        out = []
        for it, sigma in enumerate(SIGMA[:7]):
            batch.set_exploration(sigma)
            for b in range(3):
                batch.set_state(b, *_state(p, b, it))
            codes = batch.optimize_policy()
            out.append((codes, [batch.result(b) for b in range(3)],
                        [batch.action_from_policy(b, p["times"][b] + 0.01 * it + 0.05, p["states"][b]) for b in range(3)]))
        batch.close()
        return out

    before, after = run(pr), run(ch)
    assert any((a[2][1] != b[2][1]).any() for a, b in zip(after, before))
    for (ca, ra, aa), (cb, rb, ab) in zip(after, before):
        for b in (0, 2):
            assert ca[b] == cb[b]
            for key in rb[b]:
                np.testing.assert_array_equal(ra[b][key], rb[b][key], err_msg=key)
            np.testing.assert_array_equal(aa[b], ab[b])


def test_batch_ilqs_particles_reach_their_goals():
    """The criterion of the single iLQS particle test on a batch of four particles with different goals."""
    from mujoco_mpc_b200.engine import CppBatchILQSPlanner
    m = get_model("particle")
    H, B = 26, 4
    goals = [(0.1, 0.1), (-0.1, 0.05), (0.05, -0.1), (-0.08, -0.08)]
    pl = CppBatchILQSPlanner(m, B, H, num_trajectory=16, num_rollouts=8, fd_tolerance=1e-3)
    for b, goal in enumerate(goals):
        mc = mocap_of(m).copy(); mc[:2] = goal
        pl.reset(b); pl.set_state(b, np.zeros(4), 0.0, mc)
    for _ in range(30):
        pl.optimize_policy()
    for b in range(B):
        r = pl.result(b)
        assert min(r["sampling_return"], r["ilqg_return"] if r["ilqg_return"] > 0 else 1e9) < 0.05, (b, r)
    pl.close()
