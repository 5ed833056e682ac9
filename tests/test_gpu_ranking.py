"""GPU: the layer that turns rollouts into a decision - each candidate's return, the ensemble score of its member
returns and the ranking the planners read - against numpy restatements in float64 written from the definitions.

* Ranking (rank_kernel through mjpc_b200_debug_rank): every segment's order is numpy's stable argsort of its returns,
  bitwise, with subnormals read as a zero of their sign (the library is built with flush-to-zero); so NaN sorts after
  every number, NaNs among themselves by index, and every segment is a permutation of range(N).
* Ensemble score (ensemble_score_kernel through mjpc_b200_debug_ensemble_score, and mjpc_b200_host_ensemble_score):
  the member returns sorted in descending order (NaN first, ties to the lower member), the first `worst` summed left
  to right in float64, divided once by worst and rounded to float32; 1e6 and failed if any member failed.
* Return identity: a candidate's return is the float32 left-to-right sum of its own recorded costs divided by H (the
  division is the fast-math one, within 2 ulp), or exactly 1e6 with failure 1 when it diverged.
* End to end: a batched launch with a problem whose every candidate returns NaN (a NaN weight) and one where only some
  do (an infinite weight on a norm that is 0 for some candidates) ranks every segment as the reference does, leaves the
  other problems bitwise as they were, and the sampling planners decide on those returns as their Python mirrors do.

Bitwise comparisons of float arrays treat every NaN as equal: NaN payloads are not part of any definition here."""
import math

import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_batched import _problems
from test_gpu_model_ensemble import _diverging_variant
from test_gpu_model_variants import _variants

pytestmark = pytest.mark.gpu

FAIL_RETURN = np.float32(1.0e6)
MAX_CANDIDATES = 1000
TINY = np.finfo(np.float32).tiny


@pytest.fixture(scope="module")
def engine():
    from mujoco_mpc_b200.engine import Engine
    e = Engine(get_model("particle"), MAX_CANDIDATES, 4)
    yield e
    e.close()


def _same_bits(got, want, what=""):
    """float32 arrays equal bit for bit, any NaN equal to any NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what}: NaN positions")
    np.testing.assert_array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32), err_msg=what)


# ------------------------------------------------------------------------------------------ 1. ranking
def _flush(x):
    """subnormals -> a zero of the same sign (what a flush-to-zero comparison sees)"""
    x = np.array(x, np.float32)
    sub = (x != 0) & (np.abs(x) < TINY)
    x[sub] = np.copysign(np.float32(0), x[sub])
    return x


def _ref_order(x):
    return np.argsort(_flush(x), axis=-1, kind="stable").astype(np.int32)


SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0e6, 1.0e-40, -1.0e-40, 1.4e-45, -3.0e-42, 0.5, -0.5, 0.5,
                    TINY, -TINY], np.float32)


def _segment(kind, N, rng):
    """N returns of one kind"""
    if kind == "random":
        return rng.standard_normal(N).astype(np.float32)
    if kind == "permutation":
        return rng.permutation(N).astype(np.float32)
    if kind == "ties":
        return rng.choice(np.array([0.25, 1.0, 3.0, 1.0e6], np.float32), N)
    if kind == "nans":          # two or more NaNs (when N allows) among ties and distinct numbers
        x = rng.choice(np.array([0.5, 0.1, 2.0], np.float32), N) + rng.integers(0, 2, N) * rng.standard_normal(N)
        x = x.astype(np.float32)
        x[rng.choice(N, max(min(N, 2), N // 3), replace=False)] = np.nan
        return x
    if kind == "all_nan":
        return np.full(N, np.nan, np.float32)
    if kind == "special":       # +-inf, +-0, 1e6, subnormals of both signs, NaN
        return rng.choice(SPECIAL, N)
    raise ValueError(kind)


KINDS = ("random", "permutation", "ties", "nans", "all_nan", "special")


def _check_order(order, returns, what):
    N = returns.shape[-1]
    missing = np.argwhere(order < 0)
    assert not len(missing), f"{what}: slots never written (segment, rank): {missing[:8].tolist()}"
    for b in range(order.shape[0]):
        lost = sorted(set(range(N)) - set(order[b].tolist()))
        assert not lost, f"{what}: segment {b} is not a permutation, candidates {lost[:8]} lost"
    want = _ref_order(returns)
    bad = np.argwhere(order != want)
    assert not len(bad), (f"{what}: first differences (segment, rank) {bad[:4].tolist()}: "
                          f"got {order[tuple(bad[0])]}, want {want[tuple(bad[0])]}")


def test_two_nans_in_one_segment_each_get_a_rank(engine):
    """two NaN returns in one segment: each gets its own rank, after the numbers, the lower index first"""
    r = np.array([[0.5, np.nan, 0.1, np.nan, np.inf, 0.1]], np.float32)
    order = engine.debug_rank(r)
    np.testing.assert_array_equal(order, [[2, 5, 0, 4, 1, 3]])


@pytest.mark.parametrize("nseg", [1, 3, 64])
@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 255, 256, 257, MAX_CANDIDATES])
def test_rank_is_the_stable_argsort(engine, N, nseg):
    assert engine.info.max_candidates == MAX_CANDIDATES
    rng = np.random.default_rng(1000 * N + nseg)
    for kind in KINDS:
        r = np.stack([_segment(kind, N, rng) for _ in range(nseg)])
        _check_order(engine.debug_rank(r), r, f"{kind}, N = {N}, nseg = {nseg}")
    # every kind in one launch, segment b of kind b mod 6
    r = np.stack([_segment(KINDS[b % len(KINDS)], N, rng) for b in range(nseg)])
    _check_order(engine.debug_rank(r), r, f"mixed, N = {N}, nseg = {nseg}")


def test_rank_argument_errors_leave_the_handle_usable(engine):
    import ctypes as C
    lib, h = engine.lib, engine.h
    r = np.zeros(8, np.float32)
    o = np.zeros(8, np.int32)
    rp, op = r.ctypes.data_as(C.POINTER(C.c_float)), o.ctypes.data_as(C.POINTER(C.c_int))
    for args in ((rp, 0, 8, op), (rp, 1, 0, op), (rp, -1, 8, op), (None, 1, 8, op), (rp, 1, 8, None)):
        assert lib.mjpc_b200_debug_rank(h, *args) == -1, args
    mr = np.zeros(8, np.float32); mf = np.zeros(8, np.uint8); s = np.zeros(8, np.float32); f = np.zeros(8, np.uint8)
    mrp, sp = mr.ctypes.data_as(C.POINTER(C.c_float)), s.ctypes.data_as(C.POINTER(C.c_float))
    mfp, fp = mf.ctypes.data_as(C.POINTER(C.c_uint8)), f.ctypes.data_as(C.POINTER(C.c_uint8))
    for B, K, N, worst in ((0, 1, 1, 1), (1, 0, 1, 1), (1, 33, 1, 1), (1, 2, 0, 1), (1, 2, 4, 0), (1, 2, 4, 3)):
        assert lib.mjpc_b200_debug_ensemble_score(h, mrp, mfp, B, K, N, worst, sp, fp) == -1, (B, K, N, worst)
    assert lib.mjpc_b200_debug_ensemble_score(h, None, mfp, 1, 2, 4, 1, sp, fp) == -1
    r = np.array([[3.0, np.nan, 1.0, np.nan]], np.float32)
    np.testing.assert_array_equal(engine.debug_rank(r), [[2, 0, 1, 3]])


def test_rollout_returns_are_never_subnormal():
    """A rollout's returns are normal numbers or zero, never subnormal, so the reference may read subnormal returns
    as the zeros the ranking's flush-to-zero comparisons see.  Particles a tiny offset from their goal put every cost
    on both sides of the subnormal range."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model("particle")
    N, H = 24, 4
    e = Engine(m, N, H)
    mocap = mocap_of(m).copy()
    mocap[:3] = 0.0                                          # the goal at the origin
    ret = []
    for x in 10.0 ** -np.arange(14.0, 26.0):
        state = np.array([x, -x, 0.0, 0.0])
        knots = np.zeros((N, 2, m.nu))
        knots[1:, :, 0] = np.float32(1e-30) * np.arange(1, N)[:, None]
        r, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, np.array([0.0, 1.0]), 1, H)
        assert not fail.any()
        ret.append(r)
    ret = np.concatenate(ret)
    assert (ret == 0).any() and (ret > 0).any()
    assert not ((ret != 0) & (np.abs(ret) < TINY)).any(), ret
    e.close()


# ------------------------------------------------------------------------------------------ 2. ensemble score
def _ref_score(r, f, worst):
    """one candidate's score from its K member returns r (float32) and failure flags f, in float64"""
    K = len(r)
    key = [(0, 0.0, k) if math.isnan(float(r[k])) else (1, -float(r[k]), k) for k in range(K)]
    ranked = [k for _, _, k in sorted(key)]
    total = 0.0
    for p in range(worst):
        total += float(r[ranked[p]])
    if np.any(f):
        return FAIL_RETURN, 1
    return np.float32(total / worst), 0


def _member_returns(B, K, N, rng):
    """[B][K][N] member returns and failure flags: candidate i of kind i mod 6 - distinct, tied, with NaNs, with
    +-inf, all NaN, and with failed members (whose return is 1e6, as a failed rollout's)"""
    r = np.empty((B, K, N), np.float32)
    f = np.zeros((B, K, N), np.uint8)
    for b in range(B):
        for i in range(N):
            kind = i % 6
            x = rng.standard_normal(K).astype(np.float32) * np.float32(10.0 ** rng.integers(-3, 4))
            if kind == 1:
                x = rng.choice(np.array([0.5, 2.0, -1.0], np.float32), K)
            elif kind == 2:
                x[rng.choice(K, min(K, 1 + rng.integers(0, 3)), replace=False)] = np.nan
            elif kind == 3:
                x[rng.choice(K, min(K, 2), replace=False)] = rng.choice(np.array([np.inf, -np.inf, np.nan], np.float32), min(K, 2))
            elif kind == 4:
                x[:] = np.nan
            elif kind == 5:
                fl = rng.random(K) < 0.3
                fl[rng.integers(K)] = True
                f[b, fl, i] = 1
                x[fl] = FAIL_RETURN
            r[b, :, i] = x
    return r, f


def _worsts(K):
    return sorted({1, (K + 1) // 2, K})


@pytest.mark.parametrize("K,worst", [(K, w) for K in (1, 2, 5, 31, 32) for w in _worsts(K)])
def test_ensemble_score_is_the_definition(engine, K, worst):
    from mujoco_mpc_b200.engine import host_ensemble_score
    B, N = 3, 37
    rng = np.random.default_rng(31 * K + worst)
    mr, mf = _member_returns(B, K, N, rng)
    got, gfail = engine.debug_ensemble_score(mr, mf, worst)
    want = np.zeros((B, N), np.float32)
    wfail = np.zeros((B, N), np.uint8)
    for b in range(B):
        for i in range(N):
            want[b, i], wfail[b, i] = _ref_score(mr[b, :, i], mf[b, :, i], worst)
            hs, hf = host_ensemble_score(mr[b, :, i], mf[b, :, i], worst)
            _same_bits(hs, want[b, i], f"host score, problem {b} candidate {i}")
            assert hf == wfail[b, i], (b, i)
    _same_bits(got, want, f"device score, K = {K}, worst = {worst}")
    np.testing.assert_array_equal(gfail, wfail)
    assert np.isnan(want).any() and np.isfinite(want).any()
    assert (wfail == 1).any() and (wfail == 0).any()


# ------------------------------------------------------------------------------------------ 3. return identity
H_MAX = 24


def _ulps(a, b):
    """distance in float32 ulps of two finite float32 arrays"""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, np.int64(-2 ** 31) - i, i)
    return np.abs(key(a) - key(b))


def _check_returns(ret, fail, costs, H, what):
    """ret / fail [n], costs [n][H]: each return the float32 left-to-right sum of its costs over H (2 ulp: the
    library's fast-math division), or exactly 1e6 if it failed.  Returns the largest distance seen in ulps."""
    ret, costs = np.asarray(ret, np.float32), np.asarray(costs, np.float32)
    assert (ret[fail == 1] == FAIL_RETURN).all(), what
    ok = fail == 0
    total = np.zeros(len(ret), np.float32)
    for t in range(H):
        total = (total + costs[:, t]).astype(np.float32)
    want = (total / np.float32(H)).astype(np.float32)
    assert np.isfinite(want[ok]).all(), what
    d = _ulps(ret[ok], want[ok])
    assert d.max(initial=0) <= 2, f"{what}: {d.max()} ulp, candidate {np.flatnonzero(ok)[d.argmax()]}"
    assert not ((ret != 0) & (np.abs(ret) < TINY)).any(), what
    return int(d.max(initial=0))


@pytest.mark.parametrize("H", [1, 2, H_MAX])
@pytest.mark.parametrize("launch", ["plain", "batched", "model_ensemble", "state_ensemble"])
def test_return_is_the_mean_of_the_recorded_costs(launch, H):
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    B, N, K = 3, 8, 4
    pr = _problems(m, N, H_MAX, B=B)
    e = Engine(m, B * N, H_MAX)
    args = (pr["states"], pr["times"], pr["mocaps"], pr["knots"], pr["knot_times"], 2, H)
    task = dict(weights=pr["weights"], parameters=pr["parameters"], task_states=pr["task_states"])
    if launch == "plain":
        ret, fail, _ = e.rollout_spline(pr["states"][0], pr["times"][0], pr["mocaps"][0], pr["knots"][0],
                                        pr["knot_times"][0], 2, H)
        rows = [(ret, fail, e.fetch_all()["costs"])]
    elif launch == "batched":
        ret, fail, _ = e.rollout_spline_batched(*args, **task)
        rows = [(ret.reshape(-1), fail.reshape(-1), e.fetch_all()["costs"])]
    else:
        if launch == "model_ensemble":     # member 3 diverges on every candidate with large enough controls
            e.set_model_ensemble(_variants("quadruped")[:K - 1] + [_diverging_variant()], worst=2)
            e.rollout_spline_batched(*args, **task)
        else:
            rng = np.random.default_rng(4)
            n = 2 * m.nv
            covs = np.stack([0.01 * (1 + b) * (lambda A: A @ A.T / n + 0.2 * np.eye(n))(rng.standard_normal((n, n)))
                             for b in range(B)])
            e.rollout_spline_belief_batched(pr["states"], covs, pr["times"], pr["mocaps"], pr["knots"],
                                            pr["knot_times"], 2, H, K, 2, **task)
        mr, mf = e.fetch_ensemble()
        rows = []
        for k in range(K):
            costs = np.stack([e.fetch_trajectory_member(c, k)["costs"] for c in range(B * N)])
            rows.append((mr[:, k].reshape(-1), mf[:, k].reshape(-1), costs))
        if launch == "model_ensemble" and H == H_MAX:
            assert mf[:, K - 1].any() and not mf[:, :K - 1].any()
    worst = 0
    for k, (ret, fail, costs) in enumerate(rows):
        worst = max(worst, _check_returns(ret, fail, costs, H, f"{launch}, H = {H}, member {k}"))
    print(f"return identity, {launch} launch, H = {H}: largest distance {worst} ulp")
    e.close()


# ------------------------------------------------------------------------------------------ 4. end to end
# The Cart-Pole's terms: Vertical, Centered, Velocity, Control (residual = ctrl, quadratic norm).  A NaN Velocity weight
# makes every candidate's return NaN; an infinite Control weight gives inf * 0 = NaN for a candidate whose control is
# exactly zero at some step and +inf for the others.
VELOCITY, CONTROL = 2, 3


def _cartpole_weights(m, kind, b):
    w = np.asarray(m.task_weight, float) * (1.0 + 0.2 * b)
    if kind == "nan":
        w[VELOCITY] = np.nan
    elif kind == "partial":
        w[CONTROL] = np.inf
    return w


def _cartpole_launch(m, kinds, N, H, rng):
    """inputs of a batched Cart-Pole launch, one problem per entry of kinds; candidates 0, 3 and 5 have zero controls
    (linear interpolation of zero knots), the others a control of one sign that is never zero"""
    B, P = len(kinds), 4
    states = np.stack([[0.1 * b, np.pi - 0.2 + 0.05 * b, 0.0, 0.1] for b in range(B)])
    times = 0.3 * np.arange(B)
    knots = rng.uniform(0.05, 0.9, (B, N, P, m.nu)) * rng.choice([-1.0, 1.0], (B, N, 1, 1))
    knots[:, [0, 3, 5]] = 0.0
    kt = np.stack([t + np.linspace(0.0, (H - 1) * m.opt_timestep, P) for t in times])
    weights = np.stack([_cartpole_weights(m, k, b) for b, k in enumerate(kinds)])
    return dict(states=states, times=times, mocaps=np.zeros((B, 0)), knots=knots, knot_times=kt, weights=weights)


def _run(e, a, H):
    return e.rollout_spline_batched(a["states"], a["times"], a["mocaps"], a["knots"], a["knot_times"], 1, H,
                                    weights=a["weights"])


def test_batched_launch_with_nan_returns():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("cartpole")
    kinds = ["normal", "nan", "normal", "partial", "normal"]
    N, H = 40, 32
    a = _cartpole_launch(m, kinds, N, H, np.random.default_rng(8))
    e = Engine(m, len(kinds) * N, H)
    ret, fail, order = _run(e, a, H)
    assert not fail.any()
    assert np.isnan(ret[1]).all()
    nan3 = np.isnan(ret[3])
    assert set(np.flatnonzero(nan3)) == {0, 3, 5} and (ret[3][~nan3] == np.inf).all(), ret[3]
    normal = [b for b, k in enumerate(kinds) if k == "normal"]
    assert np.isfinite(ret[normal]).all()
    _check_order(order, ret, "batched Cart-Pole launch")
    # the normal problems alone: bitwise the same returns and order
    alone = {k: v[normal] for k, v in a.items()}
    r2, f2, o2 = _run(e, alone, H)
    _same_bits(ret[normal], r2, "normal problems, with and without the NaN problems")
    np.testing.assert_array_equal(order[normal], o2)
    np.testing.assert_array_equal(fail[normal], f2)
    e.close()


class _ArgsortBackend:
    """An engine planning one problem with its own weights, whose ranking is the reference's: numpy's stable argsort
    of the returns it computed (the planners' mirrors read the order from their backend)."""

    def __init__(self, m, N, H, weight):
        from mujoco_mpc_b200.engine import Engine
        self.e = Engine(m, N, H)
        self.e.set_task(weight=weight)

    def rollout_spline(self, *args):
        ret, fail, _ = self.e.rollout_spline(*args)
        return ret, fail, np.argsort(ret, kind="stable")

    def set_xfrc_noise(self, *args):
        self.e.set_xfrc_noise(*args)


PLANNER_N, PLANNER_H, N_ELITE = 16, 32, 4
ROBUST = dict(ncandidates=3, nrepetitions=2, xfrc_std=1.0, xfrc_rate=0.1)
SG = dict(num_gradient=4, gradient_filter=0.6)


def _mirror(kind, m, backend, seed):
    from mujoco_mpc_b200 import planner as Py
    N, H = PLANNER_N, PLANNER_H
    if kind == "sampling":
        return Py.SamplingPlanner(m, backend, num_trajectory=N, horizon=H, seed=seed)
    if kind == "ce":
        return Py.CrossEntropyPlanner(m, backend, num_trajectory=N, horizon=H, n_elite=N_ELITE, seed=seed)
    if kind == "sg":
        return Py.SampleGradientPlanner(m, backend, num_trajectory=N, horizon=H, seed=seed, **SG)
    return Py.RobustPlanner(m, backend, num_trajectory=N, horizon=H, seed=seed, **ROBUST)


def _cpp(kind, m, seeds, batched):
    from mujoco_mpc_b200 import engine as E
    N, H = PLANNER_N, PLANNER_H
    kw = {"sampling": {}, "ce": dict(n_elite=N_ELITE), "sg": SG, "robust": ROBUST}[kind]
    if batched:
        cls = {"sampling": E.CppBatchSamplingPlanner, "ce": E.CppBatchCrossEntropyPlanner,
               "sg": E.CppBatchSampleGradientPlanner, "robust": E.CppBatchRobustPlanner}[kind]
        return cls(m, len(seeds), N, H, seeds=seeds, **kw)
    cls = {"sampling": E.CppSamplingPlanner, "ce": E.CppCrossEntropyPlanner, "sg": E.CppSampleGradientPlanner,
           "robust": E.CppRobustPlanner}[kind]
    return [cls(m, N, H, seed=s, **kw) for s in seeds]


def _close(a, b, what, **tol):
    np.testing.assert_allclose(np.asarray(a, float), np.asarray(b, float), equal_nan=True, err_msg=what, **tol)


def _assert_decision(kind, got, py, ret, what):
    """the C++ planner's result against its mirror's state after the same iteration"""
    _close(got["returns"], ret, f"{what}: returns", rtol=1e-5)
    if kind == "ce":
        np.testing.assert_array_equal(got["order"][:N_ELITE], py.order[:N_ELITE], err_msg=f"{what}: elites")
        _close(got["knots"], py.values, f"{what}: policy", atol=1e-6)
        _close(got["variance"], py.variance, f"{what}: variance", rtol=1e-4, atol=1e-10)
        return
    d = py.delegate if kind == "robust" else py
    assert got["winner"] == d.winner, f"{what}: winner {got['winner']}, mirror {d.winner}"
    _close(got["knots"], d.values, f"{what}: policy", atol=1e-6)
    if kind == "sg":
        assert got["winner_type"] == py.winner_type, what
        _close(got["gradient"], py.gradient, f"{what}: gradient", atol=1e-6)
        _close(got["gradient_knots"], py.gradient_knots, f"{what}: gradient candidates", atol=1e-6)
    if kind == "robust":
        _close(got["scores"], py.scores, f"{what}: scores", rtol=1e-5)


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("kind", ["sampling", "ce", "sg", "robust"])
def test_planners_decide_on_nan_returns_as_their_mirrors(kind, batched):
    """Problem 0 plans with a NaN weight (every return NaN), problem 1 with an infinite Control weight (the zero
    nominal returns NaN, the noisy candidates +inf), problem 2 normally."""
    m = get_model("cartpole")
    kinds = ["nan", "partial", "normal"]
    seeds = [0x5EED, 7, 123456]
    B = len(kinds)
    weights = [_cartpole_weights(m, k, b) for b, k in enumerate(kinds)]
    states = [np.array([0.05 * b, np.pi - 0.3 + 0.1 * b, 0.0, 0.0]) for b in range(B)]
    mirrors = [_mirror(kind, m, _ArgsortBackend(m, PLANNER_N + 1, PLANNER_H, weights[b]), seeds[b]) for b in range(B)]
    cpp = _cpp(kind, m, seeds, batched)
    for b in range(B):
        mirrors[b].reset(np.zeros(m.nu))
        if batched:
            cpp.reset(b, np.zeros(m.nu)); cpp.set_task(b, weight=weights[b])
        else:
            cpp[b].reset(np.zeros(m.nu)); cpp[b].set_task(weight=weights[b])
    saw_nan = [False] * B
    for it in range(3):
        for b in range(B):
            t = 0.01 * it
            mirrors[b].set_state(states[b], t, np.zeros(0))
            (cpp.set_state(b, states[b], t, np.zeros(0)) if batched else cpp[b].set_state(states[b], t, np.zeros(0)))
        res = cpp.optimize_policy() if batched else [p.optimize_policy() for p in cpp]
        for b in range(B):
            ret, _ = mirrors[b].optimize_policy()
            saw_nan[b] |= bool(np.isnan(ret).any())
            _assert_decision(kind, res[b], mirrors[b], ret, f"{kind}, batched {batched}, iteration {it}, problem {b}")
            for dt in (0.0, 0.05, 0.2):
                t = 0.01 * it + dt
                a = cpp.action_from_policy(b, t) if batched else cpp[b].action_from_policy(t)
                _close(a, mirrors[b].action_from_policy(t), f"action, iteration {it}, problem {b}", atol=1e-6)
    assert saw_nan == [True, True, False]
    for p in ([cpp] if batched else cpp):
        p.close()
    for mr in mirrors:
        mr.backend.e.close()
