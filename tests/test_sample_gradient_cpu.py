"""CPU: the Sample Gradient planner mirror (mujoco_mpc_b200.planner.SampleGradientPlanner,
mjpc/planners/sample_gradient/planner.cc) against literal restatements of the reference's arithmetic on a stub backend
with prescribed returns, and the behavioural bar of the sampling planner on the oracle backend."""
import ctypes
import math
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import OracleBackend, get_model, mocap_of


def _model(ctrlrange=((-5.0, 5.0), (-5.0, 5.0)), P=3, sigma=0.1, interp=2):
    return SimpleNamespace(nu=len(ctrlrange), opt_timestep=0.01, actuator_ctrlrange=np.array(ctrlrange, float).reshape(-1),
                           numeric={"sampling_spline_points": [P], "sampling_exploration": [sigma],
                                    "sampling_representation": [interp]})


class StubBackend:
    """rollout_spline returns the next prescribed returns (and, optionally, a prescribed order) and records the knots."""

    def __init__(self, returns, orders=None):
        self.returns, self.orders, self.calls = list(returns), list(orders or []), []

    def rollout_spline(self, state, time, mocap, knots, kt, interp, H):
        ret = np.asarray(self.returns.pop(0), np.float32)
        assert len(ret) == len(knots)
        self.calls.append(dict(knots=np.array(knots, float), times=np.array(kt, float)))
        order = self.orders.pop(0) if self.orders else np.argsort(ret, kind="stable")
        return ret, np.zeros(len(ret), np.uint8), np.asarray(order)


def _planner(backend, N=7, G=3, f=0.7, horizon=16, **kw):
    from mujoco_mpc_b200.planner import SampleGradientPlanner
    pl = SampleGradientPlanner(_model(**kw), backend, num_trajectory=N, horizon=horizon, num_gradient=G, gradient_filter=f)
    pl.reset(np.array([0.3, -0.2]))
    pl.set_state(np.zeros(4), 0.25, np.zeros(0))
    return pl


def test_sample_gradient_arithmetic_matches_literal_formulas():
    from mujoco_mpc_b200.planner import philox_normal
    N, G, f, sigma, P, nu = 7, 3, 0.7, 0.1, 3, 2
    n = N - G
    rng = np.random.default_rng(11)
    rets = [rng.uniform(1.0, 2.0, N) for _ in range(4)]
    pl = _planner(StubBackend(rets), N, G, f)
    # LogScale(2, 1e-3, G): ascending from 1e-3, log-spaced
    steps = [math.exp(math.log(1e-3) + j * (math.log(2.0) - math.log(1e-3)) / (G - 1)) for j in range(G)]
    f0 = math.log(0.5 * n + 1.0)
    den = sum(max(0.0, f0 - math.log(j + 1)) for j in range(n))
    grad_prev = np.zeros((P, nu))
    weights = None
    for it in range(4):
        ret, _ = pl.optimize_policy()
        call = pl.backend.calls[-1]
        knots, nominal = call["knots"], call["knots"][0]
        np.testing.assert_allclose(call["times"], 0.25 + np.arange(P) * 15 * 0.01 / (P - 1), atol=1e-15)
        z = philox_normal(it, N, P, nu)
        np.testing.assert_allclose(knots[1:n], nominal + 0.1 * z[1:n], atol=1e-12)   # noise not scaled by ctrlrange
        if it > 0:   # the gradient candidates of the previous iteration, resampled onto the same knot times
            np.testing.assert_allclose(knots[n:], prev_candidates, atol=1e-12)
        ret = np.asarray(ret, float)
        if it == 0:
            # weights indexed by candidate index on the call that computes them: independent of the returns
            order0 = np.argsort(ret[:n], kind="stable")
            weights = np.array([max(0.0, f0 - math.log(order0[i] + 1)) / den - 1.0 / n for i in range(n)])
            np.testing.assert_allclose(pl.return_weight, weights, atol=1e-12)
            grad = sum(z[j] * (max(0.0, f0 - math.log(j + 1)) / den - 1.0 / n) / n for j in range(1, n))
        else:
            # cached weights paired with the ranking of all N; slot 0 and the gradient slots carry zero noise
            order = np.argsort(ret, kind="stable")
            zn = np.where((np.arange(N) >= 1) & (np.arange(N) < n), 1.0, 0.0)[:, None, None] * z
            grad = sum(zn[order[i]] * weights[i] / n for i in range(n))
        np.testing.assert_allclose(pl.gradient, grad, atol=1e-12)
        np.testing.assert_allclose(pl.gradient_previous, grad_prev, atol=1e-12)
        np.testing.assert_allclose(pl.step_size, steps, rtol=1e-14)
        expect = np.stack([np.clip(nominal - steps[j] / sigma * (f * grad + (1 - f) * grad_prev), -5, 5) for j in range(G)])
        np.testing.assert_allclose(pl.gradient_knots, expect, atol=1e-12)
        prev_candidates, grad_prev = expect, grad
        assert pl.iteration == it + 1
    assert len(pl.backend.calls) == 4


def test_weights_ignore_returns_on_first_call_but_not_later():
    N, G = 8, 2
    n = N - G
    rng = np.random.default_rng(5)
    r0, r1 = rng.uniform(1.0, 2.0, N), rng.uniform(1.0, 2.0, N)
    perm = np.concatenate([[0], 1 + rng.permutation(n - 1), np.arange(n, N)])     # permutes the noisy samples
    assert not np.array_equal(perm, np.arange(N))
    a = _planner(StubBackend([r0, r1]), N, G, 0.5)
    b = _planner(StubBackend([r0[perm], r1[perm]]), N, G, 0.5)
    a.optimize_policy(); b.optimize_policy()
    np.testing.assert_allclose(a.gradient, b.gradient, atol=1e-12)
    a.optimize_policy(); b.optimize_policy()
    assert np.abs(a.gradient - b.gradient).max() > 1e-6


@pytest.mark.parametrize("case", ["nominal", "noisy", "gradient", "tie"])
def test_winner_and_winner_type(case):
    N, G = 6, 2                                  # 0 nominal, 1..3 noisy, 4..5 gradient
    ret = np.full(N, 2.0)
    order = None
    if case == "nominal":
        ret[0] = 1.0
    elif case == "noisy":
        ret[2] = 1.0
    elif case == "gradient":
        ret[5] = 1.0
    else:                                        # a candidate ties the nominal and is ranked first: no strict improvement
        ret[0] = ret[3] = 1.0
        order = [[3, 0, 1, 2, 4, 5]]
    pl = _planner(StubBackend([ret], order), N, G, 1.0)
    pl.optimize_policy()
    knots = pl.backend.calls[-1]["knots"]
    winner, wtype = {"nominal": (0, 0), "noisy": (2, 1), "gradient": (5, 2), "tie": (0, 0)}[case]
    assert (pl.winner, pl.winner_type) == (winner, wtype)
    np.testing.assert_array_equal(pl.values, knots[winner])
    assert pl.improvement == max(float(ret[0]) - float(ret[winner]), 0.0)


def test_first_iteration_gradient_candidates_are_the_clamped_zero_plan():
    cr = ((0.2, 1.0), (-1.0, -0.3))
    N, G = 6, 3
    pl = _planner(StubBackend([np.arange(N, dtype=float)] * 3), N, G, 0.8, ctrlrange=cr)
    pl.optimize_policy()
    knots = pl.backend.calls[-1]["knots"]
    np.testing.assert_array_equal(knots[N - G:], np.broadcast_to([0.2, -0.3], (G, 3, 2)))
    pl.optimize_policy()
    assert not np.array_equal(pl.backend.calls[-1]["knots"][N - G:], knots[N - G:])
    pl.reset(np.array([0.5, -0.5])); pl.set_state(np.zeros(4), 0.25, np.zeros(0))     # Reset clears them again
    pl.optimize_policy()
    np.testing.assert_array_equal(pl.backend.calls[-1]["knots"][N - G:], np.broadcast_to([0.2, -0.3], (G, 3, 2)))


def test_no_gradient_candidates_is_sampling_with_unscaled_noise():
    from mujoco_mpc_b200.planner import philox_normal
    N, sigma = 9, 0.3
    rng = np.random.default_rng(2)
    rets = [rng.uniform(1.0, 2.0, N) for _ in range(3)]
    pl = _planner(StubBackend(rets), N, 0, 1.0, sigma=sigma, ctrlrange=((-0.4, 0.4), (-2.0, 2.0)))
    for it in range(3):
        ret, _ = pl.optimize_policy()
        knots = pl.backend.calls[-1]["knots"]
        z = philox_normal(it, N, 3, 2)
        np.testing.assert_allclose(knots[1:], np.clip(knots[0] + sigma * z[1:], [-0.4, -2.0], [0.4, 2.0]), atol=1e-12)
        best = int(np.argmin(ret))
        assert pl.winner == (best if ret[best] < ret[0] else 0) and pl.winner_type == (1 if pl.winner else 0)
        np.testing.assert_array_equal(pl.values, knots[pl.winner])
        assert pl.gradient_knots.shape == (0, 3, 2) and not pl.gradient.any()


def test_num_gradient_is_clamped_to_n_minus_one():
    pl = _planner(StubBackend([np.array([3.0, 2.0, 1.0])]), 3, 10, 1.0)
    pl.optimize_policy()
    assert pl.num_gradient == 2 and pl.gradient_knots.shape == (2, 3, 2)


def test_sample_gradient_particle_reaches_goal():
    # the behavioural bar of test_sampling_particle_reaches_goal (sampling_planner_test.cc:44-115)
    from mujoco_mpc_b200.planner import SampleGradientPlanner
    m = get_model("particle")
    pl = SampleGradientPlanner(m, OracleBackend(m, threads=2), num_trajectory=16, horizon=11, num_gradient=4, gradient_filter=0.5)
    pl.reset()
    pl.set_state(np.zeros(4), 0.0, mocap_of(m))
    types = set()
    for _ in range(150):
        pl.optimize_policy()
        types.add(pl.winner_type)
        assert pl.improvement >= 0
    tr = pl.backend.fetch_trajectory(pl.winner)
    assert np.abs(tr["states"][-1, :2] - mocap_of(m)[:2]).max() < 0.1
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    assert (np.abs(tr["actions"]) <= cr[:, 1] + 1e-9).all()
    assert 1 in types


def test_cpp_planner_rejects_bad_sizes_at_create():
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import ModelBlob, load_library
    lib = load_library()
    m = get_model("particle")
    blob = to_blob(m)
    buf = ctypes.create_string_buffer(blob, len(blob))
    mb = ModelBlob(ctypes.cast(buf, ctypes.c_void_p), len(blob))
    cr = np.ascontiguousarray(np.asarray(m.actuator_ctrlrange, float).reshape(-1))
    for N, P in ((4, 1), (0, 3)):
        h = ctypes.c_void_p()
        rc = lib.mjpc_b200_sg_planner_create(ctypes.byref(mb), N, 1, P, 2, ctypes.c_double(0.1), ctypes.c_double(1.0),
                                             ctypes.c_double(0.01), cr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                             ctypes.c_uint32(1), 8, 0, ctypes.byref(h))
        assert rc == -1 and not h.value                                      # MJPC_B200_ERR_BAD_ARGUMENT
