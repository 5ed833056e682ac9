"""GPU: iLQG sweeps (FD model derivatives, cost derivatives, Riccati backward pass, feedback rollouts) vs the oracle.

Tolerances: fp32 finite differences need a much larger step than the reference's 1e-6 (fp64): with eps = 1e-3 the
truncation error is O(eps) and round-off O(1e-7/eps); the device result is compared with the fp64 oracle run at the
SAME eps (same secant), so what remains is fp32 round-off amplified by 1/eps ~ 1e-4 .. 1e-3 absolute on O(1) entries.
"""
import numpy as np
import pytest

from conftest import get_model, mocap_of, quadruped_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(oracle_lib):
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    build.build()
    out = {}
    for name in ("cartpole", "quadruped", "particle", "humanoid"):
        m = get_model(name)
        out[name] = (m, Engine(m, 64, 64), oracle_lib.Oracle(to_blob(m), m, 64))
    yield out
    for _, e, _ in out.values():
        e.close()


def _nominal(m, o, H, seed=0):
    """A nominal trajectory from the oracle (spline rollout of small random knots)."""
    from mujoco_mpc_b200.planner import candidate_knots
    P = 3
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    state = np.concatenate([m.key_qpos[0] if m.nkey else m.qpos0, np.zeros(m.nv)])
    kt = np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    knots = candidate_knots(np.zeros((P, m.nu)), 0.3, cr, seed, 2)[1:2]
    r = o.rollout_spline(state, 0.0, mocap_of(m), knots, kt, 2, H)
    return state, r["states"][0], r["actions"][0], r["times"][0], r["residual"][0]


def test_backward_pass_golden_on_device(ctx, oracle_lib):
    """backward_pass_test.cc:29-140 through the device kernel: the n=2, m=1 LQR embedded in the cartpole-sized
    problem (n=4, m=1) with two decoupled, cost-free extra states."""
    m, e, _ = ctx["cartpole"]
    H, n = 3, 4
    A = np.tile(np.eye(n), (H, 1, 1)); A[:, 0, 1] = 1.0
    B = np.zeros((H, n, 1)); B[:, 1, 0] = 1.0
    u = np.full((H, 1), 0.5); x = np.zeros((H, n))
    for t in range(H - 1):
        x[t + 1, :2] = [x[t, 0] + x[t, 1], x[t, 1] + u[t, 0]]
    cx = x.copy(); cu = u.copy(); cu[H - 1] = 0
    cxx = np.zeros((H, n, n)); cxx[:, 0, 0] = cxx[:, 1, 1] = 1.0
    cuu = np.ones((H, 1, 1)); cxu = np.zeros((H, n, 1))
    o = e.backward_pass(A, B, cx, cu, cxx, cxu, cuu, u, mu=0.0, reg_type=0, limits=1)
    assert o["status"] == 1
    np.testing.assert_allclose(o["Vx"][:, :2].ravel(), [0.0, 0.0, 0.5, 1.25, 0.5, 1.0], atol=1e-5)
    np.testing.assert_allclose(o["Vxx"][:, :2, :2].ravel(), [2.71428571, 2.0, 2.0, 4.0, 2.0, 1.0, 1.0, 2.5, 1.0, 0.0, 0.0, 1.0], atol=1e-5)
    np.testing.assert_allclose(o["K"][:2, 0, :2].ravel(), [-0.285714285, -1.0, 0.0, -0.5], atol=1e-5)
    np.testing.assert_allclose(o["du"][:2].ravel(), [-0.5, -0.75], atol=1e-5)
    assert np.abs(o["K"][:, :, 2:]).max() == 0 and np.abs(o["Vxx"][:, 2:, :]).max() == 0


def _column_stats(G, R, R_half):
    """Per (time step, perturbed coordinate) column: error relative to the column's own scale, and whether the fp64
    secant itself is stable when the step is halved (a column that moves by > 2 % sits on a contact / limit toggle:
    there the finite difference is not a derivative in ANY arithmetic and is excluded explicitly)."""
    colscale = np.abs(R).max(1) + 1.0
    return np.abs(G - R).max(1) / colscale, np.abs(R - R_half).max(1) / colscale < 0.02


@pytest.mark.parametrize("name,eps", [("cartpole", 1e-3), ("quadruped", 1e-3), ("humanoid", 1e-3)])
def test_model_derivatives(ctx, name, eps):
    """mjpc_b200_model_derivatives vs the fp64 oracle at the SAME step (same secant), column by column
    (model_derivatives.cc:76-104).  fp32 bounds: the state Jacobians A, B difference two constraint solves whose per-step
    error (teacher-forced bound: median 5e-6, p99 6e-4 in qvel) is divided by eps = 1e-3, so their smooth columns are
    held to median 2e-2 / p99 0.15 / max 0.3 of the column scale AND to 3x the error of the oracle's own fp32
    instantiation; the residual Jacobians C, D involve no solve: 1e-3.  Toggle columns are classified with the fp64
    oracle alone (step halving) and must stay below 20 % of the columns."""
    from mujoco_mpc_b200.blob import to_blob
    from oracle import pyoracle
    m, e, o = ctx[name]
    H = 8
    state, xs, us, ts, res = _nominal(m, o, H)
    G = e.model_derivatives(xs, us, ts, mocap_of(m), eps)
    R = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, nthreads=8)
    Rh = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps / 2, nthreads=8)
    F = pyoracle.Oracle(to_blob(m), m, 32).model_derivatives(xs, us, ts, mocap_of(m), tol=eps, nthreads=8)
    A, B, C, D = G
    assert np.abs(A[-1]).max() == 0 and np.abs(B[-1]).max() == 0 and np.abs(D[-1]).max() == 0   # last step: only C
    contact = name in ("quadruped", "humanoid")
    for k, nm in enumerate("ABCD"):
        err, smooth = _column_stats(G[k], R[k], Rh[k])
        err32, _ = _column_stats(F[k], R[k], Rh[k])
        assert np.isfinite(G[k]).all()
        assert smooth.mean() >= (0.8 if contact else 1.0), (nm, smooth.mean())
        es, es32 = err[smooth], err32[smooth]
        print(name, nm, "columns %d, smooth %.1f %%; device err / column scale: median %.2e p99 %.2e max %.2e | fp32 oracle %.2e %.2e %.2e"
              % (smooth.size, 100 * smooth.mean(), np.median(es), np.percentile(es, 99), es.max(), np.median(es32), np.percentile(es32, 99), es32.max()))
        if nm in "CD" or not contact:
            assert es.max() < 2e-3, (nm, es.max())
        else:
            assert np.median(es) < 2e-2 and np.percentile(es, 99) < 0.15 and es.max() < 0.3
            assert np.median(es) < 3 * np.median(es32) + 1e-3 and np.percentile(es, 99) < 3 * np.percentile(es32, 99) + 1e-3
        # toggle columns: bounded by the column scale (no blow-up), nothing tighter is defined there
        if (~smooth).any():
            assert err[~smooth].max() < 2.0


@pytest.mark.parametrize("name", ["cartpole", "particle"])
def test_model_derivatives_skip_and_centred(ctx, name):
    """derivative_skip + linear interpolation (model_derivatives.cc:56-72,109-164) and fd_mode centred
    (ilqg/settings.h:24) against the oracle on the smooth models, plus the structure of the skip path on the device:
    evaluated steps equal the skip = 0 result bit for bit, skipped steps are the exact linear blend of their neighbours."""
    m, e, o = ctx[name]
    H, eps = 24, 1e-3
    state, xs, us, ts, res = _nominal(m, o, H)
    full = e.model_derivatives(xs, us, ts, mocap_of(m), eps)
    for skip in (1, 3, 5):
        G = e.model_derivatives(xs, us, ts, mocap_of(m), eps, skip=skip)
        R = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, skip=skip)
        s = skip + 1
        ev = sorted(set([0] + list(range(s, H - s, s)) + [H - 2, H - 1]))
        for k in range(4):
            np.testing.assert_array_equal(G[k][ev], full[k][ev])
            scale = np.abs(R[k]).max() + 1.0     # (the particle's slide limits toggle along the trajectory: 6e-3)
            assert np.abs(G[k] - R[k]).max() < 6e-3 * scale, (skip, "ABCD"[k])
        for t in range(H):
            if t in ev:
                continue
            e0 = max(x for x in ev if x < t); e1 = min(x for x in ev if x > t)
            w = np.float32((t - e0) / (e1 - e0))
            np.testing.assert_allclose(G[0][t], (1 - w) * full[0][e0] + w * full[0][e1], rtol=0, atol=1e-6 * (np.abs(full[0]).max() + 1))
    Gc = e.model_derivatives(xs, us, ts, mocap_of(m), eps, mode=1)
    Rc = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, mode=1)
    R1 = o.model_derivatives(xs, us, ts, mocap_of(m), tol=1e-6, mode=1)          # (nearly) the exact derivative
    for k in range(4):
        scale = np.abs(Rc[k]).max() + 1.0
        assert np.abs(Gc[k] - Rc[k]).max() < 6e-3 * scale, "ABCD"[k]
    # centred differences cancel the O(eps) truncation error of the one-sided secant (cartpole is nonlinear)
    if name == "cartpole":
        assert np.abs(Rc[0] - R1[0]).max() < 0.2 * np.abs(o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps)[0] - R1[0]).max() + 1e-9


def test_model_derivatives_centred_contact(ctx):
    """Centred mode on the quadruped (contacts): same column-wise bar as the one-sided test."""
    m, e, o = ctx["quadruped"]
    H, eps = 6, 1e-3
    state, xs, us, ts, res = _nominal(m, o, H)
    G = e.model_derivatives(xs, us, ts, mocap_of(m), eps, mode=1)
    R = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, mode=1, nthreads=8)
    Rh = o.model_derivatives(xs, us, ts, mocap_of(m), tol=eps / 2, mode=1, nthreads=8)
    for k, nm in enumerate("ABCD"):
        err, smooth = _column_stats(G[k], R[k], Rh[k])
        assert smooth.mean() >= 0.8
        es = err[smooth]
        if nm in "CD":
            assert es.max() < 2e-3
        else:
            assert np.median(es) < 2e-2 and np.percentile(es, 99) < 0.15 and es.max() < 0.3


def test_differentiable_model_matches_oracle(ctx):
    """MakeDifferentiable (utilities.cc:60-75; agent.cc:296-309): solimp[0] = 0 for joints and geoms on both sides -
    teacher-forced single steps agree to the fp32 per-step bound, and the switch really changes the dynamics."""
    m, e, o = ctx["quadruped"]
    state, xs, us, ts, res = _nominal(m, o, 24)
    q, v = xs[:-1, : m.nq], xs[:-1, m.nq:]
    plain = e.step_batch(q, v, us[:-1], mocap_of(m), ts[:-1])
    try:
        e.set_differentiable(True); o.set_differentiable(True)
        g = e.step_batch(q, v, us[:-1], mocap_of(m), ts[:-1])
        r = o.step_batch(q, v, us[:-1], mocap_of(m), ts[:-1], nthreads=4)
    finally:
        e.set_differentiable(False); o.set_differentiable(False)
    assert (g["nefc"] == r["nefc"]).all()
    err = np.abs(g["next_qvel"] - r["next_qvel"]).max(1)
    assert np.median(err) < 2e-5 and err.max() < 5e-3
    incontact = r["ncon"] > 0
    assert incontact.any() and np.abs(g["next_qvel"] - plain["next_qvel"])[incontact].max() > 1e-4
    back = e.step_batch(q, v, us[:-1], mocap_of(m), ts[:-1])          # restored: bit-identical to before the switch
    np.testing.assert_array_equal(back["next_qvel"], plain["next_qvel"])


@pytest.mark.parametrize("name", ["cartpole", "quadruped", "particle", "humanoid"])
def test_cost_derivatives(ctx, name):
    m, e, o = ctx[name]
    H = 8
    state, xs, us, ts, res = _nominal(m, o, H)
    Ao, Bo, Co, Do = o.model_derivatives(xs, us, ts, mocap_of(m), tol=1e-6)
    g = e.cost_derivatives(res, Co, Do)
    r = o.cost_derivatives(res, Co, Do)
    for G, R in zip(g, r):
        np.testing.assert_allclose(G, R, rtol=2e-4, atol=2e-5 * (np.abs(R).max() + 1e-6))


def test_backward_pass_vs_oracle(ctx, oracle_lib):
    m, e, o = ctx["quadruped"]
    H = 16
    state, xs, us, ts, res = _nominal(m, o, H)
    A, B, C, D = o.model_derivatives(xs, us, ts, mocap_of(m), tol=1e-6)
    cx, cu, cxx, cuu, cxu = o.cost_derivatives(res, C, D)
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    for reg_type, mu, limits in ((0, 1.0, 1), (1, 0.5, 1), (2, 0.1, 0), (0, 10.0, 0)):
        g = e.backward_pass(A, B, cx, cu, cxx, cxu, cuu, us, mu=mu, reg_type=reg_type, limits=limits)
        r = oracle_lib.backward_pass(A, B, cx, cu, cxx, cxu, cuu, us, cr, mu=mu, reg_type=reg_type, limits=limits)
        assert g["status"] == r["status"] == 1
        for k in ("du", "K", "Vx"):
            scale = np.abs(r[k]).max() + 1e-6
            assert np.abs(g[k] - r[k]).max() < 5e-3 * scale, (reg_type, k, np.abs(g[k] - r[k]).max(), scale)
        np.testing.assert_allclose(g["dV"], r["dV"], rtol=5e-3, atol=1e-6)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_feedback_rollouts(ctx, oracle_lib, mode):
    """FeedbackRollouts (time-indexed, 3 interpolations) and ActionRollouts (step-indexed) vs the oracle."""
    m, e, o = ctx["quadruped"]
    H = 24
    state, xs, us, ts, res = _nominal(m, o, H, seed=3)
    rng = np.random.default_rng(5)
    K = rng.normal(size=(H, m.nu, 2 * m.nv)) * 0.05
    du = rng.normal(size=(H, m.nu)) * 0.05
    steps = np.array([1.0, 0.3, 0.1, 0.0])
    ret, fail, order = e.rollout_feedback(state, 0.0, mocap_of(m), us, xs, ts, K, du, steps, mode)
    r = o.rollout_feedback(state, 0.0, mocap_of(m), us, xs, ts, K, du, steps, mode)
    assert not fail.any() and not r["failure"].any()
    np.testing.assert_allclose(ret, r["returns"], rtol=2e-3)
    tr = e.fetch_all()
    np.testing.assert_allclose(tr["actions"][:, :4], r["actions"][:, :4], atol=2e-4)
    # step 0 with zero gains reproduces the nominal rollout itself
    ret0, _, _ = e.rollout_feedback(state, 0.0, mocap_of(m), us, xs, ts, 0 * K, 0 * du, np.array([0.0]), 3)
    nominal_return = o.rollout_feedback(state, 0.0, mocap_of(m), us, xs, ts, 0 * K, 0 * du, np.array([0.0]), 3)["returns"][0]
    np.testing.assert_allclose(ret0[0], nominal_return, rtol=2e-3)


def test_ilqg_planner_on_device(ctx):
    """ilqg_test.cc:49-126 with every sweep on the device (fp32 finite differences need eps ~ 1e-3)."""
    from mujoco_mpc_b200.ilqg import ILQGPlanner
    m, e, _ = ctx["particle"]
    pl = ILQGPlanner(m, e, horizon=26, fd_tolerance=1e-3)
    pl.set_state(np.zeros(4), 0.0, mocap_of(m))
    for _ in range(25):
        pl.optimize_policy()
    goal = mocap_of(m)[:2]
    assert abs(pl.states[-1, 0] - goal[0]) < 1e-2 and abs(pl.states[-1, 1] - goal[1]) < 1e-2
    assert abs(pl.states[-1, 2]) < 0.1 and abs(pl.states[-1, 3]) < 0.1


def test_ilqg_quadruped_iteration_improves(ctx):
    """BASELINE config 4 (Quadruped, iLQG, H=64, MakeDifferentiable on): the planner must actually descend.  With the
    engine's FD settings (centred, 3e-4; csrc/host/ilqg_planner.h) eight iterations from the home keyframe take the
    return from 0.324 to 0.124 on the device; the fp64 oracle with the reference's own settings (1e-6, one-sided) reaches
    0.115.  One-sided 1e-3 - the round-1 setting - does not improve it at all: the
    perturbation crosses contact kinks and the gradient is noise (profiles/fd_gradient_check.py)."""
    from mujoco_mpc_b200.ilqg import ILQGPlanner
    m, e, _ = ctx["quadruped"]
    pl = ILQGPlanner(m, e, horizon=64, num_rollouts=10, fd_tolerance=3e-4, fd_mode=1)
    pl.set_state(np.concatenate([m.key_qpos[0], np.zeros(m.nv)]), 0.0, mocap_of(m))
    pl.nominal_trajectory()
    first = pl.cand["total_return"]          # candidate_policy[0]: the live policy is only published by an Iteration
    ok, rets = 0, []
    for _ in range(8):
        ok += bool(pl.optimize_policy()); rets.append(pl.total_return)
    print("iLQG quadruped returns:", first, "->", np.round(rets, 5))
    assert ok >= 6 and np.isfinite(pl.total_return)
    assert all(b <= a * (1 + 1e-6) for a, b in zip([first] + rets, rets))      # never worse than the nominal (line search includes step 0)
    assert pl.total_return < 0.75 * first                                          # measured 0.38 x first
    assert (np.abs(pl.actions) <= 1.0 + 1e-6).all()


def test_cpp_ilqg_quadruped_descends_with_default_settings():
    """the C++ planner with its own defaults (centred 3e-4) on the same problem"""
    from mujoco_mpc_b200.engine import CppILQGPlanner
    m = get_model("quadruped")
    pl = CppILQGPlanner(m, 64, num_rollouts=10, representation=1)
    pl.reset()
    pl.set_state(np.concatenate([m.key_qpos[0], np.zeros(m.nv)]), 0.0, mocap_of(m))
    rets = []
    for _ in range(8):
        pl.optimize_policy(); rets.append(pl.result()["total_return"])
    print("C++ iLQG quadruped returns:", np.round(rets, 5))
    assert rets[-1] < 0.75 * rets[0] or rets[-1] < 0.25
    pl.close()


def test_ilqg_humanoid_iteration_improves(ctx):
    """iLQG on the humanoid (Stand task, nv = 27, pyramidal cones, tendon limits) through the generic FD kernels."""
    from mujoco_mpc_b200.ilqg import ILQGPlanner
    m, e, _ = ctx["humanoid"]
    pl = ILQGPlanner(m, e, horizon=24, num_rollouts=10, fd_tolerance=3e-4, fd_mode=1)
    pl.set_state(np.concatenate([m.qpos0, np.zeros(m.nv)]), 0.0, mocap_of(m))
    pl.nominal_trajectory()
    first = pl.cand["total_return"]
    ok = 0
    for _ in range(5):
        ok += bool(pl.optimize_policy())
    assert ok >= 2 and np.isfinite(pl.total_return) and pl.total_return <= first
    assert (np.abs(pl.actions) <= 1.0 + 1e-6).all()


def test_cpp_ilqg_planner_matches_python_mirror(ctx):
    """The C++ iLQGPlanner (csrc/host/ilqg_planner.cc) and the Python mirror drive the same sweeps through the same
    ABI: identical nominal trajectories, returns and regularisation schedule over several planning iterations."""
    from mujoco_mpc_b200.engine import CppILQGPlanner, Engine
    from mujoco_mpc_b200.ilqg import ILQGPlanner
    m = get_model("quadruped")
    H = 32
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    cpp = CppILQGPlanner(m, H, num_rollouts=10, representation=1, fd_tolerance=3e-4, fd_mode=1)
    e = Engine(m, 16, H)
    py = ILQGPlanner(m, e, horizon=H, num_rollouts=10, fd_tolerance=3e-4, representation=1, fd_mode=1)
    cpp.reset(); cpp.set_state(state, 0.0, mocap_of(m)); py.set_state(state, 0.0, mocap_of(m))
    for it in range(4):
        ok_c = cpp.optimize_policy()
        ok_p = py.optimize_policy()
        r = cpp.result()
        assert bool(ok_c) == bool(ok_p), it
        np.testing.assert_allclose(r["total_return"], py.total_return, rtol=1e-6)
        np.testing.assert_allclose(r["regularization"], py.regularization, rtol=1e-12)
        np.testing.assert_allclose(r["actions"], py.actions, atol=1e-6)
        np.testing.assert_allclose(r["states"], py.states, atol=1e-5)
        if ok_c:
            assert r["winner"] == py.winner
            np.testing.assert_allclose(r["surprise"], py.surprise, rtol=1e-4, atol=1e-6)
    a = cpp.action_from_policy(0.055)
    assert a.shape == (m.nu,) and np.isfinite(a).all() and (np.abs(a) <= 1 + 1e-6).all()
    cpp.close(); e.close()
