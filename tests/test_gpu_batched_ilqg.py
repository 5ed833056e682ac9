"""GPU: several independent iLQG problems per launch (mjpc_b200_*_batched sweeps) and the batched iLQG planner.  The
reference for a batch is each problem run alone through the single-problem entry point after set_task with that
problem's snapshot: every output must be BITWISE equal."""
import numpy as np
import pytest

from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

TIMES = np.array([0.0, 0.13, 0.5, 1.7])
ARRAYS = ("states", "actions", "times", "residual", "costs", "trace")


def _problems(m, H, B=4):
    """B distinct problems (start state, absolute start time, mocap goal, weights, parameters, task state) and a
    nominal trajectory of each: the rollout of one small random spline from its own start."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.engine import Engine
    from mujoco_mpc_b200.planner import candidate_knots
    rng = np.random.default_rng(5)
    times = TIMES[:B]
    quad = "residual_Amplitude" in m.task_parameter_names
    base = np.concatenate([m.key_qpos[0] if m.nkey else m.qpos0, np.zeros(m.nv)])
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    P = 3
    kt = np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    states, mocaps, weights, params, tstates, knots = [], [], [], [], [], []
    for b in range(B):
        s = base.copy()
        s[m.nq:] += 0.05 * b * rng.standard_normal(m.nv)
        mc = mocap_of(m).copy().reshape(-1, 7)
        mc[:, :3] += 0.02 * b * rng.standard_normal((len(mc), 3))
        w = np.asarray(m.task_weight, float) * (1.0 + 0.3 * b)
        p = np.asarray(m.task_parameters, float).copy()
        ts = np.asarray(m.task_state, float).copy()
        if quad:                                            # gait / mode clocks (absolute), gait amplitude
            p[m.task_parameter_names.index("residual_Amplitude")] += 0.02 * b
            ts[T.QS_MODE_START_TIME] = times[b] - 0.05 * b
            ts[T.QS_PHASE_START_TIME] = times[b] - 0.03 * b
        elif len(p):
            p = p * (1.0 + 0.1 * b)
        knots.append(candidate_knots(np.zeros((P, m.nu)), 0.1, cr, b, 2, seed=17)[1:2])
        states.append(s); mocaps.append(mc.reshape(-1)); weights.append(w); params.append(p); tstates.append(ts)
    pr = dict(states=np.stack(states), times=times, mocaps=np.stack(mocaps), weights=np.stack(weights),
              parameters=np.stack(params), task_states=np.stack(tstates))
    e = Engine(m, B, H)
    e.rollout_spline_batched(pr["states"], times, pr["mocaps"], np.stack(knots), np.stack([kt + t for t in times]), 2, H,
                             weights=pr["weights"], parameters=pr["parameters"], task_states=pr["task_states"])
    tr = e.fetch_all()
    e.close()
    pr.update(x=tr["states"], u=tr["actions"], t=tr["times"], residual=tr["residual"])
    return pr


def _set_task(e, pr, b):
    e.set_task(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])


def _task(pr):
    return dict(weights=pr["weights"], parameters=pr["parameters"], task_states=pr["task_states"])


def _derivs(e, pr, tol=1e-3, skip=0, mode=0):
    return e.model_derivatives_batched(pr["x"], pr["u"], pr["t"], pr["mocaps"], tol, skip=skip, mode=mode, **_task(pr))


def _assert_same(batch, single, b, what):
    for k, (x, y) in enumerate(zip(batch, single)):
        np.testing.assert_array_equal(x[b], y, err_msg=f"problem {b}: {what}[{k}]")


@pytest.mark.parametrize("name,kernel", [("quadruped", "static"), ("quadruped", "generic"), ("cartpole", "generic")])
@pytest.mark.parametrize("mode,skip", [(0, 0), (1, 0), (1, 2), (0, 2)])
def test_derivative_sweep_equals_single_sweeps(name, kernel, mode, skip, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    if kernel == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model(name)
    H = 16
    pr = _problems(m, H)
    e = Engine(m, 8, H)
    batch = _derivs(e, pr, skip=skip, mode=mode)
    assert np.abs(batch[0][0] - batch[0][1]).max() > 0          # the problems do differ
    for b in range(4):
        _set_task(e, pr, b)
        single = e.model_derivatives(pr["x"][b], pr["u"][b], pr["t"][b], pr["mocaps"][b], 1e-3, skip=skip, mode=mode)
        _assert_same(batch, single, b, "ABCD")
    e.close()


@pytest.mark.parametrize("name", ["quadruped", "cartpole"])
def test_cost_derivatives_equal_single_calls(name):
    from mujoco_mpc_b200.engine import Engine
    m = get_model(name)
    H = 16
    pr = _problems(m, H)
    e = Engine(m, 8, H)
    _, _, Cm, D = _derivs(e, pr)
    batch = e.cost_derivatives_batched(pr["residual"], Cm, D, weights=pr["weights"])
    for b in range(4):
        _set_task(e, pr, b)
        _assert_same(batch, e.cost_derivatives(pr["residual"][b], Cm[b], D[b]), b, "cost")
    # NULL weights: the handle's
    _set_task(e, pr, 2)
    implicit = e.cost_derivatives_batched(pr["residual"], Cm, D)
    explicit = e.cost_derivatives_batched(pr["residual"], Cm, D, weights=np.tile(pr["weights"][2], (4, 1)))
    for x, y in zip(implicit, explicit):
        np.testing.assert_array_equal(x, y)
    e.close()


def _lq(e, pr):
    A, B, Cm, D = _derivs(e, pr)
    cx, cu, cxx, cuu, cxu = e.cost_derivatives_batched(pr["residual"], Cm, D, weights=pr["weights"])
    return dict(A=A, B=B, cx=cx, cu=cu, cxx=cxx, cxu=cxu, cuu=cuu, actions=pr["u"])


@pytest.mark.parametrize("reg_type", [0, 1, 2, 3])
@pytest.mark.parametrize("limits", [0, 1])
def test_backward_pass_equals_single_calls(reg_type, limits):
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    H = 16
    pr = _problems(m, H)
    e = Engine(m, 8, H)
    lq = _lq(e, pr)
    mu = np.array([1e-3, 0.5, 1.0, 4.0], np.float32)
    # problem 3 is built to fail: cuu = -I with mu = 0 and no limits is not positive definite
    if not limits:
        lq["cuu"][3] = -np.eye(m.nu); mu[3] = 0.0
    batch = e.backward_pass_batched(**lq, mu=mu, reg_type=reg_type, limits=limits)
    keys = ("K", "du", "dV", "Vx", "Vxx")
    for b in range(4):
        s = e.backward_pass(*[lq[k][b] for k in ("A", "B", "cx", "cu", "cxx", "cxu", "cuu", "actions")], mu=float(mu[b]),
                            reg_type=reg_type, limits=limits)
        assert batch["status"][b] == s["status"], b
        if s["status"] == 1:
            for k in keys:
                np.testing.assert_array_equal(batch[k][b], s[k], err_msg=f"problem {b}: {k}")
        else:
            np.testing.assert_array_equal(batch["dV"][b], s["dV"], err_msg=f"problem {b}: dV")
    if not limits:
        assert batch["status"][3] == 0
    assert batch["status"][:3].all()
    e.close()


def _feedback_inputs(m, pr, K, with_du):
    rng = np.random.default_rng(3)
    Bn, H = pr["u"].shape[:2]
    gains = 0.01 * rng.standard_normal((Bn, H, m.nu, 2 * m.nv))
    du = 0.05 * rng.standard_normal((Bn, H, m.nu)) if with_du else None
    steps = np.stack([np.concatenate([np.logspace(0, -3, K - 1) * (1 + 0.1 * b), [0.0]]) for b in range(Bn)])
    return gains, du, steps


def _fb_batched(e, pr, gains, du, steps, mode):
    ret, fail, order = e.rollout_feedback_batched(pr["states"], pr["times"], pr["mocaps"], pr["u"], pr["x"], pr["t"], gains,
                                                  du, steps, mode, **_task(pr))
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _fb_single(e, pr, b, gains, du, steps, mode):
    _set_task(e, pr, b)
    ret, fail, order = e.rollout_feedback(pr["states"][b], pr["times"][b], pr["mocaps"][b], pr["u"][b], pr["x"][b], pr["t"][b],
                                          gains[b], None if du is None else du[b], steps[b], mode)
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _assert_fb_equal(batch, single, b, K):
    for k in ("returns", "failure", "order"):
        np.testing.assert_array_equal(batch[k][b], single[k], err_msg=f"problem {b}: {k}")
    for k in ARRAYS:
        np.testing.assert_array_equal(batch[k][b * K:(b + 1) * K], single[k], err_msg=f"problem {b}: {k}")


@pytest.mark.parametrize("shape", ["wide", "plain", "generic"])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("with_du", [False, True])
def test_feedback_rollouts_equal_single_launches(shape, mode, with_du, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    if shape == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    if shape == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model("quadruped")
    H, K = 16, 10
    pr = _problems(m, H)
    gains, du, steps = _feedback_inputs(m, pr, K, with_du)
    e = Engine(m, 4 * K, H)
    batch = _fb_batched(e, pr, gains, du, steps, mode)
    assert e.last_kernel_shape == {"wide": 1, "plain": 2, "generic": 0}[shape]
    assert not batch["failure"].any()
    assert np.abs(batch["returns"][0] - batch["returns"][1]).max() > 1e-5
    for b in range(4):
        _assert_fb_equal(batch, _fb_single(e, pr, b, gains, du, steps, mode), b, K)
    e.close()


def test_single_problem_batches_equal_single_entry_points():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    H, K = 16, 10
    pr = _problems(m, H)
    one = {k: v[:1] for k, v in pr.items()}
    e = Engine(m, K, H)
    _set_task(e, pr, 0)
    nt = dict(weights=None, parameters=None, task_states=None)
    D1 = e.model_derivatives_batched(one["x"], one["u"], one["t"], one["mocaps"], 1e-3, mode=1, **nt)
    D0 = e.model_derivatives(pr["x"][0], pr["u"][0], pr["t"][0], pr["mocaps"][0], 1e-3, mode=1)
    _assert_same(D1, D0, 0, "ABCD")
    c1 = e.cost_derivatives_batched(one["residual"], D1[2], D1[3])
    c0 = e.cost_derivatives(pr["residual"][0], D0[2], D0[3])
    _assert_same(c1, c0, 0, "cost")
    b1 = e.backward_pass_batched(D1[0], D1[1], c1[0], c1[1], c1[2], c1[4], c1[3], one["u"], mu=[0.5])
    b0 = e.backward_pass(D0[0], D0[1], c0[0], c0[1], c0[2], c0[4], c0[3], pr["u"][0], mu=0.5)
    for k in ("K", "du", "dV", "Vx", "Vxx"):
        np.testing.assert_array_equal(b1[k][0], b0[k], err_msg=k)
    assert b1["status"][0] == b0["status"] == 1
    gains, du, steps = _feedback_inputs(m, one, K, True)
    f1 = _fb_batched(e, dict(one, weights=None, parameters=None, task_states=None), gains, du, steps, 3)
    f0 = _fb_single(e, pr, 0, gains, du, steps, 3)
    _assert_fb_equal(f1, f0, 0, K)
    e.close()


def test_changing_one_problem_leaves_the_others_unchanged():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    H, K = 16, 10
    pr = _problems(m, H)
    gains, du, steps = _feedback_inputs(m, pr, K, True)
    e = Engine(m, 4 * K, H)

    def run(p, g, d, s, mu):
        out = {"derivs": _derivs(e, p, mode=1)}
        out["cost"] = e.cost_derivatives_batched(p["residual"], out["derivs"][2], out["derivs"][3], weights=p["weights"])
        A, B = out["derivs"][:2]
        cx, cu, cxx, cuu, cxu = out["cost"]
        out["bp"] = e.backward_pass_batched(A, B, cx, cu, cxx, cxu, cuu, p["u"], mu=mu)
        out["fb"] = _fb_batched(e, p, g, d, s, 3)
        return out

    mu = np.array([0.1, 0.2, 0.3, 0.4], np.float32)
    before = run(pr, gains, du, steps, mu)
    ch = {k: np.array(v, copy=True) for k, v in pr.items()}
    for k in ("x", "u", "residual"):
        ch[k][1] *= 1.01
    ch["t"][1] += 0.07; ch["times"][1] += 0.07
    ch["states"][1, m.nq:] += 0.2
    ch["mocaps"][1, :3] += 0.1
    ch["weights"][1] *= 2.0
    ch["parameters"][1, m.task_parameter_names.index("residual_Walk speed")] += 0.2
    ch["task_states"][1, 1] -= 0.2
    g2, d2, s2, mu2 = gains.copy(), du.copy(), steps.copy(), mu.copy()
    g2[1] *= 2; d2[1] *= -1; s2[1] *= 0.5; mu2[1] = 3.0
    after = run(ch, g2, d2, s2, mu2)
    assert np.abs(after["fb"]["returns"][1] - before["fb"]["returns"][1]).max() > 1e-5
    for b in (0, 2, 3):
        for x, y in zip(after["derivs"] + after["cost"], before["derivs"] + before["cost"]):
            np.testing.assert_array_equal(x[b], y[b])
        for k in ("K", "du", "dV", "Vx", "Vxx", "status"):
            np.testing.assert_array_equal(after["bp"][k][b], before["bp"][k][b], err_msg=k)
        for k in ("returns", "failure", "order"):
            np.testing.assert_array_equal(after["fb"][k][b], before["fb"][k][b], err_msg=k)
        for k in ARRAYS:
            np.testing.assert_array_equal(after["fb"][k][b * K:(b + 1) * K], before["fb"][k][b * K:(b + 1) * K], err_msg=k)
    e.close()


def test_batched_argument_errors_leave_the_handle_usable():
    from mujoco_mpc_b200.engine import Engine, EngineError
    m = get_model("quadruped")
    H, K = 16, 10
    pr = _problems(m, H)
    gains, du, steps = _feedback_inputs(m, pr, K, True)
    e = Engine(m, 4 * K, H)
    ref_d = _derivs(e, pr)
    ref_f = _fb_batched(e, pr, gains, du, steps, 3)
    cut = {k: v[:0] for k, v in pr.items()}
    with pytest.raises(EngineError, match="error -1"):                    # B = 0
        _derivs(e, cut)
    with pytest.raises(EngineError, match="error -1"):
        e.cost_derivatives_batched(pr["residual"][:0], ref_d[2][:0], ref_d[3][:0])
    with pytest.raises(EngineError, match="error -1"):
        _fb_batched(e, cut, gains[:0], du[:0], steps[:0], 3)
    with pytest.raises(EngineError, match="error -1"):                    # required NULL pointer
        e.model_derivatives_batched(pr["x"], None, pr["t"], pr["mocaps"], 1e-3)
    with pytest.raises(EngineError, match="error -1"):
        e.backward_pass_batched(ref_d[0], ref_d[1], None, None, None, None, None, pr["u"], mu=np.zeros(4))
    with pytest.raises(EngineError, match="error -3"):                    # B * K > max_candidates
        big = {k: np.concatenate([v, v[:1]]) for k, v in pr.items()}
        _fb_batched(e, big, np.concatenate([gains, gains[:1]]), np.concatenate([du, du[:1]]),
                    np.concatenate([steps, steps[:1]]), 3)
    with pytest.raises(EngineError, match="error -3"):                    # H > max_horizon
        long = dict(pr, x=np.concatenate([pr["x"], pr["x"][:, :1]], 1), u=np.concatenate([pr["u"], pr["u"][:, :1]], 1),
                    t=np.concatenate([pr["t"], pr["t"][:, -1:] + 0.01], 1))
        _derivs(e, long)
    again_d = _derivs(e, pr)
    again_f = _fb_batched(e, pr, gains, du, steps, 3)
    for x, y in zip(ref_d, again_d):
        np.testing.assert_array_equal(x, y)
    for k in ref_f:
        np.testing.assert_array_equal(ref_f[k], again_f[k], err_msg=k)
    e.close()


def test_unsupported_warps_per_cta_batch(monkeypatch):
    from mujoco_mpc_b200.engine import Engine, EngineError
    m = get_model("cartpole")
    H, K = 16, 10
    pr = _problems(m, H)
    gains, du, steps = _feedback_inputs(m, pr, K, True)
    monkeypatch.setenv("MJPC_B200_WARPS_PER_CTA", "4")          # read at create: four candidates per CTA
    e = Engine(m, 4 * K, H)
    with pytest.raises(EngineError, match="error -5"):          # K = 10 would put two problems in one CTA
        _fb_batched(e, pr, gains, du, steps, 3)
    g8, d8, s8 = _feedback_inputs(m, pr, 8, True)
    ret = _fb_batched(e, pr, g8, d8, s8, 3)["returns"]
    assert ret.shape == (4, 8) and np.isfinite(ret).all()
    e.close()


@pytest.mark.parametrize("name,B,H,iters", [("quadruped", 3, 32, 5), ("humanoid", 2, 12, 2)])
def test_batch_ilqg_planner_equals_independent_planners(name, B, H, iters):
    """CppBatchILQGPlanner (one launch per sweep) vs one CppILQGPlanner per problem (its own launches)."""
    from mujoco_mpc_b200.engine import CppBatchILQGPlanner, CppILQGPlanner
    m = get_model(name)
    pr = _problems(m, H, B=B)
    batch = CppBatchILQGPlanner(m, B, H, num_rollouts=10, representation=1)
    singles = [CppILQGPlanner(m, H, num_rollouts=10, representation=1) for _ in range(B)]
    for b in range(B):
        batch.reset(b); singles[b].reset()
    updated_any = 0
    for it in range(iters):
        for b in range(B):
            t = pr["times"][b] + 0.01 * it
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
            singles[b].set_state(pr["states"][b], t, pr["mocaps"][b])
        up = batch.optimize_policy()
        for b in range(B):
            ok = singles[b].optimize_policy()
            assert up[b] == ok, (it, b)
            updated_any += ok
            r, s = batch.result(b), singles[b].result()
            for k in ("total_return", "regularization", "improvement", "expected", "surprise", "winner"):
                assert r[k] == s[k], (it, b, k)
            for k in ("states", "actions", "times"):
                np.testing.assert_array_equal(r[k], s[k], err_msg=f"iteration {it} problem {b}: {k}")
            tq = pr["times"][b] + 0.01 * it + 0.02
            np.testing.assert_array_equal(batch.action_from_policy(b, tq, pr["states"][b]),
                                          singles[b].action_from_policy(tq, pr["states"][b]))
    assert updated_any > 0
    with pytest.raises(Exception):
        batch.set_state(B, pr["states"][0], 0.0, pr["mocaps"][0])
    batch.close()
    for s in singles:
        s.close()


def test_batch_ilqg_planner_particles_reach_their_goals():
    """ilqg_test.cc's bar on a batch: four particles with different goals, planned together, each reach their own."""
    from mujoco_mpc_b200.engine import CppBatchILQGPlanner
    m = get_model("particle")
    H, B = 26, 4
    goals = [(0.1, 0.1), (-0.1, 0.05), (0.05, -0.1), (-0.08, -0.08)]
    pl = CppBatchILQGPlanner(m, B, H, num_rollouts=10, representation=1, fd_tolerance=1e-3, fd_mode=0)
    for b, g in enumerate(goals):
        mc = mocap_of(m).copy(); mc[:2] = g
        pl.reset(b); pl.set_state(b, np.zeros(4), 0.0, mc)
    for _ in range(30):
        pl.optimize_policy()
    for b, g in enumerate(goals):
        st = pl.result(b)["states"]
        assert np.abs(st[-1, :2] - np.asarray(g)).max() < 1e-2, (b, st[-1])
    pl.close()
