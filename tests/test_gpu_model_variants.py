"""GPU: per-problem model variants (mjpc_b200_set_model_variants, the batch planners' and filter banks' set_models).

A variant is a model compiled from its own MJCF text that differs from the handle's model only in physical parameters.
The reference for problem b of a batch with variants is a handle, planner or filter built from variant b alone: every
output must be BITWISE equal.  The closed-form and fp64-oracle tests show that each variant's own parameters take
effect, and the refusal tests that a variant of another structure, option, task or ctrlrange is refused and leaves the
handle as it was."""
import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_batched import _problems

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, UNSUPPORTED = -1, -5
SEEDS = [0x5EED, 7, 123456, 99]
XML = {"quadruped": "quadruped_flat_xml", "humanoid_track": "humanoid_track_xml", "particle": "particle_xml"}


def _variant(name, edit):
    """models.load(name) with its MJCF text passed through edit first."""
    from mujoco_mpc_b200 import models
    fn = XML[name]
    orig = getattr(models, fn)
    setattr(models, fn, lambda *a, **k: edit(orig(*a, **k)))
    try:
        return models.load(name)
    finally:
        setattr(models, fn, orig)


def _sub(text, old, new):
    assert old in text, old
    return text.replace(old, new)


def _quadruped_variant(k):
    """Variant k of the Quadruped: trunk mass, foot friction, actuator gain, joint damping and armature all differ."""
    def edit(x):
        x = _sub(x, '<inertial mass="4.713"', f'<inertial mass="{4.713 * (1 + 0.15 * k):g}"')
        x = _sub(x, 'friction="0.8 0.02 0.01"', f'friction="{0.8 + 0.1 * k:g} 0.02 0.01"')
        x = _sub(x, 'gainprm="40"', f'gainprm="{40 + 3 * k:g}"')
        return _sub(x, 'damping="2" armature="0.01"', f'damping="{2 + 0.5 * k:g}" armature="{0.01 * (1 + 0.5 * k):g}"')
    return _variant("quadruped", edit)


def _track_variant(k):
    """Variant k of the Humanoid Track: torso mass, geom friction, motor gears, joint damping and armature differ."""
    def edit(x):
        x = _sub(x, '<geom name="torso" fromto="0 -.07 0 0 .07 0" size=".07"/>',
                 f'<geom name="torso" fromto="0 -.07 0 0 .07 0" size=".07" mass="{8.9 * (1 + 0.15 * k):g}"/>')
        x = _sub(x, 'condim="1" friction=".7"', f'condim="1" friction="{0.7 + 0.1 * k:g}"')
        x = _sub(x, 'gear="40"', f'gear="{40 + 4 * k:g}"')
        return _sub(x, 'damping=".2" stiffness="1" armature=".01"',
                    f'damping="{0.2 + 0.05 * k:g}" stiffness="1" armature="{0.01 * (1 + 0.5 * k):g}"')
    return _variant("humanoid_track", edit)


_CACHE = {}


def _variants(name, B=4):
    key = (name, B)
    if key not in _CACHE:
        make = _quadruped_variant if name == "quadruped" else _track_variant
        _CACHE[key] = [make(k) for k in range(B)]
    return _CACHE[key]


def _engine(m, N, H):
    from mujoco_mpc_b200.engine import Engine
    return Engine(m, N, H)


def _set_shape(shape, monkeypatch):
    if shape == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    elif shape == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")


def _spline(e, pr, H, sl=slice(None)):
    a = {k: v[sl] for k, v in pr.items()}
    ret, fail, order = e.rollout_spline_batched(a["states"], a["times"], a["mocaps"], a["knots"], a["knot_times"], 2, H,
                                                weights=a["weights"], parameters=a["parameters"],
                                                task_states=a["task_states"])
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _feedback_inputs(m, traj, pr, B, K, H):
    rng = np.random.default_rng(3)
    ds, n = m.nq + m.nv, 2 * m.nv
    x = traj["states"].reshape(B, -1, H, ds)[:, 0]
    u = traj["actions"].reshape(B, -1, H, m.nu)[:, 0]
    t = traj["times"].reshape(B, -1, H)[:, 0]
    gains = 0.01 * rng.standard_normal((B, H, m.nu, n))
    du = 0.02 * rng.standard_normal((B, H, m.nu))
    steps = np.tile(np.linspace(0.0, 1.0, K), (B, 1))
    return x, u, t, gains, du, steps


def _feedback(e, pr, fb, sl=slice(None)):
    x, u, t, gains, du, steps = (v[sl] for v in fb)
    ret, fail, order = e.rollout_feedback_batched(pr["states"][sl], pr["times"][sl], pr["mocaps"][sl], u, x, t, gains,
                                                  du, steps, 1, weights=pr["weights"][sl],
                                                  parameters=pr["parameters"][sl], task_states=pr["task_states"][sl])
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


def _derivatives(e, pr, fb, sl=slice(None)):
    x, u, t = fb[0][sl], fb[1][sl], fb[2][sl]
    kw = dict(weights=pr["weights"][sl], parameters=pr["parameters"][sl], task_states=pr["task_states"][sl])
    A, Bm, Cm, D = e.model_derivatives_batched(x, u, t, pr["mocaps"][sl], 3e-4, 0, 1, **kw)
    return dict(A=A, B=Bm, C=Cm, D=D), x, u, t, kw


def _sweeps(e, pr, fb, traj_res, sl=slice(None)):
    """model, cost and gradient sweeps and a backward pass of the problems in sl."""
    d, x, u, t, kw = _derivatives(e, pr, fb, sl)
    res = traj_res[sl]
    cx, cu, cxx, cuu, cxu = e.cost_derivatives_batched(res, d["C"], d["D"], weights=kw["weights"])
    bp = e.backward_pass_batched(d["A"], d["B"], cx, cu, cxx, cxu, cuu, u, 1e-6)
    k, dV0 = e.gradient_batched(x, u, t, pr["mocaps"][sl], res, 3e-4, 0, 1, **kw)
    return dict(d, cx=cx, cu=cu, cxx=cxx, cuu=cuu, cxu=cxu, k=k, dV0=dV0, **{"bp_" + n: v for n, v in bp.items()})


def _assert_equal(a, b, what):
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=f"{what}: {k}")


def _row(d, b, per):
    """problem b's rows of a flat-candidate result dict (per candidates per problem), or of a [B]-leading one"""
    out = {}
    for k, v in d.items():
        v = np.asarray(v)
        out[k] = v[b * per:(b + 1) * per] if k in ("states", "actions", "times", "residual", "costs", "trace") else v[b]
    return out


# ------------------------------------------------------------------------------------------ 1. bitwise per variant
@pytest.mark.parametrize("name,shape", [("quadruped", "wide"), ("quadruped", "plain"), ("quadruped", "generic"),
                                        ("humanoid_track", "wide"), ("humanoid_track", "plain"),
                                        ("humanoid_track", "generic")])
def test_every_sweep_equals_a_handle_per_variant(name, shape, monkeypatch):
    _set_shape(shape, monkeypatch)
    base, V = get_model(name), _variants(name)
    B, N, K, H = 4, 4, 3, 12
    pr = _problems(base, N, H, B=B)
    e = _engine(base, B * N, H)
    e.set_model_variants(V)
    spl = _spline(e, pr, H)
    fb = _feedback_inputs(base, spl, pr, B, K, H)
    fbk = _feedback(e, pr, fb)
    res = spl["residual"].reshape(B, N, H, -1)[:, 0]
    sw = _sweeps(e, pr, fb, res)
    e.close()
    for b in range(B):
        s = _engine(V[b], N, H)
        sl = slice(b, b + 1)
        _assert_equal(_row(spl, b, N), _row(_spline(s, pr, H, sl), 0, N), f"{name} {shape} spline problem {b}")
        _assert_equal(_row(fbk, b, K), _row(_feedback(s, pr, fb, sl), 0, K), f"{name} {shape} feedback problem {b}")
        _assert_equal({k: v[b] for k, v in sw.items()}, {k: v[0] for k, v in _sweeps(s, pr, fb, res, sl).items()},
                      f"{name} {shape} sweeps problem {b}")
        s.close()
    # the variants do differ, and a handle of the base model computes something else
    assert len({float(spl["returns"][b, 0]) for b in range(B)}) == B


def test_clearing_and_set_task_with_variants():
    """After clearing, a handle computes bitwise what a fresh one does; set_task moves a handle with variants exactly
    as it moves the per-variant handles."""
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 4, 4, 12
    pr = _problems(base, N, H, B=B)
    pr_h = {k: v for k, v in pr.items()}
    for k in ("weights", "parameters", "task_states"):
        pr_h[k] = None
    e = _engine(base, B * N, H)
    e.set_model_variants(V)
    w = np.asarray(base.task_weight, float) * 1.7
    e.set_task(weight=w)
    got = _spline_handle_task(e, pr, H)
    for b in range(B):
        s = _engine(V[b], N, H)
        s.set_task(weight=w)
        _assert_equal(_row(got, b, N), _row(_spline_handle_task(s, pr, H, slice(b, b + 1)), 0, N), f"set_task problem {b}")
        s.close()
    e.set_task(weight=np.asarray(base.task_weight, float))
    e.set_model_variants(None)
    fresh = _engine(base, B * N, H)
    _assert_equal(_spline(e, pr, H), _spline(fresh, pr, H), "cleared")
    e.close(); fresh.close()


def _spline_handle_task(e, pr, H, sl=slice(None)):
    """a spline launch that reads the handle's set_task values (no per-problem task rows)"""
    a = {k: v[sl] for k, v in pr.items()}
    ret, fail, order = e.rollout_spline_batched(a["states"], a["times"], a["mocaps"], a["knots"], a["knot_times"], 2, H)
    return dict(e.fetch_all(), returns=ret, failure=fail, order=order)


# ------------------------------------------------------------------------------------------ 2. every batch planner
def _planner_pair(kind, m, V, B, N, H, seeds):
    from mujoco_mpc_b200 import engine as E
    if kind == "sampling":
        return E.CppBatchSamplingPlanner(m, B, N, H, seeds=seeds), [E.CppSamplingPlanner(V[b], N, H, seed=seeds[b]) for b in range(B)]
    if kind == "ce":
        return E.CppBatchCrossEntropyPlanner(m, B, N, H, seeds=seeds), [E.CppCrossEntropyPlanner(V[b], N, H, seed=seeds[b]) for b in range(B)]
    if kind == "sg":
        kw = dict(num_gradient=4, gradient_filter=0.6)
        return (E.CppBatchSampleGradientPlanner(m, B, N, H, seeds=seeds, **kw),
                [E.CppSampleGradientPlanner(V[b], N, H, seed=seeds[b], **kw) for b in range(B)])
    if kind == "robust":
        kw = dict(ncandidates=3, nrepetitions=4, xfrc_std=1.0, xfrc_rate=0.1)
        return (E.CppBatchRobustPlanner(m, B, N, H, seeds=seeds, **kw),
                [E.CppRobustPlanner(V[b], N, H, seed=seeds[b], **kw) for b in range(B)])
    if kind == "gradient":
        return E.CppBatchGradientPlanner(m, B, H), [E.CppGradientPlanner(V[b], H) for b in range(B)]
    if kind == "ilqs":
        return (E.CppBatchILQSPlanner(m, B, H, seeds=seeds),
                [E.CppILQSPlanner(V[b], H, seed=seeds[b]) for b in range(B)])
    return E.CppBatchILQGPlanner(m, B, H, num_rollouts=4), [E.CppILQGPlanner(V[b], H, num_rollouts=4) for b in range(B)]


KINDS = ["sampling", "ce", "sg", "robust", "gradient", "ilqs", "ilqg"]


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_batch_planner_equals_a_planner_per_variant(kind, B):
    base, V = get_model("quadruped"), _variants("quadruped")[:B]
    N, H, iters = 8, 16, 3
    pr = _problems(base, 4, H, B=B)
    seeds = SEEDS[:B]
    batch, singles = _planner_pair(kind, base, V, B, N, H, seeds)
    batch.set_models(V)
    feedback = kind in ("ilqs", "ilqg")
    for b in range(B):
        batch.reset(b); singles[b].reset()
        task = dict(weight=pr["weights"][b], parameters=pr["parameters"][b], task_state=pr["task_states"][b])
        batch.set_task(b, **task); singles[b].set_task(**task)
    for it in range(iters):
        for b in range(B):
            t = pr["times"][b] + 0.01 * it
            batch.set_state(b, pr["states"][b], t, pr["mocaps"][b])
            singles[b].set_state(pr["states"][b], t, pr["mocaps"][b])
        got = batch.optimize_policy()
        for b in range(B):
            ref = singles[b].optimize_policy()
            if isinstance(ref, dict):
                _assert_equal(got[b], ref, f"{kind} iteration {it} problem {b}")
            else:
                assert int(np.asarray(got)[b]) == int(ref), f"{kind} iteration {it} problem {b}"
                a, r = batch.result(b), singles[b].result()     # (a batch result may carry more fields)
                _assert_equal({k: a[k] for k in r}, r, f"{kind} iteration {it} problem {b}")
            for dt in (0.0, 0.013, 0.05):
                tt = pr["times"][b] + 0.01 * it + dt
                if feedback:
                    a, r = batch.action_from_policy(b, tt, pr["states"][b]), singles[b].action_from_policy(tt, pr["states"][b])
                else:
                    a, r = batch.action_from_policy(b, tt), singles[b].action_from_policy(tt)
                np.testing.assert_array_equal(a, r, err_msg=f"{kind} iteration {it} problem {b} action")
    batch.close()
    for s in singles:
        s.close()


# ------------------------------------------------------------------------------------------ 3. filter bank
@pytest.mark.parametrize("kind", ["kalman", "unscented"])
def test_filter_bank_equals_a_filter_per_variant(kind):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from estimator_backends import mocap_vector
    from quadruped_filtering import plant
    from mujoco_mpc_b200.estimator import CppBatchEstimator, CppKalman, CppUnscented
    base, V = get_model("quadruped"), _variants("quadruped")
    X, Y, U = plant(base)
    B, T = 4, 10
    mc = mocap_vector(base)
    bank = CppBatchEstimator(base, kind, B)
    bank.set_models(V)
    singles = [(CppKalman if kind == "kalman" else CppUnscented)(V[b]) for b in range(B)]
    for b in range(B):
        bank.reset(b, state=X[0]); singles[b].reset(state=X[0])
    for t in range(T):
        st = bank.update(np.tile(U[t], (B, 1)), np.tile(Y[t], (B, 1)), np.tile(mc, (B, 1)))
        assert not st.any()
        for b in range(B):
            singles[b].update(U[t], Y[t], mc)
            x, P, tm, _ = bank.get(b)
            np.testing.assert_array_equal(x, singles[b].state, err_msg=f"{kind} update {t} filter {b}")
            np.testing.assert_array_equal(P, singles[b].covariance, err_msg=f"{kind} update {t} filter {b}")
    assert len({float(bank.state(b)[0]) for b in range(B)}) > 1
    bank.close()
    for s in singles:
        s.close()


# ------------------------------------------------------------------------------------------ 4. known physics
def _particle_variant(mass, damping):
    def edit(x):
        x = _sub(x, 'range="-.29 .29" damping="1"', f'range="-.29 .29" damping="{damping:g}"')
        return _sub(x, 'size=".01" mass=".3"', f'size=".01" mass="{mass:g}"')
    return _variant("particle", edit)


PARTICLES = [(0.3, 1.0), (0.2, 0.5), (0.5, 2.0), (0.8, 0.25)]


def test_particle_variants_follow_their_damped_euler_step():
    """Each variant's rollout is the implicit-damping Euler step of its own mass m and damping d:
    v' = v + h (u - d v) / (m + h d), q' = q + h v' (gear 1, no armature, no contact, away from the limits)."""
    base = get_model("particle")
    V = [_particle_variant(*p) for p in PARTICLES]
    B, H, h = len(V), 3, base.opt_timestep
    e = _engine(base, B, H)
    e.set_model_variants(V)
    u = np.array([0.3, -0.2])
    states = np.tile([0.0, 0.0, 0.05, -0.02], (B, 1))
    knots = np.tile(u, (B, 1, 2, 1))
    times = np.zeros(B)
    kt = np.tile([0.0, 1.0], (B, 1))
    mocaps = np.tile(mocap_of(base), (B, 1))
    e.rollout_spline_batched(states, times, mocaps, knots, kt, 0, H)
    got = e.fetch_all()["states"].reshape(B, H, 4)
    for b, (m, d) in enumerate(PARTICLES):
        q, v = states[b, :2].copy(), states[b, 2:].copy()
        for t in range(1, H):
            v = v + h * (u - d * v) / (m + h * d)
            q = q + h * v
            np.testing.assert_allclose(got[b, t], np.concatenate([q, v]), rtol=1e-5, atol=1e-7, err_msg=f"variant {b} step {t}")
    # the FD control Jacobian of the velocity: dv'/du = h / (m + h d), of the position h times that
    x = got.astype(np.float32)
    uu = np.tile(u, (B, H, 1))
    tt = np.tile(np.arange(H) * h, (B, 1))
    A, Bm, _, _ = e.model_derivatives_batched(x, uu, tt, mocaps, 1e-3, 0, 1)
    for b, (m, d) in enumerate(PARTICLES):
        g = h / (m + h * d)
        np.testing.assert_allclose(Bm[b, 0], np.array([[h * g, 0], [0, h * g], [g, 0], [0, g]]), rtol=2e-3, atol=1e-6,
                                   err_msg=f"variant {b}")
    e.close()


def test_quadruped_variants_match_their_own_fp64_oracle():
    """One launch of four Quadruped variants: each problem's return is within the smoke test's 1e-4 relative of the
    fp64 oracle of its own variant, and variants 1-3 miss the base model's oracle by more than that."""
    from conftest import quadruped_inputs
    from mujoco_mpc_b200.blob import to_blob
    from oracle import pyoracle
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 4, 8, 16
    state, mocap, knots, kt = quadruped_inputs(base, N=N, H=H)
    e = _engine(base, B * N, H)
    e.set_model_variants(V)
    ret, fail, _ = e.rollout_spline_batched(np.tile(state, (B, 1)), np.zeros(B), np.tile(mocap, (B, 1)),
                                            np.tile(knots, (B, 1, 1, 1)), np.tile(kt, (B, 1)), 2, H)
    assert not fail.any()
    ref0 = pyoracle.Oracle(to_blob(base), base, 64).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=2,
                                                                   full=False)["returns"]
    for b in range(B):
        ref = pyoracle.Oracle(to_blob(V[b]), V[b], 64).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=2,
                                                                      full=False)["returns"]
        assert (np.abs(ret[b] - ref) / np.abs(ref)).max() < 1e-4, b
        if b:
            assert (np.abs(ret[b] - ref0) / np.abs(ref0)).max() > 1e-4, b
    e.close()


# ------------------------------------------------------------------------------------------ 5. refusals
def _refusal_variants():
    return {
        "extra geom": _variant("quadruped", lambda x: _sub(x, '<site name="torso"/>',
                                                           '<site name="torso"/><geom class="collision" size="0.01" pos="0 0 0.1"/>')),
        "contype": _variant("quadruped", lambda x: _sub(x, '<geom name="floor" size="0 0 0.1"',
                                                        '<geom name="floor" contype="0" conaffinity="0" size="0 0 0.1"')),
        "frictionloss 0": _variant("quadruped", lambda x: _sub(x, 'frictionloss="0.2"', 'frictionloss="0"')),
        "timestep": _variant("quadruped", lambda x: _sub(x, '<numeric name="agent_timestep" data="0.01"/>',
                                                         '<numeric name="agent_timestep" data="0.012"/>')),
        "ctrlrange": _variant("quadruped", lambda x: _sub(x, 'gainprm="40" ctrllimited="true" ctrlrange="-1 1"',
                                                          'gainprm="40" ctrllimited="true" ctrlrange="-0.9 0.9"')),
    }


def test_refusals_leave_the_handle_usable_and_unchanged():
    from mujoco_mpc_b200.engine import EngineError
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 4, 4, 12
    pr = _problems(base, N, H, B=B)
    e, ref = _engine(base, B * N, H), _engine(base, B * N, H)
    want_plain = _spline(ref, pr, H)
    for what, v in _refusal_variants().items():
        with pytest.raises(EngineError, match="variant 2"):
            e.set_model_variants(V[:2] + [v] + V[3:])
        _assert_equal(_spline(e, pr, H), want_plain, f"after refusing {what}")
    ref.set_model_variants(V)
    want = _spline(ref, pr, H)
    e.set_model_variants(V)
    with pytest.raises(EngineError, match="variant 0"):
        e.set_model_variants([_refusal_variants()["ctrlrange"]] + V[1:])
    # launches of another B, and the calls without a problem index
    with pytest.raises(EngineError, match="model variants are for 4"):
        _spline(e, pr, H, slice(0, 3))
    x = np.tile(pr["states"][0], (H, 1)).astype(np.float32)
    u = np.zeros((H, base.nu), np.float32)
    calls = {
        "rollout_spline": lambda: e.rollout_spline(pr["states"][0], 0.0, pr["mocaps"][0], pr["knots"][0],
                                                   pr["knot_times"][0], 2, H),
        "rollout_spline_sharded": lambda: e.rollout_spline_sharded(pr["states"][0], 0.0, pr["mocaps"][0], pr["knots"][0],
                                                                   pr["knot_times"][0], 2, H),
        "step_debug": lambda: e.step_debug(x[0, :base.nq], x[0, base.nq:], u[0], pr["mocaps"][0]),
        "step_batch": lambda: e.step_batch(x[:2, :base.nq], x[:2, base.nq:], u[:2], pr["mocaps"][0], np.zeros(2)),
        "model_derivatives": lambda: e.model_derivatives(x, u, np.arange(H) * 0.01, pr["mocaps"][0], 3e-4),
    }
    for name, call in calls.items():
        with pytest.raises(EngineError, match=f"error -5: {name}: not available while model variants are set"):
            call()
    _assert_equal(_spline(e, pr, H), want, "after the refusals")
    e.close(); ref.close()


def test_batch_planner_set_models_refuses_a_wrong_count():
    from mujoco_mpc_b200.engine import CppBatchRobustPlanner, EngineError
    base, V = get_model("quadruped"), _variants("quadruped")
    pl = CppBatchRobustPlanner(base, 4, 10, 16)
    for models in (V[:2], V[:1]):
        with pytest.raises(EngineError):
            pl.set_models(models)
    with pytest.raises(EngineError, match="variant 1"):
        pl.set_models([V[0], _refusal_variants()["timestep"], V[2], V[3]])
    pl.set_models(V)
    pl.set_models([])
    pl.close()
