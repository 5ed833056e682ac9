"""GPU: the rollout's policy stage against the fp64 oracle - the spline (zero-order, linear, cubic) and the iLQG feedback
policy (time-indexed modes 0/1/2, step-indexed mode 3) - on the same float32-rounded knots and nominal arrays.

A spline action does not depend on the state, so the recorded actions are compared with the oracle's directly.  A
feedback action is compared with the oracle's policy evaluated at the device's own recorded state of that step and at
the fp64 rollout time, so dynamics drift can neither hide nor fake a policy error.

Bars: where the step holds one knot (zero-order, or before the first / after the last knot) the device action is
float32(clamp(knot)) bitwise; otherwise 1e-5 (1 + max |knot|) for the spline and 1e-5 (1 + max |u| + step G D) for the
feedback policy (G the largest gain row sum, D a bound on the state difference).  Recorded times are bitwise the
oracle's.  Knots land on steps where the planner spaces zero-order knots by horizon / P with H - 1 a multiple of P
(the Shadow spacing, P = 5 and H = 26, on particle, cartpole and Shadow), so a step that picks the neighbouring
interval moves an action by a whole knot difference, 0.1 or more here."""
import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_policy_intervals_cpu import agent_times, planner_knot_times

pytestmark = pytest.mark.gpu

RATIOS = {}


def note(group, ratio):
    RATIOS[group] = max(RATIOS.get(group, 0.0), float(ratio))


def ref_times(time0, dt, H):
    out, t = [], time0
    for _ in range(H):
        out.append(t)
        t += dt
    return np.array(out)


@pytest.fixture(scope="module")
def engines():
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import Engine
    build.build()
    cache = {}

    def get(name, N=512, H=80):
        key = (name, N, H)
        if key not in cache:
            cache[key] = Engine(get_model(name), N, H)
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.fixture(scope="module")
def oracles(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    cache = {}

    def get(name):
        if name not in cache:
            m = get_model(name)
            cache[name] = oracle_lib.Oracle(to_blob(m), m, 64)
        return cache[name]
    return get


def initial_state(m):
    return np.concatenate([m.key_qpos[0] if len(m.key_qpos) else np.zeros(m.nq), np.zeros(m.nv)])


def random_knots(m, rng, B, N, P, spread=1.5):
    """knots spread over 1.5 x ctrlrange (some are clamped), float32, distinct per knot"""
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    mid, half = cr.mean(1), 0.5 * (cr[:, 1] - cr[:, 0])
    return (mid + spread * half * rng.uniform(-1, 1, (B, N, P, m.nu))).astype(np.float32)


def check_spline(group, m, e, o, time0s, kts, knots, interp, H, state=None, mocap=None):
    """One batched launch of B problems (time0s[b], kts[b], knots[b] of N candidates) against the fp64 oracle."""
    B, N, P, nu = knots.shape
    state = initial_state(m) if state is None else state
    mocap = mocap_of(m) if mocap is None else mocap
    ret, fail, _ = e.rollout_spline_batched(np.tile(state, (B, 1)), np.asarray(time0s, float), np.tile(mocap, (B, 1)),
                                            knots, np.asarray(kts, float), interp, H)
    tr = e.fetch_all()
    scale = 1.0 + np.abs(knots).max()
    worst = 0.0
    for b in range(B):
        r = o.rollout_spline(state, time0s[b], mocap, knots[b], kts[b], interp, H, nthreads=4, full=True)
        assert not fail[b].any() and not r["failure"].any(), group
        dev = tr["actions"][b * N:(b + 1) * N]
        ref = r["actions"]
        assert np.array_equal(tr["times"][b * N:(b + 1) * N], r["times"]), (group, b)
        T = r["times"][0]
        upper = np.searchsorted(np.asarray(kts[b], float), T, side="right")
        held = (upper == 0) | (upper == P) | (interp == 0)
        held[H - 1] = False   # the last row repeats the row before it
        if held.any():
            assert np.array_equal(dev[:, held], ref[:, held].astype(np.float32)), \
                (group, b, np.nonzero((dev[:, held] != ref[:, held].astype(np.float32)).any((0, 2)))[0])
        if H == 1:
            assert not dev.any()
        else:
            assert np.array_equal(dev[:, H - 1], dev[:, H - 2])
        worst = max(worst, np.abs(dev - ref).max() / (1e-5 * scale))
    note(group, worst)
    assert worst <= 1.0, (group, worst)


@pytest.mark.parametrize("interp", [0, 1, 2])
@pytest.mark.parametrize("name", ["particle", "cartpole"])
def test_spline_time0_grid(engines, oracles, name, interp):
    """time0 on an accumulated 0.01 s agent clock over 3 s, plus 1000.25 and 86400: the planner's knot spacing for the
    interpolation (H = 32) and the shipped Shadow spacing (P = 5, H = 26: zero-order knots on steps 5, 10, 15, 20)."""
    m, e, o = get_model(name), engines(name), oracles(name)
    rng = np.random.default_rng(interp)
    time0s = agent_times(301) + [1000.25, 86400.0]
    Pm = int(m.numeric["sampling_spline_points"][0])
    for P, H, tag in ((Pm, 32, "planner"), (5, 26, "shadow spacing")):
        kts = [planner_knot_times(t0, m.opt_timestep, H, P, interp) for t0 in time0s]
        knots = random_knots(m, rng, len(time0s), 1, P)
        check_spline(f"spline {interp} {tag}", m, e, o, time0s, kts, knots, interp, H)


@pytest.mark.parametrize("interp", [0, 1, 2])
def test_spline_edges(engines, oracles, interp):
    """P = 1, 2, 3 and the capacity 64; non-uniform knots; the first knot after time0 and the last before the end of
    the horizon (first / last value held); H = 1 (zero action) and H = 2."""
    m, e, o = get_model("cartpole"), engines("cartpole"), oracles("cartpole")
    rng = np.random.default_rng(10 + interp)
    time0s = [0.0, 0.37, 1000.25, 86400.0]
    for P in (1, 2, 3, 64):
        kts = [planner_knot_times(t0, 0.01, 64, P, interp) for t0 in time0s]
        check_spline(f"spline {interp} edges", m, e, o, time0s, kts, random_knots(m, rng, 4, 2, P), interp, 64)
    gaps = rng.uniform(0.003, 0.07, 12)
    kts = [t0 + 0.05 + np.cumsum(gaps) for t0 in time0s]                       # first knot after time0
    check_spline(f"spline {interp} edges", m, e, o, time0s, kts, random_knots(m, rng, 4, 2, 12), interp, 64)
    kts = [t0 - 0.1 + np.cumsum(gaps[:4]) for t0 in time0s]                    # last knot before the end
    check_spline(f"spline {interp} edges", m, e, o, time0s, kts, random_knots(m, rng, 4, 2, 4), interp, 64)
    for H in (1, 2):
        kts = [planner_knot_times(t0, 0.01, 26, 5, interp) for t0 in time0s]
        check_spline(f"spline {interp} edges", m, e, o, time0s, kts, random_knots(m, rng, 4, 2, 5), interp, H)


SHAPES = {"helper-warp": {}, "plain": {"MJPC_B200_SHAPE": "plain"}, "generic": {"MJPC_B200_NO_STATIC": "1"}}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_spline_static_instances(engines, oracles, monkeypatch, name, shape):
    """The static instances in all three shapes; the helper-warp shape's task warp evaluates step t+1's spline while
    the main warp solves step t."""
    for k, v in SHAPES[shape].items():
        monkeypatch.setenv(k, v)
    m, e, o = get_model(name), engines(name, 64, 64), oracles(name)
    rng = np.random.default_rng(7)
    P, H = int(m.numeric["sampling_spline_points"][0]), 48
    time0s = [0.0, 0.37, 1000.25]
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    nominal = np.zeros((P, m.nu)) if name == "quadruped" else np.clip(m.key_qpos[0][7:7 + m.nu], cr[:, 0], cr[:, 1])
    for interp in (0, 1, 2):
        kts = [planner_knot_times(t0, m.opt_timestep, H, P, interp) for t0 in time0s]
        half = 0.5 * (cr[:, 1] - cr[:, 0])
        knots = (nominal + 0.05 * half * rng.standard_normal((3, 4, P, m.nu))).astype(np.float32)
        check_spline(f"spline static {name}", m, e, o, time0s, kts, knots, interp, H)
        expect = 0 if shape == "generic" else 1 if shape == "helper-warp" else 2
        assert e.last_kernel_shape == expect


def test_spline_generic_shadow(engines, oracles):
    """The generic instance on the Shadow hand with its shipped zero-order spline (P = 5, horizon 0.25 s)."""
    from test_shadow_cpu import _hold_ctrl
    m, e, o = get_model("shadow_reorient"), engines("shadow_reorient", 64, 64), oracles("shadow_reorient")
    P, H = 5, 26
    cr = np.asarray(m.actuator_ctrlrange, float)
    rng = np.random.default_rng(8)
    time0s = [0.0, 0.37, 1000.25]
    for interp in (0, 1, 2):
        kts = [planner_knot_times(t0, m.opt_timestep, H, P, interp) for t0 in time0s]
        knots = (_hold_ctrl(m, m.key_qpos[0]) + 0.1 * 0.5 * (cr[:, 1] - cr[:, 0]) * rng.standard_normal((3, 4, P, m.nu)))
        check_spline("spline generic shadow_reorient", m, e, o, time0s, kts, knots.astype(np.float32), interp, H)
        assert e.last_kernel_shape == 0


def test_shadow_zero_order_returns(engines, oracles):
    """The Shadow task's shipped zero-order spline, 128 x 26, with the planner's knot times at time0 = 0 and 0.37:
    returns at the bars of test_gpu_shadow.py::test_shadow_returns."""
    from mujoco_mpc_b200.planner import candidate_knots
    from test_gpu_teacher_forced import _stable_mask
    from test_shadow_cpu import _hold_ctrl
    m, e, o = get_model("shadow_reorient"), engines("shadow_reorient", 128, 26), oracles("shadow_reorient")
    N, H, P = 128, 26, 5
    state = initial_state(m)
    nominal = np.tile(_hold_ctrl(m, m.key_qpos[0]), (P, 1))
    knots = candidate_knots(nominal, 0.1, np.asarray(m.actuator_ctrlrange, float), 0, N, seed=7).astype(np.float32)
    for time0 in (0.0, 0.37):
        kt = planner_knot_times(time0, m.opt_timestep, H, P, 0)
        ret, fail, order = e.rollout_spline(state, time0, mocap_of(m), knots, kt, 0, H)
        r64 = o.rollout_spline(state, time0, mocap_of(m), knots, kt, 0, H, nthreads=8, full=True)
        assert not fail.any() and not r64["failure"].any()
        tr = e.fetch_all()
        assert np.array_equal(tr["actions"][:, : H - 1], r64["actions"][:, : H - 1].astype(np.float32))
        rel = np.abs(ret - r64["returns"]) / np.abs(r64["returns"])
        stable = _stable_mask(o, m, state, mocap_of(m), knots, kt, H, r64["returns"])
        print("shadow zero-order 128 x 26 at %.2f: rel err median %.2e max %.2e, well-conditioned %d, max on them %.2e" %
              (time0, np.median(rel), rel.max(), stable.sum(), rel[stable].max() if stable.any() else 0))
        assert np.median(rel) < 2e-5
        assert (rel[stable] > 1e-4).sum() == 0
        assert (rel > 1e-4).sum() <= 4 and rel.max() < 1e-3


# ------------------------------------------------------------------------------------------ feedback policy
def quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def axis_quat(axis, angle):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * axis])


def quat_addrs(m):
    out = []
    for j in range(len(m.jnt_type)):
        if m.jnt_type[j] == 0:
            out.append(m.jnt_qposadr[j] + 3)
        elif m.jnt_type[j] == 1:
            out.append(m.jnt_qposadr[j])
    return out


def nominal(m, o, H, time0, rng):
    """A nominal trajectory: the fp64 oracle's own spline rollout from the initial state (times are its times)."""
    P = 4
    kt = planner_knot_times(time0, m.opt_timestep, H, P, 1)
    knots = random_knots(m, rng, 1, 1, P, spread=0.6)[0]
    r = o.rollout_spline(initial_state(m), time0, mocap_of(m), knots, kt, 1, H, nthreads=1, full=True)
    assert not r["failure"].any()
    return (r["states"][0].astype(np.float32), r["actions"][0].astype(np.float32), r["times"][0])


FB_MODELS = {"particle": 40, "quadruped": 40, "shadow_reorient": 26}


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("name", list(FB_MODELS))
def test_feedback_policy(engines, oracles, name, mode):
    """Nominal times from the oracle's trajectory and as arange(H) dt; time0 at node 0 and node 3 (the planner's shift),
    before node 0 and halfway (the rollout runs past the last node); step sizes 1, 0.3, 0; gains that saturate
    ctrlrange; on the quaternion joints a nominal equal to -(state quaternion), a 179 degree offset, and nominal
    quaternions that turn from node to node (interpolated ones are not unit length)."""
    m, o = get_model(name), oracles(name)
    e = engines(name, 64, 64)
    H = FB_MODELS[name]
    dt = m.opt_timestep
    n, ds = 2 * m.nv, m.nq + m.nv
    rng = np.random.default_rng(100 + mode)
    x0, u0, t0 = nominal(m, o, H, 0.37, rng)
    qa = quat_addrs(m)
    du_step = np.linspace(-0.1, 0.1, H)[:, None] * np.ones(m.nu)       # node-to-node steps of the nominal action
    problems = []   # (time0, t_nom, x_nom, u_nom, gains)

    def add(time0, t_nom, x_nom=x0, u_nom=None, gscale=0.3):
        u = (u0 + du_step) if u_nom is None else u_nom
        K = (gscale * rng.standard_normal((H, m.nu, n))).astype(np.float32)
        problems.append((time0, np.asarray(t_nom, float), x_nom, u.astype(np.float32), K))
    add(t0[0], t0)
    add(t0[3], t0)
    add(t0[0] - 0.037, t0)
    add(t0[H // 2], t0)
    add(0.0, np.arange(H) * dt)
    add(3 * dt, np.arange(H) * dt)
    add(1000.25, ref_times(1000.25, dt, H))
    # the device's own recorded times as the nominal times (the iLQG planner's loop): from the start and shifted by 3
    e.rollout_spline(initial_state(m), 0.37, mocap_of(m), random_knots(m, rng, 1, 1, 2)[0], [0.37, 0.5], 0, H)
    t_dev = e.fetch_all()["times"][0].copy()
    add(t_dev[0], t_dev)
    add(t_dev[3], t_dev)
    add(t0[0], t0, gscale=50.0)
    if qa:
        xn = x0.copy()
        for a in qa:
            xn[:, a:a + 4] = -xn[:, a:a + 4]
        add(t0[0], t0, xn)
        xr = x0.copy()
        for a in qa:
            for t in range(H):
                xr[t, a:a + 4] = quat_mul(x0[t, a:a + 4].astype(float), axis_quat([0.3, -0.5, 0.8], np.deg2rad(179)))
        add(t0[0], t0, xr)
        xt = x0.copy()
        for a in qa:
            for t in range(H):
                xt[t, a:a + 4] = quat_mul(x0[t, a:a + 4].astype(float), axis_quat([1, 0.2, -0.4], np.deg2rad(25 * t)))
        add(t0[0], t0, xt)
    B, Kc = len(problems), 3
    steps = np.tile(np.array([1.0, 0.3, 0.0], np.float32), (B, 1))
    state = x0[0].astype(float).copy()
    state[m.nq:] += 0.05 * rng.standard_normal(m.nv)
    du = (0.05 * rng.standard_normal((B, H, m.nu))).astype(np.float32)
    ret, fail, _ = e.rollout_feedback_batched(np.tile(state, (B, 1)), np.array([p[0] for p in problems]),
                                              np.tile(mocap_of(m), (B, 1)), np.stack([p[3] for p in problems]),
                                              np.stack([p[2] for p in problems]), np.stack([p[1] for p in problems]),
                                              np.stack([p[4] for p in problems]), du, steps, mode)
    tr = e.fetch_all()
    worst = 0.0
    for b, (time0, t_nom, x_nom, u_nom, K) in enumerate(problems):
        T = ref_times(time0, dt, H)
        G = np.abs(K).sum(2).max()
        for k in range(Kc):
            c = b * Kc + k
            if fail[b, k]:
                continue
            assert np.array_equal(tr["times"][c], T), (b, k)
            step = float(steps[b, k])
            for t in range(H - 1):
                s = tr["states"][c, t].astype(float)
                if mode == 3:
                    u = u_nom[t:].astype(float) + step * du[b, t:].astype(float)
                    ref = o.ilqg_policy_action(u, x_nom[t:], t_nom[t:], K[t:], 3, 0.0, s, T[t])
                else:
                    ref = o.ilqg_policy_action(u_nom, x_nom, t_nom, K, mode, step, s, T[t])
                D = np.abs(s).max() + np.abs(x_nom).max() + np.pi
                bar = 1e-5 * (1 + np.abs(u_nom).max() + (1 if mode == 3 else step) * G * D + np.abs(du).max())
                err = np.abs(tr["actions"][c, t] - ref).max() / bar
                worst = max(worst, err)
                assert err <= 1.0, (name, mode, b, k, t, tr["actions"][c, t], ref)
    assert fail.sum() <= B * Kc // 4
    note(f"feedback mode {mode} {name}", worst)


def test_zz_report():
    """Largest error as a fraction of its bar, per group (printed with -s)."""
    for k in sorted(RATIOS):
        print(f"{k:45s} {RATIOS[k]:.3f}")
