"""GPU: the Riccati backward pass (backward_pass_kernel: warp box-QP, plain Cholesky, the four regularisations) against
the fp64 oracle (oracle/ilqg.h backward_pass) at the edges the planner tests do not reach: box limits that actually
bind, the largest shipped size (humanoid, n = 54, m = 21), one actuator (cartpole), reg_type 3, and failing
factorisations.

Inputs.  The nominal and its derivatives come from the fp64 oracle as in test_gpu_ilqg.py; every input is rounded to
fp32 before both calls, so the two sides solve the same problem.  To make limits bind, every third actuator's nominal
action sits exactly on its upper bound and the next one's on its lower bound (their box is one-sided: [lo - u, 0] or
[0, hi - u]), and cu is scaled by 300 so that the unconstrained du leaves the box.

Bars.  The device's round-off is modelled as a relative perturbation of every input of (n + m) * 2^-24 (one rounding
per term of the longest dot product); delta_k is the largest change of output k of the fp64 oracle under two such
random perturbations, which carries the problem's own conditioning (Cholesky of Quu, the recursion over H steps).  The
bar is 128 * delta_k + 2^-20 * max|ref_k|: input perturbations do not reach the rounding of the intermediate sums
(Quu = cuu + B'WB, the Vxx update), whose cancellation costs up to ~2^6 more on these problems (measured: largest
error / delta_k of 86, humanoid du with limits).

Excluded steps (near-degenerate box-QP, decided in fp64 before any comparison), with e = 16 (n + m) 2^-24: an
actuator on a bound whose QP gradient is below e (|Qu| + |Quu_reg| |du|), or a free actuator closer to a bound than
the du bar (128 delta_du) plus e times the box width.  There an fp32 round-off can legitimately flip the clamped set; since the recursion runs backwards, that step
and every earlier one are left out, never the bar loosened; a case with no Riccati step left is skipped.
"""
import numpy as np
import pytest

from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

HORIZON = {"quadruped": 16, "humanoid": 10, "cartpole": 16}
U24 = 2.0 ** -24
OUTS = ("du", "K", "Vx", "Vxx")
CU_SCALE = 300.0


@pytest.fixture(scope="module")
def bctx(oracle_lib):
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    build.build()
    out = {}
    for name, H in HORIZON.items():
        m = get_model(name)
        o = oracle_lib.Oracle(to_blob(m), m, 64)
        out[name] = (m, Engine(m, 16, H), _problem(m, o, H))
    yield out
    for _, e, _ in out.values():
        e.close()


def _f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def _problem(m, o, H):
    """fp32-rounded backward-pass inputs with binding limits (see the module docstring)"""
    from mujoco_mpc_b200.planner import candidate_knots
    P = 3
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    state = np.concatenate([m.key_qpos[0] if m.nkey else m.qpos0, np.zeros(m.nv)])
    kt = np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    knots = candidate_knots(np.zeros((P, m.nu)), 0.3, cr, 0, 2)[1:2]
    r = o.rollout_spline(state, 0.0, mocap_of(m), knots, kt, 2, H)
    xs, us, ts, res = r["states"][0], r["actions"][0].copy(), r["times"][0], r["residual"][0]
    A, B, C, D = o.model_derivatives(xs, us, ts, mocap_of(m), tol=1e-6)
    cx, cu, cxx, cuu, cxu = o.cost_derivatives(res, C, D)
    j = np.arange(m.nu)
    if m.nu == 1:
        us[::2, 0] = cr[0, 1]
    else:
        us[:, j % 3 == 0] = cr[j % 3 == 0, 1]
        us[:, j % 3 == 1] = cr[j % 3 == 1, 0]
    cu = CU_SCALE * cu
    return dict(A=_f32(A), B=_f32(B), cx=_f32(cx), cu=_f32(cu), cxx=_f32(cxx), cxu=_f32(cxu), cuu=_f32(cuu),
                actions=_f32(us), cr=cr)


def _oracle(oracle_lib, p, mu, reg_type, limits, **over):
    q = dict(p, **over)
    return oracle_lib.backward_pass(q["A"], q["B"], q["cx"], q["cu"], q["cxx"], q["cxu"], q["cuu"], q["actions"], q["cr"],
                                    mu=mu, reg_type=reg_type, limits=limits)


def _device(e, p, mu, reg_type, limits, **over):
    q = dict(p, **over)
    return e.backward_pass(q["A"], q["B"], q["cx"], q["cu"], q["cxx"], q["cxu"], q["cuu"], q["actions"], mu=mu,
                           reg_type=reg_type, limits=limits)


def _quu_reg(p, r, t, mu, reg_type):
    """the matrix the box QP / Cholesky sees at step t (oracle/ilqg.h: regularisation 0 control, 1 state-control,
    2 value, 3 none)"""
    Bt = p["B"][t]
    n, m = Bt.shape
    if reg_type == 2:
        Q = p["cuu"][t] + Bt.T @ (r["Vxx"][t + 1] + mu * np.eye(n)) @ Bt
    else:
        Q = r["Quu"][t].copy()
    if mu != 0 and reg_type == 0:
        Q += mu * np.eye(m)
    elif mu != 0 and reg_type == 1:
        Q += mu * Bt.T @ Bt
    return Q


def _clamped_and_degenerate(p, r, mu, reg_type, limits, du_bar):
    """per step: the fp64 clamped set (on a bound with a zeroed K row) and whether the step is near-degenerate"""
    H, m = r["du"].shape
    lo = p["cr"][:, 0][None, :] - p["actions"]
    hi = p["cr"][:, 1][None, :] - p["actions"]
    clamped = np.zeros((H, m), bool)
    degenerate = np.zeros(H, bool)
    if limits != 1:
        return clamped, degenerate
    eps = 16 * (p["B"].shape[1] + m) * U24
    for t in range(H - 1):
        du = r["du"][t]
        on_lo, on_hi = du == lo[t], du == hi[t]
        clamped[t] = (on_lo | on_hi) & (np.abs(r["K"][t]).max(1) == 0)
        Q = _quu_reg(p, r, t, mu, reg_type)
        grad = Q @ du + r["Qu"][t]
        gscale = np.abs(r["Qu"][t]).max() + np.abs(Q).max() * np.abs(du).max() + 1e-30
        width = hi[t] - lo[t]
        weak = (on_lo | on_hi) & (np.abs(grad) < eps * gscale)
        close = ~(on_lo | on_hi) & (np.minimum(du - lo[t], hi[t] - du) < du_bar + eps * width)
        degenerate[t] = weak.any() or close.any()
    clamped[H - 1] = clamped[H - 2]
    return clamped, degenerate


def _sensitivity(oracle_lib, p, mu, reg_type, limits, ref):
    """largest change of each fp64 output under two random relative input perturbations of (n + m) * 2^-24"""
    rng = np.random.default_rng(7)
    n, m = p["B"].shape[1:]
    eps = (n + m) * U24
    delta = {k: 0.0 for k in OUTS}
    delta["dV"] = 0.0
    for _ in range(2):
        over = {k: p[k] * (1 + eps * rng.uniform(-1, 1, p[k].shape)) for k in ("A", "B", "cx", "cu", "cxx", "cxu", "cuu")}
        rp = _oracle(oracle_lib, p, mu, reg_type, limits, **over)
        if rp["status"] != ref["status"]:
            continue
        for k in delta:
            delta[k] = max(delta[k], float(np.abs(rp[k] - ref[k]).max()))
    return delta


@pytest.mark.parametrize("mu", [0.0, 1e-3, 10.0])
@pytest.mark.parametrize("limits", [0, 1])
@pytest.mark.parametrize("reg_type", [0, 1, 2, 3])
@pytest.mark.parametrize("name", list(HORIZON))
def test_backward_pass_vs_fp64(bctx, oracle_lib, name, reg_type, limits, mu):
    m, e, p = bctx[name]
    H = HORIZON[name]
    ref = _oracle(oracle_lib, p, mu, reg_type, limits)
    dev = _device(e, p, mu, reg_type, limits)
    assert dev["status"] == ref["status"], (dev["status"], ref["status"])
    if ref["status"] != 1:
        return
    delta = _sensitivity(oracle_lib, p, mu, reg_type, limits, ref)
    clamped, degenerate = _clamped_and_degenerate(p, ref, mu, reg_type, limits, 128 * delta["du"])
    t0 = int(np.nonzero(degenerate)[0].max()) + 1 if degenerate.any() else 0   # compared steps: t0 .. H-1
    if t0 > H - 2:
        pytest.skip("every Riccati step at or after a near-degenerate box QP: %s" % np.nonzero(degenerate)[0].tolist())
    steps = np.arange(t0, H)
    if limits == 1:
        assert clamped[steps].sum() > 0, "no active limit in the compared steps"
        lo = p["cr"][:, 0][None, :] - p["actions"]
        hi = p["cr"][:, 1][None, :] - p["actions"]
        dev_du = dev["du"].astype(np.float64)
        dev_clamped = ((dev_du == _f32(lo)) | (dev_du == _f32(hi))) & (dev["K"] == 0).all(2)
        # (step H-1 only repeats du and K of step H-2, whose box came from that step's actions)
        np.testing.assert_array_equal(dev_clamped[steps[:-1]], clamped[steps[:-1]])
        # clamped du sits exactly on its (fp32) bound and the K rows of clamped actuators are exactly zero
        on = np.where(ref["du"] == lo, _f32(lo), _f32(hi))
        inner = steps[:-1]
        assert (dev_du[inner][clamped[inner]] == on[inner][clamped[inner]]).all()
        assert (dev["K"][inner][clamped[inner]] == 0).all()
    report = []
    for k in OUTS:
        G, R = dev[k][steps].astype(np.float64), ref[k][steps]
        assert np.isfinite(G).all(), k
        bar = 128 * delta[k] + 2.0 ** -20 * np.abs(R).max()
        err = float(np.abs(G - R).max())
        report.append("%s %.2e/%.2e" % (k, err, bar))
        assert err <= bar, (k, err, bar, delta[k])
    if t0 == 0:
        err = float(np.abs(dev["dV"] - ref["dV"]).max())
        bar = 128 * delta["dV"] + 2.0 ** -20 * np.abs(ref["dV"]).max()
        report.append("dV %.2e/%.2e" % (err, bar))
        assert err <= bar, ("dV", err, bar)
    print("backward pass %-9s reg %d limits %d mu %-6g steps %d..%d clamped %3d: err/bar %s" % (
        name, reg_type, limits, mu, t0, H - 1, int(clamped[steps].sum()), " ".join(report)))


@pytest.mark.parametrize("limits", [0, 1])
@pytest.mark.parametrize("name", list(HORIZON))
def test_backward_pass_failure_status(bctx, oracle_lib, name, limits):
    """an indefinite cuu at one interior step: with mu = 0 both sides report failure (status 0) from the box-QP path
    (limits 1) and the plain Cholesky path (limits 0); control regularisation large enough to restore definiteness
    makes both succeed"""
    m, e, p = bctx[name]
    H = HORIZON[name]
    t = H // 2
    # nominal actions inside the box and zero gradients (du = 0 at every step): no actuator starts step t's box QP on
    # a bound, so the factorisation of its free block is reached
    over = dict(actions=np.zeros_like(p["actions"]), cx=np.zeros_like(p["cx"]), cu=np.zeros_like(p["cu"]))
    Q = _oracle(oracle_lib, p, 0.0, 0, limits, **over)["Quu"][t]
    shift = float(np.linalg.eigvalsh(Q).max()) + 1.0
    cuu = p["cuu"].copy()
    cuu[t] -= shift * np.eye(m.nu)        # Quu at step t: every eigenvalue <= -1
    over["cuu"] = _f32(cuu)
    for mu, want in ((0.0, 0), (2 * shift + 1.0, 1)):
        ref = _oracle(oracle_lib, p, mu, 0, limits, **over)
        dev = _device(e, p, mu, 0, limits, **over)
        assert ref["status"] == want, (mu, ref["status"])
        assert dev["status"] == want, (mu, dev["status"])
