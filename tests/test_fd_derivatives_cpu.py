"""CPU: the fp64 oracle's finite-difference transition Jacobians (oracle/ilqg.h model_derivatives, the restatement of
ModelDerivatives::Compute and mjd_transitionFD) against the closed forms of tests/fd_scenes.py, the control-limit rule
case by case, and the evaluate / interpolate schedule against a transcription of model_derivatives.cc.

The device sweep and the oracle are transliterations of each other, so a rule both get wrong passes the device-vs-oracle
tests; these checks state the Jacobians from the step's closed form instead.
  linear scenes     a secant of a linear map is the map: the oracle equals the closed form to round-off (1e-9)
  nonlinear scenes  the one-sided error shrinks like eps, the centred error like eps^2 (asserted over a step ratio of 4)
"""
import numpy as np
import pytest

import fd_scenes as F

SCENES = F.scenes()
NONLINEAR = [k for k in SCENES if k not in F.LINEAR]


@pytest.fixture(scope="module")
def oracles(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    out = {}
    for name, s in SCENES.items():
        m = s.compile()
        out[name] = (m, oracle_lib.Oracle(to_blob(m), m, 64))
    return out


def _mocap(m):
    return np.concatenate([np.concatenate([m.mocap_pos0[i], m.mocap_quat0[i]]) for i in range(m.nmocap)])


def fd(o, m, s, eps, mode, H=2, skip=0, xs=None, us=None):
    """The oracle's A, B, C, D with the scene's pose at every step (or the given per-step states / controls)."""
    xs = np.tile(s.x, (H, 1)) if xs is None else xs
    us = np.tile(s.u, (H, 1)) if us is None else us
    return o.model_derivatives(xs, us, np.arange(H) * m.opt_timestep, _mocap(m), tol=eps, skip=skip, mode=mode)


def _err(G, R):
    return max(np.abs(g - r).max() / (np.abs(r).max() + 1) for g, r in zip(G, R))


@pytest.mark.parametrize("name", list(SCENES))
def test_closed_forms_match_the_numeric_step(name):
    """The closed forms' sign and ordering conventions (R(h w)^T, h J_r(h w), 1/2 Q (x) (0, e_i), [dq; dv]) against a
    centred fp64 difference of the numpy step; the control-limit scene's B columns are the table's business."""
    s = SCENES[name]
    A, B, C, D = s.jacobians()
    An, Bn, Cn = s.numeric_jacobians()
    np.testing.assert_allclose(A, An, atol=1e-8)
    np.testing.assert_allclose(C, Cn, atol=1e-8)
    if name != "fd_ctrl_limits":
        np.testing.assert_allclose(B, Bn, atol=1e-8)
    assert not D.any()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", F.LINEAR)
def test_linear_scenes_exact(oracles, name, mode):
    m, o = oracles[name]
    s = SCENES[name]
    A, B, C, D = s.jacobians()
    if name == "fd_ctrl_limits":
        B = B * np.array([c[4] for c in F.ctrl_cases()])
    G = fd(o, m, s, F.EPS, mode)
    for k, R in enumerate((A, B, C, D)):
        assert np.abs(G[k][0] - R).max() <= 1e-9 * (np.abs(R).max() + 1), ("ABCD"[k], np.abs(G[k][0] - R).max())
    # the last step carries C only
    assert not G[0][1].any() and not G[1][1].any() and not G[3][1].any()
    np.testing.assert_allclose(G[2][1], C, atol=1e-9)


@pytest.mark.parametrize("mode", [0, 1])
def test_ctrl_limit_table(oracles, mode):
    """Which secant the rule takes, by value: the full slope where one side (or both) stays inside ctrlrange, exactly
    zero where neither does.  A secant that reached past a limit would read 0.5 (hi - eps/2 nudged forward, outside
    nudged back) or 0 (a limit nudged outward), a nudge inside a range narrower than eps 1/8."""
    m, o = oracles["fd_ctrl_limits"]
    s = SCENES["fd_ctrl_limits"]
    full = s.jacobians()[1]
    B = fd(o, m, s, F.EPS, mode)[1][0]
    for i, (case, _, _, _, want) in enumerate(F.ctrl_cases()):
        col, ref = B[:, i], full[:, i]
        dof = s.dadr[i]
        assert not np.delete(col, [dof, s.nv + dof]).any(), case
        if want == 0:
            assert not col.any(), (case, col)
        else:
            np.testing.assert_allclose(col, ref, rtol=1e-9, atol=1e-12, err_msg=case)


def _order(o, m, s, mode, eps):
    """Error against the closed form at eps and eps / 4, and its ratio."""
    R = s.jacobians()
    e1, e2 = (_err([g[0] for g in fd(o, m, s, e, mode)], R) for e in (eps, eps / 4))
    return e1, e2, e1 / e2


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", NONLINEAR)
def test_nonlinear_scenes_truncation_order(oracles, name, mode):
    """One-sided: error ~ eps (ratio 4 over a step ratio of 4); centred: ~ eps^2 (ratio 16).  At the fp32 step
    EPS the error is the truncation alone (bounded), and the rotation blocks are asserted on their own."""
    m, o = oracles[name]
    s = SCENES[name]
    eps = 1e-2
    e1, e2, ratio = _order(o, m, s, mode, eps)
    print(name, mode, "err(eps=%.0e) %.3e  err(eps/4) %.3e  ratio %.2f" % (eps, e1, e2, ratio))
    want = 4.0 if mode == 0 else 16.0
    assert 0.8 * want < ratio < 1.25 * want, (e1, e2, ratio)
    assert e1 < (2e-2 if mode == 0 else 2e-4)
    # at the step the device uses, the error is the truncation of that order
    G = [g[0] for g in fd(o, m, s, F.EPS, mode)]
    R = s.jacobians()
    assert _err(G, R) < e1 * (F.EPS / eps) ** (1 + mode) * 1.3
    for b, body in enumerate(s.bodies):
        if body.kind in ("ball", "free"):
            r0 = s.dadr[b] + (3 if body.kind == "free" else 0)
            rows = np.r_[r0:r0 + 3]
            cols = np.r_[r0:r0 + 3, s.nv + r0:s.nv + r0 + 3]
            rot = np.abs(G[0][np.ix_(rows, cols)] - R[0][np.ix_(rows, cols)]).max()
            assert rot < (2e-5 if mode == 0 else 1e-9), (body.kind, rot)


def _find_interval(seq, value):
    """FindInterval (utilities.h:125-144)."""
    upper = 0
    while upper < len(seq) and not value < seq[upper]:
        upper += 1
    lower = upper - 1
    if lower < 0:
        return 0, 0
    if lower > len(seq) - 1:
        return len(seq) - 1, len(seq) - 1
    return max(lower, 0), min(upper, len(seq) - 1)


def reference_schedule(T, skip):
    """model_derivatives.cc:56-72 (evaluate / interpolate lists) and :109-164 (each interpolated step's e0, e1 and
    weight).  For T = 1 the reference's list would hold T - 2 = -1; the project evaluates step 0 alone (C only)."""
    if T == 1:
        return [0], []
    s = skip + 1
    evaluate = [0]
    t = s
    while t < T - s:
        evaluate.append(t)
        t += s
    evaluate += [T - 2, T - 1]
    interp, e = [], 0
    for t in range(T):
        if e == len(evaluate) or evaluate[e] > t:
            b0, b1 = _find_interval(evaluate, t)
            e0, e1 = evaluate[b0], evaluate[b1]
            interp.append((t, e0, e1, 0.0 if b0 == b1 else (t - e0) / (e1 - e0)))
        else:
            e += 1
    return evaluate, interp


@pytest.mark.parametrize("mode", [0, 1])
def test_schedule(oracles, mode):
    """H 1..12 x skip 0..6 on the pendulum with a different state at every step: evaluated steps equal the skip = 0
    sweep, interpolated steps are the reference's blend of their neighbours, the last step carries C only."""
    m, o = oracles["fd_pendulum"]
    s = SCENES["fd_pendulum"]
    rng = np.random.default_rng(3)
    blended = 0
    for T in range(1, 13):
        xs = np.stack([np.concatenate([s.q + 0.3 * rng.standard_normal(1), s.v + rng.standard_normal(1)])
                       for _ in range(T)])
        us = rng.uniform(-0.9, 0.9, (T, 1))
        full = fd(o, m, s, 1e-3, mode, H=T, xs=xs, us=us)
        for skip in range(7):
            G = fd(o, m, s, 1e-3, mode, H=T, skip=skip, xs=xs, us=us)
            evaluate, interp = reference_schedule(T, skip)
            assert sorted(set(evaluate) | {t for t, *_ in interp}) == list(range(T))
            for k in range(4):
                for t in set(evaluate):
                    np.testing.assert_array_equal(G[k][t], full[k][t])
                for t, e0, e1, w in interp:
                    np.testing.assert_allclose(G[k][t], (1 - w) * full[k][e0] + w * full[k][e1], rtol=1e-14, atol=1e-15)
                    blended += int(k == 0 and np.abs(G[k][t] - full[k][t]).max() > 1e-6)
            assert not G[0][T - 1].any() and not G[1][T - 1].any() and not G[3][T - 1].any(), (T, skip)
            np.testing.assert_allclose(G[2][T - 1], np.eye(2), atol=1e-9)
    assert blended > 50          # the interpolated steps really differ from an evaluation there
