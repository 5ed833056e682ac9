"""GPU: the finite-difference sweep (csrc/ilqg_kernels.cuh fd_center_kernel / fd_column_kernel / fd_interp_kernel) at
its edges, against the closed forms of tests/fd_scenes.py and the fp64 oracle at the SAME step.

fp32 bars: a device column is a difference of two fp32 steps divided by eps, so its round-off is a few ulps of the next
state over eps.  Each block must be within 32 ulps of the state's scale over eps (ROUNDOFF) and within 3x the error of
the oracle's own fp32 instantiation plus 4 ulps over eps.  The closed-form check is the CPU test's (the fp64 oracle
against the closed form, test_fd_derivatives_cpu.py) plus this one: device - closed form <= oracle - closed form + bar.
"""
import numpy as np
import pytest

import fd_scenes as F
from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

SCENES = F.scenes()
ULP = 2.0 ** -23


@pytest.fixture(scope="module")
def scene_ctx(oracle_lib):
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    build.build()
    out = {}
    for name, s in SCENES.items():
        m = s.compile()
        out[name] = (m, Engine(m, 8, 16), oracle_lib.Oracle(to_blob(m), m, 64), oracle_lib.Oracle(to_blob(m), m, 32))
    yield out
    for _, e, _, _ in out.values():
        e.close()


def _bars(x, eps):
    scale = np.abs(x).max() + 1
    return 32 * ULP * scale / eps, 4 * ULP * scale / eps


def _scene_run(ctx, name, mode, eps=F.EPS, H=2):
    m, e, o64, o32 = ctx[name]
    s = SCENES[name]
    xs, us, ts = np.tile(s.x, (H, 1)), np.tile(s.u, (H, 1)), np.arange(H) * m.opt_timestep
    G = e.model_derivatives(xs, us, ts, mocap_of(m), eps, mode=mode)
    R = o64.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, mode=mode)
    R32 = o32.model_derivatives(xs, us, ts, mocap_of(m), tol=eps, mode=mode)
    return s, G, R, R32


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", [n for n in SCENES if n != "fd_ctrl_limits"])
def test_scene_against_fp64_and_closed_form(scene_ctx, name, mode):
    s, G, R, R32 = _scene_run(scene_ctx, name, mode)
    closed = s.jacobians()
    roundoff, floor = _bars(s.x, F.EPS)
    for k, nm in enumerate("ABCD"):
        g, r, r32, c = G[k][0], R[k][0], R32[k][0], closed[k]
        err, err32, errc, errc64 = (np.abs(a - b).max() for a, b in ((g, r), (r32, r), (g, c), (r, c)))
        print("FD %s mode %d %s: device - fp64 %.2e (fp32 oracle %.2e, bar %.2e); device - closed form %.2e "
              "(fp64 oracle %.2e)" % (name, mode, nm, err, err32, min(roundoff, 3 * err32 + floor), errc, errc64))
        assert np.isfinite(g).all()
        assert err <= roundoff and err <= 3 * err32 + floor, (nm, err, err32)
        assert errc <= errc64 + roundoff, (nm, errc, errc64)
    assert not G[3].any()                                   # the state copy does not depend on the control
    assert not G[0][1].any() and not G[1][1].any()          # the last step carries C only
    np.testing.assert_allclose(G[2][1], closed[2], atol=roundoff)
    # the ball and free orientation blocks on their own: rows and columns of the rotation dofs
    for b, body in enumerate(s.bodies):
        if body.kind not in ("ball", "free"):
            continue
        r0 = s.dadr[b] + (3 if body.kind == "free" else 0)
        rows, cols = np.r_[r0:r0 + 3], np.r_[r0:r0 + 3, s.nv + r0:s.nv + r0 + 3]
        blk = lambda X: X[np.ix_(rows, cols)]
        err, err32 = np.abs(blk(G[0][0]) - blk(R[0][0])).max(), np.abs(blk(R32[0][0]) - blk(R[0][0])).max()
        errc = np.abs(blk(G[0][0]) - blk(closed[0])).max()
        qr = s.qadr[b] + (3 if body.kind == "free" else 0)
        cq = np.abs(G[2][0][qr:qr + 4, r0:r0 + 3] - closed[2][qr:qr + 4, r0:r0 + 3]).max()
        print("FD %s mode %d %s orientation: A block device - fp64 %.2e (fp32 oracle %.2e), device - closed form %.2e;"
              " C quaternion rows device - closed form %.2e" % (name, mode, body.kind, err, err32, errc, cq))
        assert err <= roundoff and err <= 3 * err32 + floor
        # R(h w)^T and h J_r(h w) are far from the identity here, so a wrong sign or tangent index is O(0.1) off
        assert errc <= np.abs(blk(R[0][0]) - blk(closed[0])).max() + roundoff
        assert cq <= (0.2 * F.EPS if mode == 0 else 0.05 * F.EPS ** 2) + roundoff


@pytest.mark.parametrize("mode", [0, 1])
def test_ctrl_limit_table_on_device(scene_ctx, mode):
    """Which secant the device takes, by value: the v row of each control column is the full slope (not half of it,
    not zero) where the table says 1, and exactly zero where it says 0."""
    s, G, R, R32 = _scene_run(scene_ctx, "fd_ctrl_limits", mode)
    full = s.jacobians()[1]
    B = G[1][0]
    roundoff, _ = _bars(s.x, F.EPS)
    for i, (case, _, _, _, want) in enumerate(F.ctrl_cases()):
        dof = s.dadr[i]
        col = B[:, i]
        slope = full[s.nv + dof, i]
        assert not np.delete(col, [dof, s.nv + dof]).any(), case
        ratio = col[s.nv + dof] / slope
        print("FD ctrl table mode %d %-22s expected %.0f, device v-row / full slope %.6f" % (mode, case, want, ratio))
        if want == 0:
            assert not col.any(), (case, col)
        else:
            assert abs(ratio - 1) < 5e-3, (case, ratio)
            assert abs(col[dof] - full[dof, i]) <= roundoff, case
    np.testing.assert_array_equal(B == 0, R[1][0] == 0)


# ---------------------------------------------------------------------------------------------- hand and humanoid track
def _hand_nominal(m, o, H):
    """The stand-in hand from its grasp keyframe with the first finger's tendon at length 2: controls at ctrlrange
    limits (FFJ4 / THJ4 at upper limits whose fp32 rounding lies above the fp64 value, as THJ2's keyframe target
    0.6981 clamped to 0.698 is; FFJ0 at 3.1415 on a tendon, MFJ0 at 0 on a tendon), and both wrist actuators (kp 10) driven into their forcerange clamp of +-2, one at a limit
    and one inside its range."""
    from test_shadow_cpu import _hold_ctrl
    acts, jn = list(m.actuator_names), list(m.jnt_names)
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    q0 = np.array(m.key_qpos[0], float)
    qa = lambda j: m.jnt_qposadr[jn.index("rh_" + j)]
    q0[qa("FFJ1")] = q0[qa("FFJ2")] = 1.0
    q0[qa("WRJ2")], q0[qa("WRJ1")] = -0.2, -0.3
    u = _hold_ctrl(m, q0)
    ai = {n: acts.index("rh_A_" + n) for n in ("FFJ0", "MFJ0", "FFJ4", "THJ4", "THJ2", "WRJ2", "WRJ1")}
    u[ai["FFJ0"]], u[ai["MFJ0"]] = cr[ai["FFJ0"], 1], cr[ai["MFJ0"], 0]
    u[ai["FFJ4"]], u[ai["THJ4"]] = cr[ai["FFJ4"], 1], cr[ai["THJ4"], 1]
    u[ai["WRJ2"]], u[ai["WRJ1"]] = cr[ai["WRJ2"], 1], 0.3
    state = np.concatenate([q0, np.zeros(m.nv)])
    r = o.rollout_spline(state, 0.0, mocap_of(m), np.tile(u, (1, 2, 1)), np.array([0.0, 1.0]), 0, H)
    return r["states"][0], r["actions"][0], r["times"][0], ai


def _columnwise(name, G, R, Rh, F32):
    """test_gpu_ilqg's column-wise bar (toggle columns found by halving the step); returns the per-column errors."""
    from test_gpu_ilqg import _column_stats
    out = []
    for k, nm in enumerate("ABCD"):
        err, smooth = _column_stats(G[k], R[k], Rh[k])
        err32, _ = _column_stats(F32[k], R[k], Rh[k])
        es, es32 = err[smooth], err32[smooth]
        print("FD %s %s columns %d, smooth %.1f %%; device err / column scale: median %.2e p99 %.2e max %.2e | "
              "fp32 oracle %.2e %.2e %.2e" % (name, nm, smooth.size, 100 * smooth.mean(), np.median(es),
                                              np.percentile(es, 99), es.max(), np.median(es32),
                                              np.percentile(es32, 99), es32.max()))
        assert np.isfinite(G[k]).all() and smooth.mean() >= 0.8
        if nm in "CD":
            assert es.max() < 2e-3, (nm, es.max())
        else:
            assert np.median(es) < 2e-2 and np.percentile(es, 99) < 0.15 and es.max() < 0.3
            assert np.median(es) < 3 * np.median(es32) + 1e-3 and np.percentile(es, 99) < 3 * np.percentile(es32, 99) + 1e-3
        if (~smooth).any():
            assert err[~smooth].max() < 2.0
        out.append((err, err32, smooth))
    return out


@pytest.fixture(scope="module")
def hand(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    m = get_model("shadow_reorient")
    o = oracle_lib.Oracle(to_blob(m), m, 64)
    e = Engine(m, 8, 16)
    yield m, e, o, oracle_lib.Oracle(to_blob(m), m, 32)
    e.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_hand_against_fp64(hand, mode):
    """nv = 33 (more than one warp of dofs), 20 position actuators with forcerange, four on fixed tendons."""
    m, e, o, o32 = hand
    H, eps = 5, 1e-3
    xs, us, ts, ai = _hand_nominal(m, o, H)
    mc = mocap_of(m)
    G = e.model_derivatives(xs, us, ts, mc, eps, mode=mode)
    R = o.model_derivatives(xs, us, ts, mc, tol=eps, mode=mode, nthreads=8)
    Rh = o.model_derivatives(xs, us, ts, mc, tol=eps / 2, mode=mode, nthreads=8)
    F32 = o32.model_derivatives(xs, us, ts, mc, tol=eps, mode=mode, nthreads=8)
    stats = _columnwise("hand mode %d" % mode, G, R, Rh, F32)
    assert not G[0][-1].any() and not G[1][-1].any() and not G[3][-1].any()
    # B's columns: [time step][perturbed control] in _column_stats' flattening
    errB, err32B, smoothB = (x.reshape(H, m.nu) for x in stats[1])
    tendon = [i for i in range(m.nu) if m.actuator_trntype[i] != 0]
    assert len(tendon) == 4
    te, te32 = errB[:H - 1, tendon], err32B[:H - 1, tendon]
    print("FD hand mode %d tendon-actuator B columns: device err / column scale max %.2e | fp32 oracle %.2e"
          % (mode, te.max(), te32.max()))
    assert smoothB[:H - 1, tendon].all() and te.max() <= 3 * te32.max() + 1e-2
    # the force-clamped wrist actuators: zero columns on the device and in fp64, up to the contact solve's round-off
    # (the nudged evaluation starts from the centre's qacc, the centre from zero) over eps
    clamped = (ai["WRJ2"], ai["WRJ1"])
    active = min(np.abs(G[1][:H - 1, :, i]).max() for i in range(m.nu) if i not in clamped)
    for n in ("WRJ2", "WRJ1"):
        dev, ref, f32 = (np.abs(X[1][:H - 1, :, ai[n]]).max() for X in (G, R, F32))
        print("FD hand mode %d force-clamped %s B column max: device %.2e fp64 %.2e fp32 oracle %.2e (smallest "
              "unclamped column %.2e)" % (mode, n, dev, ref, f32, active))
        assert ref < 1e-9 and dev < 1e-2 * active, (n, dev, ref, f32)
    # controls at limits: the side that stays inside, the same secant on both sides
    for n in ("FFJ0", "MFJ0", "FFJ4", "THJ4", "THJ2"):
        assert np.abs(G[1][:H - 1, :, ai[n]]).max() > 1.0, n
        assert smoothB[:H - 1, ai[n]].all() and errB[:H - 1, ai[n]].max() <= 3 * err32B[:H - 1, ai[n]].max() + 1e-2, n
    # documented (DESIGN.md section 3): the limit test runs in the model's precision.  The fp32 rounding of the upper
    # limits 0.349 (FFJ4), 1.222 (THJ4) and 0.698 (THJ2) lies above their fp64 values, so the fp32 control the device holds at that
    # limit is, in fp64, outside the range: the fp64 oracle fed that fp32 value leaves a zero column where the device
    # (and the fp64 oracle fed the fp64 limit) takes the backward secant.  3.1415 rounds down: no difference there.
    R_f32_in = o.model_derivatives(xs, us.astype(np.float32).astype(float), ts, mc, tol=eps, mode=mode, nthreads=8)
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    u32 = us[0].astype(np.float32).astype(float)
    outside = {i for i in range(m.nu) if not cr[i, 0] <= u32[i] <= cr[i, 1]}
    assert outside == {ai["FFJ4"], ai["THJ4"], ai["THJ2"]}, outside
    for i in range(m.nu):
        col = np.abs(R_f32_in[1][:H - 1, :, i]).max()
        if i in outside:
            assert col == 0, m.actuator_names[i]
        elif i not in clamped:
            assert col > 1.0 and np.abs(G[1][:H - 1, :, i]).max() > 1.0, m.actuator_names[i]


def test_humanoid_track_against_fp64(oracle_lib):
    """Humanoid Track: the generic instance with the keyframe-tracking residual (time-dependent targets)."""
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    from test_gpu_ilqg import _nominal
    m = get_model("humanoid_track")
    o, o32 = oracle_lib.Oracle(to_blob(m), m, 64), oracle_lib.Oracle(to_blob(m), m, 32)
    H, eps = 6, 1e-3
    state, xs, us, ts, res = _nominal(m, o, H)
    mc = mocap_of(m)
    e = Engine(m, 8, 16)
    try:
        G = e.model_derivatives(xs, us, ts, mc, eps)
    finally:
        e.close()
    R = o.model_derivatives(xs, us, ts, mc, tol=eps, nthreads=8)
    Rh = o.model_derivatives(xs, us, ts, mc, tol=eps / 2, nthreads=8)
    F32 = o32.model_derivatives(xs, us, ts, mc, tol=eps, nthreads=8)
    _columnwise("humanoid_track", G, R, Rh, F32)
    assert not G[0][-1].any() and not G[1][-1].any() and not G[3][-1].any()


# ---------------------------------------------------------------------------------------------- small sizes, batched
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("skip", [0, 5])
@pytest.mark.parametrize("H", [1, 2, 3])
def test_small_horizons_batched(scene_ctx, H, skip, mode):
    """H = 1 (C at t = 0 only), 2 and 3 with skip 0 and 5 (the skip reaches past the horizon) through
    model_derivatives_batched with three problems of different states on the free-body scene."""
    m, e, o64, o32 = scene_ctx["fd_free"]
    s = SCENES["fd_free"]
    rng = np.random.default_rng(H * 10 + skip)
    Bn = 3
    xs = np.tile(s.x, (Bn, H, 1))
    xs[:, :, s.nq:] += 0.5 * rng.standard_normal((Bn, H, s.nv))
    us = rng.uniform(-0.9, 0.9, (Bn, H, s.nu))
    ts = np.tile(np.arange(H) * m.opt_timestep, (Bn, 1)) + np.arange(Bn)[:, None]
    mcs = np.tile(mocap_of(m), (Bn, 1))
    G = e.model_derivatives_batched(xs, us, ts, mcs, F.EPS, skip=skip, mode=mode)
    roundoff, floor = _bars(xs, F.EPS)
    for b in range(Bn):
        R = o64.model_derivatives(xs[b], us[b], ts[b], mocap_of(m), tol=F.EPS, skip=skip, mode=mode)
        R32 = o32.model_derivatives(xs[b], us[b], ts[b], mocap_of(m), tol=F.EPS, skip=skip, mode=mode)
        for k, nm in enumerate("ABCD"):
            err, err32 = np.abs(G[k][b] - R[k]).max(), np.abs(R32[k] - R[k]).max()
            assert err <= roundoff and err <= 3 * err32 + floor, (b, nm, err, err32)
        assert not G[0][b, H - 1].any() and not G[1][b, H - 1].any() and not G[3][b, H - 1].any(), b
        assert np.abs(G[2][b, H - 1]).max() > 0.4                # C at the last step (quaternion and identity rows)
        if H > 1:
            assert (np.abs(G[0][b, :H - 1]).max(axis=(1, 2)) > 0.5).all()
