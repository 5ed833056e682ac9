"""GPU: the device's joint-space rows and forces - dof friction loss, joint limits, springs / damping / armature,
actuation, the <option><flag> switches and the constraint capacity - against the fp64 oracle on the scenes of
tests/joint_scenes.py (the oracle itself is pinned to closed forms by tests/test_oracle_joint_constraints.py).

Compared per pose, step_debug (the generic instance) against forward_debug: nefc and the warning exactly; efc_force,
qacc and next_qvel with the bars of tests/test_gpu_contacts.py (2e-3 of the qacc scale max |qacc| + 1; 2e-3 dt of it
plus 1e-5; 2e-3 of the force scale max |efc_force| + 1).  A friction row in the linear zone carries exactly the
friction loss, so there |efc_force| must equal fp32(frictionloss) bit for bit.  The same poses also run batched through
step_batch, and the mixed scene through a short rollout_spline.

Poses keep every limit row's dist - margin at least 5e-3 away from zero.  Whether a row exists is the sign of
dist - margin, computed in fp32 on the device from a rounded qpos (relative error 6e-8, so about 1e-7 at these joint
angles): a pose closer to the boundary than that could list the row on one side only, which is rounding, not a bug.

The path scenes assert from the host-side model which device branch they reach (the generic Hessian and jt_force /
row_dot for nv != 18, the uncached line search k_ls_eval for more than 32 work items, the second 32-lane chunk of the
limit compaction, the NQ = 6 and NQ = 4 Hessians of nv = 18), so that a model edit cannot silently drop the coverage.

On the A1 quadruped, teacher-forced poses with knees and hips beyond their ranges and joints in friction stick run
through the static helper-warp rollout, its one-warp twin (MJPC_B200_SHAPE=plain) and the generic instance
(MJPC_B200_NO_STATIC=1), each against fp64.  test_zz_report prints the largest error as a fraction of its bar per group.
"""
import numpy as np
import pytest

import joint_scenes as JS
from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

MOCAP = np.array([0, 0, 3, 1.0, 0, 0, 0])
RATIOS = {}
_CACHE = {}


def _ratio(group, err, bar):
    RATIOS[group] = max(RATIOS.get(group, 0.0), float(err) / bar)
    return err < bar


def _get(key, scene):
    if key not in _CACHE:
        from mujoco_mpc_b200.blob import to_blob
        from mujoco_mpc_b200.engine import Engine
        from oracle import pyoracle
        m = JS.compile_scene(scene.text())
        _CACHE[key] = (m, Engine(m, 8, 4), pyoracle.Oracle(to_blob(m), m, 64))
    return _CACHE[key]


def _dynamics(group, g, r, dt, force=True):
    scale = np.abs(r["qacc"]).max() + 1.0
    e = np.abs(g["qacc"] - r["qacc"]).max()
    assert _ratio(group + " qacc", e, 2e-3 * scale), (e, scale, g["qacc"], r["qacc"])
    e = np.abs(g["next_qvel"] - r["next_qvel"]).max()
    assert _ratio(group + " next_qvel", e, 2e-3 * dt * scale + 1e-5), e
    if force and r["nefc"]:
        fs = np.abs(r["efc_force"]).max() + 1.0
        e = np.abs(g["efc_force"] - r["efc_force"]).max()
        assert _ratio(group + " efc_force", e, 2e-3 * fs), (e, g["efc_force"], r["efc_force"])


def _compare(group, m, e, o, q, v, u, warmstart=None):
    g = e.step_debug(q, v, u, MOCAP, warmstart=warmstart)
    r = o.forward_debug(q, v, u, MOCAP, warmstart=warmstart)
    assert g["warning"] == r["warning"] == 0, (g["warning"], r["warning"])
    assert g["ncon"] == r["ncon"] and g["nefc"] == r["nefc"], (g["ncon"], r["ncon"], g["nefc"], r["nefc"])
    _dynamics(group, g, r, m.opt_timestep)
    return g, r


def _batched(group, m, e, o, poses):
    q = np.stack([p[1] for p in poses]); v = np.stack([p[2] for p in poses]); u = np.stack([p[3] for p in poses])
    t = np.zeros(len(poses))
    g = e.step_batch(q, v, u, MOCAP, t)
    r = o.step_batch(q, v, u, MOCAP, t)
    assert (g["nefc"] == r["nefc"]).all() and not g["warning"].any() and not r["warning"].any()
    for i in range(len(poses)):
        _dynamics(group + " (step_batch)", {k: g[k][i] for k in ("qacc", "next_qvel")},
                  {k: r[k][i] for k in ("qacc", "next_qvel")} | {"nefc": 0}, m.opt_timestep, force=False)


# ---------------------------------------------------------------------------------- closed-form scenes
SCENES = JS.closed_form_scenes()
CASES = [(k, p) for k, s in SCENES.items() for p in s.poses]


@pytest.mark.parametrize("key,pose", CASES, ids=[f"{k}-{p[0]}" for k, p in CASES])
def test_joint_scene_matches_fp64(key, pose):
    m, e, o = _get(key, SCENES[key])
    group = key.split("_")[0]
    _, q, v, u = pose
    g, r = _compare(group, m, e, o, q, v, u)
    # linear zone: the row carries exactly the friction loss (fp32 of it on the device)
    nf = int((m.dof_frictionloss > 0).sum()) if not m.opt_disable_frictionloss else 0
    fl = m.dof_frictionloss[m.dof_frictionloss > 0]
    for k in range(nf):
        if abs(r["efc_force"][k]) == fl[k]:
            assert abs(g["efc_force"][k]) == np.float32(fl[k]), (k, g["efc_force"][k], fl[k])


@pytest.mark.parametrize("key", list(SCENES))
def test_joint_scene_step_batch_matches_fp64(key):
    m, e, o = _get(key, SCENES[key])
    _batched(key.split("_")[0], m, e, o, SCENES[key].poses)


# ---------------------------------------------------------------------------------- flags
def _flag_compare(flag, iterations=None):
    m, e, o = _get(("flag", flag, iterations), JS.flag_scene(flag, iterations))
    q, v, u = JS.flag_pose()
    # warm start: the fp64 solution of the full solve of the unswitched scene
    ws = _get(("flag", None, None), JS.flag_scene(None))[2].forward_debug(q, v, u, MOCAP)["qacc"]
    return _compare("flags", m, e, o, q, v, u, warmstart=ws)


@pytest.mark.parametrize("flag", JS.FLAGS)
def test_flag_matches_fp64_and_changes_the_step(flag):
    # warmstart: with no Newton iterations the step is the starting point itself, the warm start (when it is on and
    # beats qacc_smooth, as the solution does) or qacc_smooth (when it is off), so the switch shows in the result
    iterations = 0 if flag == "warmstart" else None
    g0, r0 = _flag_compare(None, iterations)
    g1, r1 = _flag_compare(flag, iterations)
    # the switch moves the step by far more than the device's distance from fp64
    change = np.abs(r0["next_qvel"] - r1["next_qvel"]).max()
    err = max(np.abs(g0["next_qvel"] - r0["next_qvel"]).max(), np.abs(g1["next_qvel"] - r1["next_qvel"]).max())
    assert change > 1e-4 and change > 10 * err, (change, err)
    assert np.abs(g0["next_qvel"] - g1["next_qvel"]).max() > 0.5 * change
    if flag in ("frictionloss", "limit"):
        assert r1["nefc"] < r0["nefc"] and g1["nefc"] == r1["nefc"]


# ---------------------------------------------------------------------------------- device paths
PATHS = JS.path_scenes()


def _path_poses(m, n, seed, spread):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        q = spread * rng.uniform(-1, 1, m.nq)
        v = 0.5 * rng.standard_normal(m.nv) if i else 1e-3 * rng.standard_normal(m.nv)   # the first: near stick
        u = rng.uniform(-1, 1, m.nu) * (0.01 if i == 0 else 1)
        out.append((f"p{i}", q, v, u))
    return out


def _limit_rows(m, q):
    """Which limit rows (limited joints x lower / upper) exist at q; asserts that q is off every row boundary."""
    j = np.flatnonzero(m.jnt_limited)
    lo, hi, qj, mg = m.jnt_range[j, 0], m.jnt_range[j, 1], q[m.jnt_qposadr[j]], m.jnt_margin[j, None]
    d = np.stack([qj - lo, hi - qj], 1)
    assert d.size == 0 or np.abs(d - mg).min() > 5e-3, np.abs(d - mg).min()     # (module docstring)
    return d < mg


@pytest.mark.parametrize("key", [k for k in PATHS if not k.startswith("capacity")])
def test_path_scene_matches_fp64(key):
    scene = PATHS[key]
    m, e, o = _get(key, scene)
    nf = int((m.dof_frictionloss > 0).sum())
    nlimit = int(m.jnt_limited.sum())
    poses = _path_poses(m, 6, list(PATHS).index(key), 0.7 if nlimit else 1.5)
    for _, q, _, _ in poses:       # off the limit boundaries (every margin is 0 here)
        for j in np.flatnonzero(m.jnt_limited):
            a = m.jnt_qposadr[j]
            for b in m.jnt_range[j]:
                if abs(q[a] - b) < 5e-3:
                    q[a] = b + 1e-2 * (1 if q[a] >= b else -1)
    for name, q, v, u in poses:
        active = _limit_rows(m, q)
        nitem = nf + int(active.sum())
        if key == "chain10_floss":
            assert m.nv != 18 and nf == m.nv and nitem <= 32          # generic Hessian, cached line search
        elif key == "chain34_floss":
            assert m.nv != 18 and nf == m.nv and nitem > 32           # k_ls_eval
        elif key == "hinges40_limits":
            assert nlimit > 32 and active[32:].any() and active[:32].any()   # the second compaction chunk
        elif key == "chain18":
            assert m.nv == 18 and JS.nhpair(m) == 171                 # NQ = 6
        elif key == "branches3x6":
            assert m.nv == 18 and JS.nhpair(m) == 63                  # NQ = 4 (nhpair <= 128)
        _compare(key, m, e, o, q, v, u)
    _batched(key, m, e, o, poses)


@pytest.mark.parametrize("case", ["capacity_fits", "capacity_overflow"])
def test_joint_row_capacity_matches_fp64(case):
    """Friction-loss and joint-limit rows against the 96-row constraint buffer: the device drops the rows that do not
    fit and raises the warning, and so must the oracle; the warning makes the rollout a failure on both."""
    m, e, o = _get(case, PATHS[case])
    overflow = case.endswith("overflow")
    q, v, u = np.zeros(m.nq), 0.1 * np.ones(m.nv), np.zeros(m.nu)
    rows = int((m.dof_frictionloss > 0).sum()) + 2 * int(m.jnt_limited.sum())
    assert (rows > 96) == overflow and rows >= 96
    g = e.step_debug(q, v, u, MOCAP)
    r = o.forward_debug(q, v, u, MOCAP)
    assert g["warning"] == r["warning"] == int(overflow), (g["warning"], r["warning"])
    assert g["nefc"] == r["nefc"] == 96, (g["nefc"], r["nefc"])
    if not overflow:
        _dynamics("capacity", g, r, m.opt_timestep)
    sb = e.step_batch(q[None], v[None], u[None], MOCAP, np.zeros(1))
    ob = o.step_batch(q[None], v[None], u[None], MOCAP, np.zeros(1))
    assert int(sb["warning"][0]) == int(ob["warning"][0]) == int(overflow)
    H, P = 4, 2
    state = np.concatenate([q, v])
    knots = np.zeros((2, P, m.nu))
    kt = np.arange(P) * (H - 1) * m.opt_timestep
    ret, fail, _ = e.rollout_spline(state, 0.0, MOCAP, knots, kt, 0, H)
    ro = o.rollout_spline(state, 0.0, MOCAP, knots, kt, 0, H, nthreads=1, full=False)
    assert np.array_equal(fail.astype(bool), ro["failure"].astype(bool)) and bool(fail.all()) == overflow
    if not overflow:
        assert np.abs(ret - ro["returns"]).max() < 1e-4 * np.abs(ro["returns"]).max() + 1e-6


# ---------------------------------------------------------------------------------- mixed scene
def _mixed_pose(legs, z=0.163):
    q = np.concatenate([[0.01, -0.02, z], [1, 0, 0, 0], legs])
    v = np.concatenate([[0.1, -0.05, -0.2, 0.3, -0.2, 0.1], np.resize([0.4, -0.3, 0.2], len(legs))])
    return q, v, np.resize([0.3, -0.2, 0.1], len(legs))


@pytest.mark.parametrize("variant", ["cached", "uncached"])
def test_mixed_scene_matches_fp64(variant):
    """Friction loss, limits and floor contacts in one model, on both sides of the 32-item line-search split.
    cached: three legs on elliptic contacts with a 5 mm geom margin (one item per contact), whose friction rows sit at
    pos - margin = -5e-3, so their aref holds only while K = 0 for them; uncached: six legs on pyramidal contacts,
    every row its own item."""
    narrow = variant == "uncached"
    scene = JS.mixed_scene(narrow=True) if narrow else JS.mixed_scene(cone="elliptic", margin=0.005)
    m, e, o = _get(("mixed", variant), scene)
    legs = np.resize([0.07, -0.07, 0.04], 6) if narrow else np.array([0.53, 0.0, -0.49])
    q, v, u = _mixed_pose(legs)
    g, r = _compare("mixed", m, e, o, q, v, u)
    active = _limit_rows(m, q)
    assert r["ncon"] >= 1 and active.any() and int((m.dof_frictionloss > 0).sum()) == len(legs)
    assert (r["nefc"] > 32) == narrow and m.opt_cone == int(not narrow), r["nefc"]
    _batched("mixed", m, e, o, [("p", q, v, u)])
    # a short rollout: the rollout kernel runs the same rows
    state = np.concatenate([q, v])
    H, P = 4, 2
    knots = np.tile(u, (2, P, 1)) * np.array([1.0, -1.0])[:, None, None]
    kt = np.arange(P) * (H - 1) * m.opt_timestep
    ret, fail, _ = e.rollout_spline(state, 0.0, MOCAP, knots, kt, 0, H)
    ro = o.rollout_spline(state, 0.0, MOCAP, knots, kt, 0, H, nthreads=1, full=True)
    assert not fail.any() and not ro["failure"].any()
    tr = e.fetch_all()
    es = np.abs(tr["states"][:, :, : m.nq] - ro["states"][:, :, : m.nq]).max()
    assert _ratio("mixed rollout qpos", es, 1e-4), es
    assert _ratio("mixed rollout return", np.abs(ret - ro["returns"]).max(), 1e-4 * np.abs(ro["returns"]).max() + 1e-6)


@pytest.mark.parametrize("legs", [1, 3])
def test_pyramidal_condim6_contacts_on_hinged_legs(legs):
    """Hinged legs standing on condim-6 contacts in a pyramidal cone: 10 rows per contact, more than the six rows an
    elliptic contact has.  The generic J^T force (jt_force) once summed only the first six rows of each contact, which
    dropped the rolling-friction edges of every pyramidal condim-6 contact (qacc 1.7 off fp64 at |qacc| 38)."""
    m, e, o = _get(("pyramidal_condim6", legs), JS.mixed_scene(condim=6, joint_rows=False, legs=legs))
    q, v, u = _mixed_pose(np.resize([0.07, -0.07, 0.04], legs))
    assert m.nv != 18 and m.opt_cone == 0                       # the generic compact rows
    g, r = _compare("pyramidal condim 6", m, e, o, q, v, u)
    assert r["nefc"] == 10 * legs and np.abs(r["efc_force"].reshape(legs, 10)[:, 6:]).max() > 1e-3   # rolling edges carry force
    _batched("pyramidal condim 6", m, e, o, [("p", q, v, u)])


# ---------------------------------------------------------------------------------- A1 teacher-forced poses
def _a1_poses(m):
    """(name, qpos, qvel, ctrl): knees and hips beyond their ranges (in the air and standing), joints in friction
    stick (|torque| 40 * 0.003 = 0.12 below the 0.2 friction loss, velocities 1e-3)."""
    home = m.key_qpos[0].copy()
    rng = np.random.default_rng(11)
    lo, hi = m.jnt_range[1:, 0], m.jnt_range[1:, 1]
    out = []
    air = home.copy(); air[2] = 0.8
    q = air.copy(); q[7 + 2::3] = hi[2::3] + 0.05; q[7 + 1::3] = lo[1::3] - 0.04        # knees above, hips below
    out.append(("air_knees_hi_hips_lo", q, 0.3 * rng.standard_normal(m.nv), rng.uniform(-1, 1, m.nu)))
    q = air.copy(); q[7 + 2::3] = lo[2::3] - 0.03; q[7 + 0::3] = hi[0::3] + 0.02        # knees below, abduction above
    out.append(("air_knees_lo_abd_hi", q, 0.3 * rng.standard_normal(m.nv), rng.uniform(-1, 1, m.nu)))
    stand = home.copy(); stand[2] -= 0.012                                              # feet 2 mm into the floor
    v = np.zeros(m.nv); v[6:] = 1e-3 * rng.standard_normal(12)
    out.append(("standing_stick", stand, v, 0.003 * rng.uniform(-1, 1, m.nu)))
    q = stand.copy(); q[7 + 2] = hi[2] + 0.04; q[7 + 5] = hi[5] + 0.02                 # two knees beyond, standing
    out.append(("standing_knees_beyond", q, v, 0.003 * rng.uniform(-1, 1, m.nu)))
    for _, q, _, _ in out:
        _limit_rows(m, q)
    return out


@pytest.mark.parametrize("instance", ["static", "plain", "generic"])
def test_a1_teacher_forced_limits_and_stick(instance, monkeypatch):
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    from oracle import pyoracle
    if instance == "plain":
        monkeypatch.setenv("MJPC_B200_SHAPE", "plain")
    elif instance == "generic":
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model("quadruped")
    mocap = mocap_of(m)
    o = pyoracle.Oracle(to_blob(m), m, 64)
    e = Engine(m, 8, 4)
    shape = {"static": 1, "plain": 2, "generic": 0}[instance]
    group = f"A1 ({instance})"
    try:
        poses = _a1_poses(m)
        nf = int((m.dof_frictionloss > 0).sum())
        for name, q, v, u in poses:
            ref = o.step_batch(q[None], v[None], u[None], mocap, np.zeros(1))
            dev = e.step_batch(q[None], v[None], u[None], mocap, np.zeros(1))
            assert e.last_kernel_shape == min(shape, 1)
            assert int(dev["nefc"][0]) == int(ref["nefc"][0]) and int(dev["ncon"][0]) == int(ref["ncon"][0])
            assert _limit_rows(m, q).any() == ("stick" not in name)           # limit rows where the pose means them
            if "stick" in name:      # every friction-loss row in the quadratic zone
                f = o.forward_debug(q, v, u, mocap)["efc_force"][:nf]
                assert np.all(np.abs(f) < 0.999 * m.dof_frictionloss[6:]), f
            assert not dev["warning"].any() and not ref["warning"].any()
            _dynamics(group + " step", {k: dev[k][0] for k in ("qacc", "next_qvel")},
                      {k: ref[k][0] for k in ("qacc", "next_qvel")} | {"nefc": 0}, m.opt_timestep, force=False)
            # one rollout step from the pose (zero-order hold of the pose's ctrl): the rollout kernel's instance
            H, P = 2, 2
            knots = np.tile(u, (1, P, 1))
            kt = np.arange(P) * m.opt_timestep
            state = np.concatenate([q, v])
            ret, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 0, H)
            assert e.last_kernel_shape == shape and not fail.any()
            ro = o.rollout_spline(state, 0.0, mocap, knots, kt, 0, H, nthreads=1, full=True)
            tr = e.fetch_all()
            scale = np.abs(ref["qacc"][0]).max() + 1.0
            ev = np.abs(tr["states"][0, 1, m.nq:] - ro["states"][0, 1, m.nq:]).max()
            assert _ratio(group + " rollout next_qvel", ev, 2e-3 * m.opt_timestep * scale + 1e-5), (name, ev)
    finally:
        e.close()


def test_zz_report():
    """Largest error as a fraction of its bar, per group (printed with -s)."""
    for k in sorted(RATIOS):
        print(f"{k:50s} {RATIOS[k]:.3f}")
    assert all(v < 1 for v in RATIOS.values())
    for m, e, o in _CACHE.values():
        e.close()
    _CACHE.clear()
