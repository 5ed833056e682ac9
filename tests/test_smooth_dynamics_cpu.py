"""CPU: the smooth dynamics - kinematics, composite inertia, the bias force and the Euler step - of the fp64 oracle
against an independent fp64 restatement, on the purpose-built scenes of tests/smooth_scenes.py.

The oracle (oracle/physics.h) and the device kernels are transliterations of the same recursions (composite rigid
bodies for qM, recursive Newton-Euler over cdof / cdof_dot for qfrc_bias), so an error they share passes every
device-vs-oracle test.  The restatement here shares none of those recursions:

  kinematics   refmath.kinematics (body by body in world coordinates), with every quaternion normalised first as
               MuJoCo's mju_normalize4 does (an all-zero one becomes the identity);
  qM           refmath: sum_b J_b^T diag(m_b, I_b) J_b with world-frame Jacobians J_b at each body's centre of mass,
               plus armature;
  qfrc_bias    Newton-Euler per body: sum_b J_b^T [m_b (a_b - g); I_b wdot_b + w_b x I_b w_b], where (a_b, wdot_b) =
               Jdot_b v is each body's acceleration at qacc = 0, taken as a central difference of J_b(q (+) s v) v
               over s = +-eps, +-2 eps (Richardson-extrapolated; (+) is estimator.integrate_pos);
  qacc         M^-1 (-qfrc_bias) (the scenes have no passive, actuator or constraint force);
  Euler        v' = v + h qacc, q' = integrate_pos(q, v', h).

Difference bound: eps moves the state by STEP = 1e-3 (radians or metres per unit of |v|_inf).  The Richardson
estimate's truncation error is O(STEP^4) ~ 1e-12 relative, and its round-off is about 1e-16 |J v| / eps.  The test
states the bound by recomputing Jdot v with 2 eps: the two estimates must agree to JDOT_BOUND = 1e-10 of the bias
scale, ten times below the 1e-9 relative at which the oracle is compared.

The restatement itself is pinned to closed forms: Euler's equations of the torque-free asymmetric top in its principal
frame, qacc = g . axis on a slide, the offset-com hinge pendulum and the textbook M(q), C(q, qdot) of the planar double
pendulum.
"""
import numpy as np
import pytest

import smooth_scenes as S

STEP = 1e-3
JDOT_BOUND = 1e-10
TOL = 1e-9


def _normalize4(q):
    """mju_normalize4: unit quaternion, the identity when |q| < 1e-15."""
    n = np.linalg.norm(q)
    return np.array([1.0, 0, 0, 0]) if n < 1e-15 else np.asarray(q, float) / n


def normalize_qpos(m, qpos):
    from mujoco_mpc_b200.mjcf import JNT_BALL, JNT_FREE
    q = np.array(qpos, float)
    for j in range(m.njnt):
        a = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == JNT_FREE else 0)
        if m.jnt_type[j] in (JNT_FREE, JNT_BALL):
            q[a:a + 4] = _normalize4(q[a:a + 4])
    return q


def split_mocap(m, mocap):
    if mocap is None or m.nmocap == 0:
        return m.mocap_pos0, m.mocap_quat0
    mc = np.asarray(mocap, float).reshape(m.nmocap, 7)
    return mc[:, :3].copy(), np.array([_normalize4(x) for x in mc[:, 3:]])


def mocap_input(m, mocap):
    """The mocap array the oracle and the device take: the case's, or the model's poses."""
    if mocap is not None:
        return np.asarray(mocap, float)
    return np.concatenate([np.concatenate([m.mocap_pos0[i], m.mocap_quat0[i]]) for i in range(m.nmocap)]) \
        if m.nmocap else np.zeros(0)


def _jacobians(m, q, mp, mq):
    from mujoco_mpc_b200 import refmath
    kin = refmath.kinematics(m, q, mp, mq)
    return kin, {b: refmath.body_jacobian(m, kin, b, kin["xipos"][b]) for b in range(1, m.nbody)}


def _jdot_v(m, q, v, mp, mq, eps):
    """Richardson-extrapolated central difference of J_b(q (+) s v) v at s = 0, per body: [nbody-1, 6]."""
    from mujoco_mpc_b200.estimator import integrate_pos

    def Jv(s):
        _, J = _jacobians(m, integrate_pos(m, q, v, s), mp, mq)
        return np.array([J[b] @ v for b in range(1, m.nbody)])
    d1 = (Jv(eps) - Jv(-eps)) / (2 * eps)
    d2 = (Jv(2 * eps) - Jv(-2 * eps)) / (4 * eps)
    return (4 * d1 - d2) / 3, (d1, d2)


def restatement(m, qpos, qvel, mocap, eps_scale=1.0):
    """The fp64 restatement of one smooth step (module docstring)."""
    from mujoco_mpc_b200 import refmath
    from mujoco_mpc_b200.estimator import integrate_pos
    q, v = normalize_qpos(m, qpos), np.asarray(qvel, float)
    mp, mq = split_mocap(m, mocap)
    M, J = refmath.mass_matrix_and_jacobians(m, q, mp, mq)
    kin = refmath.kinematics(m, q, mp, mq)
    eps = eps_scale * STEP / max(1.0, np.abs(v).max())
    jdv, _ = _jdot_v(m, q, v, mp, mq, eps)
    g = np.asarray(m.opt_gravity, float)
    bias = np.zeros(m.nv)
    for b in range(1, m.nbody):
        Jb = J[b]
        w = Jb[3:6] @ v
        Iw = kin["ximat"][b] @ np.diag(m.body_inertia[b]) @ kin["ximat"][b].T
        f = m.body_mass[b] * (jdv[b - 1, :3] - g)
        t = Iw @ jdv[b - 1, 3:] + np.cross(w, Iw @ w)
        bias += Jb[:3].T @ f + Jb[3:].T @ t
    qacc = np.linalg.solve(M, -bias) if m.nv else np.zeros(0)
    v1 = v + m.opt_timestep * qacc
    q1 = integrate_pos(m, q, v1, m.opt_timestep)
    # subtree centres of mass (parents precede children in body order)
    ms = m.body_mass[:, None] * kin["xipos"]
    mass = np.array(m.body_mass, float)
    for b in range(m.nbody - 1, 0, -1):
        ms[m.body_parentid[b]] += ms[b]; mass[m.body_parentid[b]] += mass[b]
    scom = np.where(mass[:, None] < 1e-15, kin["xipos"], ms / np.maximum(mass, 1e-300)[:, None])
    return dict(qM=M, qfrc_bias=bias, qacc=qacc, xpos=kin["xpos"], subtree_com=scom, next_qpos=q1, next_qvel=v1,
                kin=kin, J=J, jdot_v=jdv)


SCENES = S.scenes()
CASES = [(k, c) for k, s in SCENES.items() for c in s.cases]
_CACHE = {}


def _model(key):
    if key not in _CACHE:
        from mujoco_mpc_b200.blob import to_blob
        from oracle import pyoracle
        m = SCENES[key].compile()
        _CACHE[key] = (m, pyoracle.Oracle(to_blob(m), m, 64))
    return _CACHE[key]


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.abs(a - b).max(initial=0.0) <= tol * (np.abs(b).max(initial=0.0) + 1.0)


# ---------------------------------------------------------------------------------------------- the restatement
def test_scenes_cover_the_tree_features():
    """Every feature the scenes exist for is present in the compiled models (a scene edit cannot drop one)."""
    from mujoco_mpc_b200.mjcf import JNT_BALL, JNT_FREE, JNT_HINGE, JNT_SLIDE
    ms = {k: _model(k)[0] for k in SCENES}
    top = ms["free_top"]
    assert np.abs(np.abs(top.body_iquat[1]) - [1, 0, 0, 0]).max() > 0.1 and np.abs(top.body_ipos[1]).min() > 0
    assert len(set(np.round(top.body_inertia[1], 6))) == 3
    bp = ms["ball_pendulum"]
    assert bp.jnt_type[0] == JNT_BALL and np.abs(bp.jnt_pos[0]).max() > 0 and bp.jnt_type[1] == JNT_HINGE
    mj = ms["multi_joint"]
    assert list(mj.jnt_type[mj.body_jntadr[1]:][:3]) == [JNT_SLIDE, JNT_HINGE, JNT_HINGE] and mj.body_jntnum[1] == 3
    assert list(mj.jnt_type[mj.body_jntadr[2]:][:2]) == [JNT_HINGE, JNT_BALL] and mj.body_jntnum[2] == 2
    assert np.abs(ms["joint_ref"].qpos0).min() > 0.2
    oc = ms["odd_chain"]
    assert oc.body_mocapid[1] == 0 and oc.body_jntnum[2] == 1 and oc.body_parentid[2] == 1
    welded = [b for b in range(2, oc.nbody) if oc.body_jntnum[b] == 0]
    assert any(oc.body_mass[b] > 0 for b in welded) and sum(oc.body_mass[b] == 0 for b in welded) >= 2
    assert (oc.body_subtreemass < 1e-15).any()
    assert (ms["forest"].body_parentid == 0).sum() >= 4          # world + three trees
    w = ms["wide"]
    depth = np.zeros(w.nbody, int)
    for b in range(1, w.nbody):
        depth[b] = depth[w.body_parentid[b]] + 1
    assert np.bincount(depth).max() >= 40 and 33 <= w.nv <= 64
    assert {JNT_FREE, JNT_BALL} <= set(ms["quat_edges"].jnt_type) and ms["quat_edges"].nmocap == 1


@pytest.mark.parametrize("key,case", CASES, ids=[f"{k}-{c[0]}" for k, c in CASES])
def test_oracle_matches_restatement(oracle_lib, key, case):
    m, o = _model(key)
    _, qpos, qvel, mocap = case
    ref = restatement(m, qpos, qvel, mocap)
    # the difference bound (module docstring): Jdot v at eps and at 2 eps agree to JDOT_BOUND of the bias scale
    alt = restatement(m, qpos, qvel, mocap, eps_scale=2.0)
    scale = np.abs(ref["qfrc_bias"]).max() + np.abs(ref["qM"]).max() * np.abs(ref["qacc"]).max() + 1.0
    assert np.abs(ref["qfrc_bias"] - alt["qfrc_bias"]).max() < JDOT_BOUND * scale
    r = o.forward_debug(qpos, qvel, np.zeros(m.nu), mocap_input(m, mocap))
    assert r["warning"] == 0 and r["nefc"] == 0 and r["ncon"] == 0
    for k in ("qM", "qacc", "xpos", "subtree_com", "next_qvel"):
        assert _close(r[k], ref[k]), (k, np.abs(r[k] - ref[k]).max(), r[k], ref[k])
    assert np.abs(r["qfrc_bias"] - ref["qfrc_bias"]).max() <= TOL * scale, (r["qfrc_bias"], ref["qfrc_bias"])
    assert _close(r["next_qpos"], ref["next_qpos"]), (r["next_qpos"], ref["next_qpos"])


def test_far_cases_translate(oracle_lib):
    """The far-from-origin cases and their twin at the origin: the same qM, bias, qacc and velocity step, and
    positions moved by the translation, in the restatement and in the fp64 oracle."""
    m, o = _model("far")
    base = {c[0]: c for c in SCENES["far"].cases}["origin"]
    r0 = o.forward_debug(base[1], base[2], np.zeros(0), np.zeros(0))
    s0 = restatement(m, base[1], base[2], None)
    for name, q, v, _ in SCENES["far"].cases:
        x = S.far_twin(name)
        if not x:
            continue
        r, s = o.forward_debug(q, v, np.zeros(0), np.zeros(0)), restatement(m, q, v, None)
        for k in ("qM", "qacc", "next_qvel", "qfrc_bias"):
            for a, b in ((r[k], r0[k]), (s[k], s0[k])):
                assert _close(a, b, 1e-12 * x), (name, k, np.abs(a - b).max())
        for a, b in ((r["next_qpos"], r0["next_qpos"]), (s["next_qpos"], s0["next_qpos"])):
            d = a - b
            assert abs(d[0] - x) < 1e-12 * x and np.abs(d[1:]).max() < 1e-12 * x, (name, d)


def test_restatement_has_no_velocity_or_acceleration_shortcut():
    """The restatement's bias is not the gravity part alone: on the fast top the velocity terms dominate."""
    m = _model("free_top")[0]
    c = {c[0]: c for c in SCENES["free_top"].cases}
    fast, rest = restatement(m, *c["fast_3.1"][1:]), restatement(m, *c["at_rest"][1:])
    assert np.abs(fast["qfrc_bias"] - rest["qfrc_bias"]).max() > 100 * np.abs(rest["qfrc_bias"]).max()


# ---------------------------------------------------------------------------------------------- closed forms
@pytest.mark.parametrize("case", [c[0] for c in S.free_top().cases])
def test_restatement_euler_equations_of_the_top(case):
    """Torque-free asymmetric top: in the principal frame I wdot = -w x I w; the origin of the free joint accelerates
    as g - wdot x r - w x (w x r), r = xipos - xpos (the centre of mass falls freely)."""
    from mujoco_mpc_b200.mjcf import quat2mat
    m = _model("free_top")[0]
    _, q, v, _ = {c[0]: c for c in SCENES["free_top"].cases}[case]
    ref = restatement(m, q, v, None)
    Ri = quat2mat(m.body_iquat[1])
    I = m.body_inertia[1]
    wp = Ri.T @ v[3:6]
    wdot = Ri @ (-np.cross(wp, I * wp) / I)
    R = quat2mat(_normalize4(q[3:7]))
    r = ref["kin"]["xipos"][1] - ref["kin"]["xpos"][1]
    ww, wdw = R @ v[3:6], R @ wdot
    lin = m.opt_gravity - np.cross(wdw, r) - np.cross(ww, np.cross(ww, r))
    assert _close(ref["qacc"], np.concatenate([lin, wdot])), (ref["qacc"], lin, wdot)


def test_restatement_slide_under_gravity():
    from mujoco_mpc_b200.mjcf import quat2mat
    m = _model("slide_gravity")[0]
    axis = quat2mat(m.body_quat[1]) @ S.SLIDE_AXIS
    for _, q, v, _ in SCENES["slide_gravity"].cases:
        ref = restatement(m, q, v, None)
        assert _close(ref["qacc"], [m.opt_gravity @ axis]), (ref["qacc"], m.opt_gravity @ axis)


def test_restatement_hinge_pendulum():
    p, m = S.PEND, _model("hinge_pendulum")[0]
    g = -m.opt_gravity[2]
    for _, q, v, _ in SCENES["hinge_pendulum"].cases:
        ref = restatement(m, q, v, None)
        want = -p["m"] * g * p["d"] * np.cos(q[0] - p["ref"]) / (p["Ixx"] + p["m"] * p["d"] ** 2 + p["arm"])
        assert _close(ref["qacc"], [want]), (ref["qacc"], want)


def test_restatement_double_pendulum():
    """M(q) and C(q, qdot) qdot of the planar double pendulum (relative angle t2):
    M11 = I1 + I2 + m1 c1^2 + m2 (l1^2 + c2^2 + 2 l1 c2 cos t2), M12 = I2 + m2 (c2^2 + l1 c2 cos t2),
    M22 = I2 + m2 c2^2;  C qdot = [-m2 l1 c2 sin t2 (2 t1' t2' + t2'^2), m2 l1 c2 sin t2 t1'^2]."""
    p, m = S.DP, _model("double_pendulum")[0]
    for _, q, v, _ in SCENES["double_pendulum"].cases:
        ref = restatement(m, q, v, None)
        c2, s2 = np.cos(q[1]), np.sin(q[1])
        k = p["m2"] * p["l1"] * p["c2"]
        M = np.array([[p["I1"] + p["I2"] + p["m1"] * p["c1"] ** 2 + p["m2"] * (p["l1"] ** 2 + p["c2"] ** 2) + 2 * k * c2,
                       p["I2"] + p["m2"] * p["c2"] ** 2 + k * c2],
                      [0.0, p["I2"] + p["m2"] * p["c2"] ** 2]])
        M[1, 0] = M[0, 1]
        C = np.array([-k * s2 * (2 * v[0] * v[1] + v[1] ** 2), k * s2 * v[0] ** 2])
        assert _close(ref["qM"], M), (ref["qM"], M)
        assert _close(ref["qfrc_bias"], C), (ref["qfrc_bias"], C)


def test_quaternion_inputs_normalise_like_mujoco(oracle_lib):
    """A non-unit or negative-w quaternion stands for its normalised rotation, and an all-zero one for the identity:
    the step from a scaled copy of the state is the step from the state, and next_qpos holds unit quaternions even
    where the angular velocity is zero."""
    from mujoco_mpc_b200.mjcf import JNT_BALL, JNT_FREE
    m, o = _model("quat_edges")
    quats = [m.jnt_qposadr[j] + (3 if m.jnt_type[j] == JNT_FREE else 0) for j in range(m.njnt)
             if m.jnt_type[j] in (JNT_FREE, JNT_BALL)]
    for name, q, v, mocap in SCENES["quat_edges"].cases:
        r = o.forward_debug(q, v, np.zeros(0), mocap_input(m, mocap))
        unit = o.forward_debug(normalize_qpos(m, q), v, np.zeros(0), mocap_input(m, mocap))
        for k in ("qM", "qfrc_bias", "qacc", "next_qvel", "next_qpos"):
            assert _close(r[k], unit[k], 1e-14), (name, k)
        for a in quats:
            assert abs(np.linalg.norm(r["next_qpos"][a:a + 4]) - 1) < 1e-15, (name, a, r["next_qpos"][a:a + 4])


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_task_models_extreme_states_match_restatement(oracle_lib, name):
    """The airborne extreme states the device's static instances run (smooth_scenes.extreme_states): the fp64 oracle's
    qM and qfrc_bias against the restatement."""
    from conftest import get_model, mocap_of
    from mujoco_mpc_b200.blob import to_blob
    from oracle import pyoracle
    m = get_model(name)
    o = pyoracle.Oracle(to_blob(m), m, 64)
    mc = mocap_of(m)
    for case, q, v in S.extreme_states(m):
        ref = restatement(m, q, v, mc if m.nmocap else None)
        r = o.forward_debug(q, v, np.zeros(m.nu), mc)
        assert r["ncon"] == 0, case
        scale = np.abs(ref["qfrc_bias"]).max() + np.abs(ref["qM"]).max() * np.abs(ref["qacc"]).max() + 1.0
        assert _close(r["qM"], ref["qM"]), (case, np.abs(r["qM"] - ref["qM"]).max())
        assert np.abs(r["qfrc_bias"] - ref["qfrc_bias"]).max() <= TOL * scale, (case, r["qfrc_bias"], ref["qfrc_bias"])
        assert _close(r["xpos"], ref["xpos"]) and _close(r["subtree_com"], ref["subtree_com"]), case
