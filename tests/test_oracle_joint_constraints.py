"""CPU: the fp64 oracle's joint-space laws (oracle/physics.h make_constraint, passive, actuation, the Newton solve and
the Euler step) against closed forms on the independent-unit scenes of tests/joint_scenes.py, and the MJCF loader's
refusals of what neither the device nor the oracle implements.

The device kernels and the oracle are transliterations of each other, so a law both misread passes the device-vs-oracle
tests; these checks restate the laws from MuJoCo's documentation instead.  Per dof (M = inertia + armature, closed form
in joint_scenes.Unit; tau = gravity + passive + actuation):

  passive      tau_p = -k (q - springref) - b v                   (slide / hinge)
  actuation    force = clamp(gain clamp(ctrl) + b0 + b1 gear q + b2 gear v),  tau_u = sum of gear force on the dof
  rows         friction loss: J = 1, K = 0;  limit: lower J = +1, dist = q - lo;  upper J = -1, dist = hi - q,
               present when dist < margin
  impedance    imp(dist - margin) with solimp's (dmin, dmax, width, mid, power)
  reference    K = 1 / (dmax^2 tc^2 dr^2), B = 2 / (dmax tc) (tc raised to 2 dt unless refsafe is off);
               solref < 0: K = -solref0 / dmax^2, B = -solref1 / dmax;  aref = -B J v - K imp (dist - margin)
  R, D         R = (1 - imp) / imp * invweight0 with invweight0 = 1 / M,  D = 1 / R
  forces       limit row: -D x for x = J a - aref < 0, else 0;  friction: -D x in |x| < R f (quadratic zone),
               -+f outside (linear zone)
  qacc         the a solving M (a - tau / M) = sum J force(a): with the set of quadratic rows Q and linear rows L,
               (M + sum_Q D) a = tau + sum_Q D J aref + sum_L J force; e.g. one friction row in the quadratic zone
               a = (tau + D aref) / (M + D), in the linear zone a = (tau -+ f) / M
  next_qvel    v + h M a / (M + h b) with eulerdamp (implicit damping), v + h a without.
Every zone assignment of a dof's rows is tried; exactly one is consistent.
"""
import itertools
import re

import numpy as np
import pytest

import joint_scenes as JS

SOLREF0, SOLIMP0 = [0.02, 1.0], [0.9, 0.95, 0.001, 0.5, 2.0]
MINIMP, MAXIMP = 1e-4, 0.9999


def _attrs(s):
    return {k: np.array([float(x) for x in v.split()]) for k, v in re.findall(r'(\w+)="([^"]*)"', s)}


def impedance(solimp, x_pos):
    dmin, dmax = (min(MAXIMP, max(MINIMP, s)) for s in solimp[:2])
    width, mid, power = max(0.0, solimp[2]), min(MAXIMP, max(MINIMP, solimp[3])), max(1.0, solimp[4])
    if dmin == dmax or width <= 1e-15:
        return 0.5 * (dmin + dmax)
    x = abs(x_pos) / width
    if x >= 1:
        return dmax
    if power == 1:
        y = x
    elif x <= mid:
        y = x ** power / mid ** (power - 1)
    else:
        y = 1 - (1 - x) ** power / (1 - mid) ** (power - 1)
    return dmin + y * (dmax - dmin)


def kb(solref, solimp, refsafe):
    dmax = min(MAXIMP, max(MINIMP, solimp[1]))
    if solref[0] > 0:
        tc = max(solref[0], 2 * JS.DT) if refsafe else solref[0]
        return 1 / (dmax * dmax * tc * tc * solref[1] ** 2), 2 / (dmax * tc)
    return -solref[0] / dmax ** 2, -solref[1] / dmax


class Row:
    def __init__(self, J, dist, margin, solref, solimp, M, v, floss, refsafe):
        K, B = kb(solref, solimp, refsafe)
        imp = impedance(solimp, dist - margin)
        if floss:
            K = 0.0
        self.J, self.f = J, floss
        self.aref = -B * J * v - K * imp * (dist - margin)
        self.R = max(1e-15, (1 - imp) / imp / M)
        self.D = 1 / self.R

    def force(self, a):
        x = self.J * a - self.aref
        if self.f:
            return float(np.clip(-self.D * x, -self.f, self.f))
        return -self.D * x if x < 0 else 0.0


def solve_dof(M, tau, rows):
    """The 1-D constraint problem by zone enumeration (module docstring)."""
    found = []
    for zones in itertools.product(*[(("q", 0), ("l", 1), ("l", -1)) if r.f else (("q", 0), ("off", 0)) for r in rows]):
        lhs, rhs = M, tau
        for r, (z, s) in zip(rows, zones):
            if z == "q":
                lhs += r.D; rhs += r.D * r.J * r.aref
            elif z == "l":
                rhs += r.J * s * r.f
        a = rhs / lhs
        ok = True
        for r, (z, s) in zip(rows, zones):
            x = r.J * a - r.aref
            if r.f:
                ok &= (abs(x) <= r.R * r.f) if z == "q" else (s * x <= -r.R * r.f)
            else:
                ok &= (x < 0) if z == "q" else (x >= 0)
        if ok:
            found.append(a)
    assert len(found) >= 1 and np.ptp(found) < 1e-12 * (1 + abs(found[0])), found
    return found[0]


def closed_form(scene, qpos, qvel, ctrl):
    """qacc, next_qvel, qfrc_smooth and the efc_force rows (in the oracle's row order) of an independent-unit scene."""
    off = {k for k in ("frictionloss", "limit", "eulerdamp", "refsafe") if f'{k}="disable"' in scene.flags}
    qa, va = 0, 0
    per_dof, frows, lrows = [], [], []
    for ui, u in enumerate(scene.units):
        a = _attrs(u.attrs)
        arm, damp = float(a.get("armature", [0])[0]), float(a.get("damping", [0])[0])
        Ms = u.inertia() + arm
        tau = u.gravity() - damp * qvel[va:va + u.nv]
        if u.kind in ("slide", "hinge"):
            q, v = qpos[qa], qvel[va]
            tau[0] -= float(a.get("stiffness", [0])[0]) * (q - float(a.get("springref", [0])[0]))
            for i, act in enumerate(scene.actuators):
                if act.joint == ui:
                    tau[0] += act.gear * act.force(ctrl[i], q, v)
        for k in range(u.nv):
            rows = []
            if "frictionloss" in a and "frictionloss" not in off:
                r = Row(1.0, 0.0, 0.0, a.get("solreffriction", SOLREF0), a.get("solimpfriction", SOLIMP0), Ms[k],
                        qvel[va + k], float(a["frictionloss"][0]), "refsafe" not in off)
                rows.append(r); frows.append(r)
            if "range" in a and "limit" not in off:
                lo, hi = a["range"]
                margin = float(a.get("margin", [0])[0])
                for J, dist in ((1.0, qpos[qa] - lo), (-1.0, hi - qpos[qa])):
                    if dist < margin:
                        r = Row(J, dist, margin, a.get("solreflimit", SOLREF0), a.get("solimplimit", SOLIMP0), Ms[k],
                                qvel[va + k], 0.0, "refsafe" not in off)
                        rows.append(r); lrows.append(r)
            per_dof.append((Ms[k], tau[k], damp, rows, qvel[va + k]))
        qa += u.nq; va += u.nv
    qacc, nxt, smooth, acc = [], [], [], {}
    for M, tau, b, rows, v in per_dof:
        a = solve_dof(M, tau, rows)
        for r in rows:
            acc[id(r)] = r.force(a)
        qacc.append(a); smooth.append(tau)
        nxt.append(v + JS.DT * (a if "eulerdamp" in off else M * a / (M + JS.DT * b)))
    efc = np.array([acc[id(r)] for r in frows + lrows])
    return np.array(qacc), np.array(nxt), np.array(smooth), efc, frows + lrows


SCENES = JS.closed_form_scenes()
CASES = [(k, p) for k, s in SCENES.items() for p in s.poses]
_CACHE = {}


def _oracle(key):
    if key not in _CACHE:
        from mujoco_mpc_b200.blob import to_blob
        from oracle import pyoracle
        m = JS.compile_scene(SCENES[key].text())
        _CACHE[key] = (m, pyoracle.Oracle(to_blob(m), m, 64))
    return _CACHE[key]


MOCAP = np.array([0, 0, 3, 1.0, 0, 0, 0])


@pytest.mark.parametrize("key,pose", CASES, ids=[f"{k}-{p[0]}" for k, p in CASES])
def test_oracle_joint_laws_closed_form(oracle_lib, key, pose):
    scene = SCENES[key]
    m, o = _oracle(key)
    _, qpos, qvel, ctrl = pose
    r = o.forward_debug(qpos, qvel, ctrl, MOCAP)
    qacc, nxt, smooth, efc, rows = closed_form(scene, qpos, qvel, ctrl)
    assert r["warning"] == 0 and r["nefc"] == len(rows), (r["nefc"], len(rows))
    scale = np.abs(qacc).max() + 1
    assert np.abs(r["qfrc_smooth"] - smooth).max() < 1e-12 * (np.abs(smooth).max() + 1), (r["qfrc_smooth"], smooth)
    assert np.abs(r["qacc"] - qacc).max() < 1e-9 * scale, (r["qacc"], qacc)
    assert np.abs(r["next_qvel"] - nxt).max() < 1e-9 * scale * JS.DT + 1e-12, (r["next_qvel"], nxt)
    if len(rows):
        assert np.abs(r["efc_force"] - efc).max() < 1e-9 * (np.abs(efc).max() + 1), (r["efc_force"], efc)


def test_closed_forms_reach_every_zone(oracle_lib):
    """The poses put friction rows in both zones (both signs of the linear one), limit rows active and inactive, and
    the refsafe / flag variants change the result."""
    zones = set()
    for key, scene in SCENES.items():
        for _, qpos, qvel, ctrl in scene.poses:
            qacc, _, _, efc, rows = closed_form(scene, qpos, qvel, ctrl)
            for r, f in zip(rows, efc):
                if r.f:
                    zones.add("linear+" if f == r.f else "linear-" if f == -r.f else "quadratic")
                else:
                    zones.add("limit active" if f > 0 else "limit inactive")
    assert zones == {"linear+", "linear-", "quadratic", "limit active", "limit inactive"}, zones
    for a, b in (("limits", "limits_refsafe_off"), ("limits", "limits_flag_off"), ("friction", "friction_flag_off"),
                 ("passive", "passive_eulerdamp_off")):
        ma, oa = _oracle(a)
        mb, ob = _oracle(b)
        _, q, v, u = SCENES[a].poses[-1]
        ra, rb = oa.forward_debug(q, v, u, MOCAP), ob.forward_debug(q, v, u, MOCAP)
        assert np.abs(ra["next_qvel"] - rb["next_qvel"]).max() > 1e-3, (a, b)


def test_linear_zone_force_is_frictionloss(oracle_lib):
    """At rest above the threshold the slide's friction row carries exactly -sign(tau) f and qacc = (tau -+ f) / M."""
    m, o = _oracle("friction")
    for name, q, v, u in SCENES["friction"].poses:
        if not name.startswith("rest_above"):
            continue
        r = o.forward_debug(q, v, u, MOCAP)
        tau = u[0]
        assert r["efc_force"][0] == -np.sign(tau) * 0.5
        assert abs(r["qacc"][0] - (tau - np.sign(tau) * 0.5) / 2.0) < 1e-12


# ---------------------------------------------------------------------------------------------- loader refusals
def _xml(joint='type="hinge"', actuator="", flag=""):
    return f"""<mujoco><option>{flag}</option><worldbody><body><joint name="j" {joint}/>
      <geom type="sphere" size="0.1"/></body></worldbody><actuator>{actuator}</actuator></mujoco>"""


REFUSALS = {
    "limited_ball": (_xml('type="ball" limited="true" range="0 1"'), "ball joint"),
    "autolimited_ball": (_xml('type="ball" range="0 1"'), "ball joint"),
    "ball_stiffness": (_xml('type="ball" stiffness="3"'), "stiffness"),
    "free_stiffness": (_xml('type="free" stiffness="3"'), "stiffness"),
    "actuator_on_ball": (_xml('type="ball"', '<motor joint="j"/>'), "ball or free joint"),
    "actuator_on_free": (_xml('type="free"', '<motor joint="j"/>'), "ball or free joint"),
    "gear_vector": (_xml('type="hinge"', '<motor joint="j" gear="1 2 3"/>'), "gear vector"),
    "gaintype_affine": (_xml('type="hinge"', '<general joint="j" gaintype="affine" gainprm="1 2 3"/>'), "gaintype"),
    "dyntype_filter": (_xml('type="hinge"', '<general joint="j" dyntype="filter" dynprm="0.1"/>'), "dyntype"),
    "dyntype_integrator": (_xml('type="hinge"', '<general joint="j" dyntype="integrator"/>'), "dyntype"),
    "position_timeconst": (_xml('type="hinge"', '<position joint="j" kp="3" timeconst="0.1"/>'), "timeconst"),
    "damper": (_xml('type="hinge"', '<damper joint="j" kv="1" ctrlrange="0 1"/>'), "<damper>"),
    "intvelocity": (_xml('type="hinge"', '<intvelocity joint="j" kp="1" actrange="-1 1"/>'), "<intvelocity>"),
    "cylinder": (_xml('type="hinge"', '<cylinder joint="j"/>'), "<cylinder>"),
    "muscle": (_xml('type="hinge"', '<muscle joint="j"/>'), "<muscle>"),
    "biastype_muscle": (_xml('type="hinge"', '<general joint="j" biastype="muscle"/>'), "biastype"),
    "site_transmission": (_xml('type="hinge"', '<motor site="s"/>'), "transmission"),
    "joint_actuatorfrcrange": (_xml('type="hinge" actuatorfrcrange="-1 1"'), "actuatorfrcrange"),
    "joint_actuatorgravcomp": (_xml('type="hinge" actuatorgravcomp="true"'), "actuatorgravcomp"),
    "position_inheritrange": (_xml('type="hinge" range="-1 1"', '<position joint="j" kp="3" inheritrange="1"/>'),
                              "inheritrange"),
    "general_actdim": (_xml('type="hinge"', '<general joint="j" actdim="1"/>'), "actdim"),
    "general_actlimited": (_xml('type="hinge"', '<general joint="j" actlimited="true" actrange="-1 1"/>'), "actlimited"),
    "flag_gravity": (_xml(flag='<flag gravity="disable"/>'), "gravity"),
    "flag_passive": (_xml(flag='<flag passive="disable"/>'), "passive"),
    "flag_override": (_xml(flag='<flag override="enable"/>'), "override"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_loader_refuses_unimplemented_features(case):
    from mujoco_mpc_b200.mjcf import compile_xml
    text, word = REFUSALS[case]
    with pytest.raises(NotImplementedError, match=re.escape(word)):
        compile_xml(text)


def test_loader_accepts_what_is_implemented():
    """The neighbours of the refusals still compile, with the values the device reads."""
    from mujoco_mpc_b200.mjcf import compile_xml
    m = compile_xml(_xml('type="ball" frictionloss="0.1" damping="0.2" armature="0.3"',
                         flag='<flag energy="enable" frictionloss="disable" refsafe="enable"/>'))
    assert m.nv == 3 and np.all(m.dof_frictionloss == 0.1) and m.opt_disable_frictionloss == 1 and m.opt_disable_refsafe == 0
    m = compile_xml(_xml('type="hinge"', '<motor joint="j" gear="-2 0 0 0 0 0"/>'
                                         '<general joint="j" gaintype="fixed" dyntype="none" biastype="affine" '
                                         'gainprm="3" biasprm="1 2 3"/>'))
    assert m.nu == 2 and list(m.actuator_gear) == [-2, 1] and list(m.actuator_biastype) == [0, 1]
    assert list(m.actuator_biasprm[1]) == [1, 2, 3] and m.actuator_gainprm[1][0] == 3


@pytest.mark.parametrize("name", ["particle", "cartpole", "quadruped", "humanoid", "humanoid_track", "shadow_reorient"])
def test_shipped_models_compile(name):
    from mujoco_mpc_b200 import models
    m = models.load(name)
    assert m.nv > 0 and m.nu > 0
