"""Purpose-built scenes for the contact constraint solve (oracle/physics.h make_constraint / solve_constraints,
csrc/dev_physics.cuh k_update_constraint, the Hessians, k_line_search, k_solve).

Every scene is a small model whose contacts are against the static floor or between free bodies, built for each cone
(pyramidal, elliptic) and impratio (1, 10, 100).  A state is (name, qpos, qvel).  Box-box pairs are not collided by
the narrow phase, so contacts between moving bodies are sphere-box and sphere-sphere.

Each Scene records which device path it must reach (`path`, asserted from the host-side model by the tests):
  generic   the generic Hessian and jt_force (nv != 18);
  nq4       hessian_dense_reg<SP, 18, 4> (nv = 18, nhpair <= 128), with contacts between moving bodies (ndrow > 0);
  nq6       hessian_dense_reg<SP, 18, 6> (nv = 18, nhpair 171);
and (`cached`) whether its line search is cached (at most 32 work items: one per friction-loss or limit row, one per elliptic
contact, one per pyramidal or frictionless row) or uncached (k_ls_eval).

Shared by tests/test_constraint_solve_cpu.py (the fp64 oracle against a restatement of the convex problem) and
tests/test_gpu_constraint_solve.py (the device against the fp64 oracle).
"""
import numpy as np

G = 9.81
DT = 0.002
CONES = ("pyramidal", "elliptic")
IMPRATIOS = (1, 10, 100)
# default soft-contact parameters (solref 0.02 1, solimp 0.9 0.95 0.001 0.5 2)
TC, DR, D0, DMAX, WIDTH, MID, POWER = 0.02, 1.0, 0.9, 0.95, 0.001, 0.5, 2.0
BOX = (0.1, 0.1, 0.05)
BOX_MASS = 2.0
MU = 0.5


def qaxis(axis, angle):
    a = np.asarray(axis, float)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * a / np.linalg.norm(a)])


def qrot(q, v):
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return R @ np.asarray(v, float)


def impedance(r):
    """solimp impedance at penetration r (default solimp)."""
    a = min(abs(r) / WIDTH, 1.0)
    y = a ** POWER / MID ** (POWER - 1) if a <= MID else 1 - (1 - a) ** POWER / (1 - MID) ** (POWER - 1)
    return D0 + y * (DMAX - D0)


def rest_penetration(per_contact_force, tran, cone, impratio, friction0=MU, condim=3):
    """Penetration r at which a resting contact carries per_contact_force (qacc = 0, v = 0), by fixed point.
    At rest aref = K imp r on every row that carries normal force; elliptic: the normal row's force is aref / R,
    R = (1 - imp) / imp * tran; pyramidal: 2 (condim - 1) edges of R = 2 mu^2 (1 - imp) / imp * tran (1 + f0^2),
    mu = f0 / sqrt(impratio)."""
    K = 1.0 / (DMAX * DMAX * TC * TC * DR * DR)
    if cone == "elliptic":
        per_r = lambda imp: K * imp * imp / ((1 - imp) * tran)
    else:
        mu = friction0 / np.sqrt(impratio)
        per_r = lambda imp: 2 * (condim - 1) * K * imp * imp / (2 * mu * mu * (1 - imp) * tran * (1 + friction0 ** 2))
    r = 1e-4
    for _ in range(500):
        r = per_contact_force / per_r(impedance(r))
    return r


# ---------------------------------------------------------------------------------------------- models
def _xml(name, cone, impratio, bodies, floor='<geom name="floor" type="plane" size="5 5 .1"/>', option="", flags=""):
    fl = f"<flag {flags}/>" if flags else ""
    return f"""
<mujoco model="{name}">
  <option timestep="{DT}" cone="{cone}" impratio="{impratio}"{option}>{fl}</option>
  <custom><numeric name="agent_planner" data="0"/><numeric name="agent_horizon" data="0.1"/></custom>
  <worldbody>
    {floor}
    {bodies}
  </worldbody>
  {{sensor}}
</mujoco>"""


def _box(name, pos, quat=(1, 0, 0, 0), mass=BOX_MASS, attrs=f'friction="{MU} 0.005 0.0001"'):
    p, q = " ".join(map(str, pos)), " ".join(map(str, quat))
    return (f'<body name="{name}" pos="{p}" quat="{q}"><freejoint/><geom type="box" size="{BOX[0]} {BOX[1]} {BOX[2]}" '
            f'mass="{mass}" {attrs}/></body>')


def _free(q, v=None, quat=(1, 0, 0, 0)):
    return np.concatenate([q, quat]), (np.zeros(6) if v is None else np.asarray(v, float))


class Scene:
    """name, xml(cone, impratio) -> text, states(m, cone, impratio) -> [(name, qpos, qvel)], path, cached."""

    def __init__(self, name, bodies, states, path, cached, floor=None, option="", cones=CONES):
        self.name, self.bodies, self._states, self.path, self.cached = name, bodies, states, path, cached
        self.floor, self.option, self.cones = floor, option, cones

    def xml(self, cone, impratio, option="", flags=""):
        kw = {} if self.floor is None else {"floor": self.floor}
        return _xml(self.name, cone, impratio, self.bodies, option=self.option + option, flags=flags, **kw)

    def states(self, m, cone, impratio):
        return self._states(m, cone, impratio)

    def is_cached(self, cone):
        return self.cached[cone] if isinstance(self.cached, dict) else self.cached


def compile_scene(text):
    import joint_scenes as JS
    return JS.compile_scene(text)


def _rest_z(m, cone, impratio, body=1, ncontact=4, friction0=MU, condim=3):
    tran = float(m.body_invweight0[body][0])
    return rest_penetration(BOX_MASS * G / ncontact, tran, cone, impratio, friction0, condim)


def _box_rest_states(m, cone, impratio):
    r = _rest_z(m, cone, impratio)
    z = BOX[2] - r
    out = []
    for name, vx in (("rest", 0.0), ("slide", 1.0), ("creep", 1e-4)):
        q, v = _free([0, 0, z], [vx, 0, 0, 0, 0, 0])
        out.append((name, q, v))
    return out


def _incline_scene(deg):
    th = np.radians(deg)
    quat = qaxis([0, 1, 0], -th)        # the plane's normal tilts towards +x: the box would slide down -x ... +x
    n = qrot(quat, [0, 0, 1])
    floor = f'<geom name="floor" type="plane" size="5 5 .1" quat="{" ".join(map(str, quat))}" friction="{MU} 0.005 0.0001"/>'

    def states(m, cone, impratio):
        pen = 2e-4
        c = n * (BOX[2] - pen)
        q, v = _free(c, quat=quat)
        return [("rest", q, v)]
    return Scene(f"incline{deg}", _box("box", [0, 0, 1]), states, "generic", True, floor=floor)


def _aniso_scene(condim):
    quat = qaxis([1, 0, 0], np.radians(20))   # normal (0, -0.34, 0.94): away from make_frame's |n_y| = 0.5 switch
    n = qrot(quat, [0, 0, 1])
    fr = 'friction="1.0 0.1 0.005"'
    floor = f'<geom name="floor" type="plane" size="5 5 .1" quat="{" ".join(map(str, quat))}" {fr} condim="{condim}"/>'

    def states(m, cone, impratio):
        c = n * (BOX[2] - 3e-4)
        t1, t2 = qrot(quat, [1, 0, 0]), qrot(quat, [0, 1, 0])
        out = []
        for name, vt, w in (("slide", 0.6 * t1 + 0.3 * t2, 2.0 * n), ("stick", 1e-4 * t1, 0.0 * n)):
            q, v = _free(c, np.concatenate([vt, w]), quat=quat)
            out.append((name, q, v))
        return out
    return Scene(f"aniso_condim{condim}", _box("box", [0, 0, 1], attrs=f'{fr} condim="{condim}"'), states, "generic",
                 True, floor=floor)


def _cylinder_states(m, cone, impratio):
    q, v = _free([0, 0, 0.12 - 3e-4], [0.2, 0, 0, 0, 0, 5.0])
    q2, v2 = _free([0, 0, 0.12 - 3e-4], [0, 0, 0, 0, 0, 0.05])
    return [("spin", q, v), ("slow_spin", q2, v2)]


def _sphere_states(m, cone, impratio):
    r = 0.1
    q, v = _free([0, 0, r - 4e-4], [1.0, 0, 0, 0, 1.0 / r * 0.8, 0.5])      # rolling and slipping, spinning
    q2, v2 = _free([0, 0, r - 4e-4], [0.3, 0, 0, 0, 0.3 / r, 0])             # pure rolling
    return [("roll_slip", q, v), ("roll", q2, v2)]


def _stack_bodies(n, masses):
    """A box on the floor, then n - 1 spheres stacked on it (sphere-box, sphere-sphere contacts)."""
    r = 0.06
    out = _box("b0", [0, 0, 1], mass=masses[0])
    for k in range(1, n):
        out += (f'<body name="s{k}" pos="0 0 {1 + k}"><freejoint/><geom type="sphere" size="{r}" mass="{masses[k]}" '
                f'friction="{MU} 0.005 0.0001"/></body>')
    return out


def _stack_states(n, masses):
    def states(m, cone, impratio):
        r = 0.06
        pen = 3e-4
        zb = BOX[2] - pen
        q = list(_free([0, 0, zb])[0])
        v = [0.0] * 6
        z = zb + BOX[2] + r - pen
        for k in range(1, n):
            q += [0.01 * k, -0.005 * k, z, 1, 0, 0, 0]
            v += [0.2 * (-1) ** k, 0.1, -0.05, 0.5, -0.3, 0.2 * k]
            z += 2 * r - 4 * pen
        q, v = np.array(q), np.array(v)
        v2 = v.copy(); v2[:6] = [0.5, -0.2, 0, 0, 0, 1.0]
        return [("rest", q, v), ("moving", q, v2)]
    return states


def _chain_bodies(n=18, r=0.04):
    """A chain of n hinges lying on the floor along x (axes alternating y / z), a sphere on every other link up to the
    16th (a floor contact on a deeper link would couple more than the device's 16 compact Jacobian columns); the
    spheres touch the floor only (contype 2)."""
    body = ""
    for k in range(n):
        ax = "0 1 0" if k % 2 == 0 else "0 0 1"
        geom = (f'<geom type="sphere" size="{r}" mass="0.1" friction="{MU} 0.005 0.0001" contype="2"/>'
                if k % 2 == 1 and k < 16 else
                f'<geom type="capsule" fromto="0 0 0 0.06 0 0" size="0.01" mass="0.05" contype="0" conaffinity="0"/>')
        body += f'<body name="c{k}" pos="0.1 0 0"><joint name="h{k}" type="hinge" axis="{ax}" damping="0.1"/>{geom}'
    return f'<body name="root" pos="0 0 {r - 4e-4}">{body}{"</body>" * n}</body>'


def _chain_states(m, cone, impratio):
    rng = np.random.default_rng(5)
    v = 0.3 * rng.standard_normal(m.nv)
    q0 = np.zeros(m.nq)
    q1 = 0.02 * np.where(np.arange(m.nq) % 2 == 1, 1.0, 0.0) * rng.uniform(-1, 1, m.nq)   # turns about z only
    return [("rest", q0, 0 * v), ("moving", q1, v)]


def _many_bodies(nbox, condim1_boxes=0, floss=False):
    out = ""
    for k in range(nbox):
        cd = 1 if k >= nbox - condim1_boxes else 3
        out += _box(f"b{k}", [0.4 * k, 0, 1], attrs=f'friction="{MU} 0.005 0.0001" condim="{cd}"')
    if floss:
        out += ('<body name="slider" pos="0 2 1"><joint name="sl" type="slide" axis="1 0 0" frictionloss="0.5"/>'
                '<geom type="sphere" size="0.05" mass="1" contype="0" conaffinity="0"/></body>')
    return out


def _many_states(nbox, floss):
    def states(m, cone, impratio):
        q, v = [], []
        for k in range(nbox):
            q += [0.4 * k, 0, BOX[2] - 2e-4 * (1 + 0.1 * k), 1, 0, 0, 0]
            v += [0.3 * np.cos(k), 0.3 * np.sin(k), -0.01, 0.1 * k, -0.2, 0.5]
        if floss:
            q += [0.0]; v += [0.01]
        return [("moving", np.array(q), np.array(v))]
    return states


def scenes():
    """name -> Scene.  cached: whether the line search has at most 32 work items (asserted by the tests)."""
    floor1 = '<geom name="floor" type="plane" size="5 5 .1" condim="1"/>'
    floor_mu = f'<geom name="floor" type="plane" size="5 5 .1" friction="{MU} 0.005 0.0001"/>'
    out = {
        "box": Scene("box", _box("box", [0, 0, 1]), _box_rest_states, "generic", True, floor=floor_mu),
        "incline15": _incline_scene(15), "incline26": _incline_scene(26), "incline40": _incline_scene(40),
        "aniso_condim3": _aniso_scene(3), "aniso_condim4": _aniso_scene(4),
        "cylinder": Scene("cylinder", '<body name="cyl" pos="0 0 1"><freejoint/><geom type="cylinder" size="0.08 0.12" '
                                      'mass="1.5" condim="4" friction="0.6 0.05 0.001"/></body>',
                          _cylinder_states, "generic", True),
        "sphere": Scene("sphere", '<body name="ball" pos="0 0 1"><freejoint/><geom type="sphere" size="0.1" mass="1" '
                                  'condim="6" friction="0.8 0.02 0.01"/></body>', _sphere_states, "generic", True),
        "stack2": Scene("stack2", _stack_bodies(2, (2.0, 1.0)), _stack_states(2, (2.0, 1.0)), "generic", True,
                        floor=floor_mu),
        "stack2_heavy_top": Scene("stack2_heavy_top", _stack_bodies(2, (1.0, 1e3)), _stack_states(2, (1.0, 1e3)),
                                  "generic", True, floor=floor_mu),
        "stack2_heavy_bottom": Scene("stack2_heavy_bottom", _stack_bodies(2, (1e3, 1.0)), _stack_states(2, (1e3, 1.0)),
                                     "generic", True, floor=floor_mu),
        "stack3": Scene("stack3", _stack_bodies(3, (2.0, 1.0, 0.5)), _stack_states(3, (2.0, 1.0, 0.5)), "nq4", True,
                        floor=floor_mu),
        "chain18": Scene("chain18", _chain_bodies(), _chain_states, "nq6", True, floor=floor_mu),
        # 8 one-sided contacts: pyramidal 32 rows = 32 items (cached); + a friction-loss row = 33 (uncached)
        "many2": Scene("many2", _many_bodies(2), _many_states(2, False), "generic", True, floor=floor1,
                       cones=("pyramidal",)),
        "many2_floss": Scene("many2_floss", _many_bodies(2, floss=True), _many_states(2, True), "generic", False,
                             floor=floor1, cones=("pyramidal",)),
        # 32 contacts: elliptic one item each (cached); + a friction-loss row = 33 items (uncached); 89 rows
        "many8": Scene("many8", _many_bodies(8, condim1_boxes=1), _many_states(8, False), "generic", True,
                       floor=floor1, cones=("elliptic",)),
        "many8_floss": Scene("many8_floss", _many_bodies(8, condim1_boxes=1, floss=True), _many_states(8, True),
                             "generic", False, floor=floor1, cones=("elliptic",)),
    }
    return out


def line_search_items(m, r):
    """Work items of the device line search for the oracle's constraint problem r (Oracle.efc_debug): one per
    friction-loss / limit / frictionless / pyramidal row, one per elliptic contact."""
    return int(sum(1 for i, t in enumerate(r["efc_type"]) if t != 3 or i == r["efc_address"][r["efc_id"][i]]))


def model_path(m):
    """The Hessian path the generic instance takes for model m."""
    import joint_scenes as JS
    if m.nv != 18:
        return "generic"
    return "nq4" if JS.nhpair(m) <= 128 else "nq6"


def variants():
    """[(scene key, cone, impratio)] over every scene."""
    return [(k, c, i) for k, s in scenes().items() for c in s.cones for i in IMPRATIOS]


# ---------------------------------------------------------------------------------------------- Quadruped states
def quadruped_states(m):
    """(name, qpos, qvel): four feet 2 mm into the floor, at rest and sliding; a self-contact state in the air."""
    home = np.asarray(m.key_qpos[0], float).copy()
    stand = home.copy(); stand[2] -= 0.012
    rng = np.random.default_rng(2)
    v = np.zeros(m.nv); v[6:] = 1e-3 * rng.standard_normal(m.nv - 6)
    slide = np.zeros(m.nv); slide[0], slide[1], slide[5] = 0.6, -0.2, 0.4; slide[6:] = 0.3 * rng.standard_normal(m.nv - 6)
    return [("stance", stand, v), ("stance_sliding", stand, slide)]


def self_contact_state(m, oracle):
    """The first state of a seeded sweep whose legs touch each other in the air (the dense-fallback path)."""
    from test_gpu_tree_factor import _self_contact_states
    rng = np.random.default_rng(3)
    qs, vs = _self_contact_states(m, rng, 256)
    mc = np.concatenate([np.concatenate([m.mocap_pos0[i], m.mocap_quat0[i]]) for i in range(m.nmocap)]) \
        if m.nmocap else np.zeros(0)
    ref = oracle.step_batch(qs, vs, np.zeros((len(qs), m.nu)), mc, np.zeros(len(qs)), nthreads=4)
    k = int(np.flatnonzero((ref["ncon"] >= 2) & (ref["warning"] == 0))[0])
    return ("self_contact", qs[k], vs[k])


# ---------------------------------------------------------------------------------------------- fp64 restatement
KMINMU, KMINIMP, KMAXIMP = 1e-5, 0.0001, 0.9999


def _imp(solimp, pos, margin):
    dmin, dmax = (min(KMAXIMP, max(KMINIMP, x)) for x in solimp[:2])
    width, mid, power = max(0.0, solimp[2]), min(KMAXIMP, max(KMINIMP, solimp[3])), max(1.0, solimp[4])
    if dmin == dmax or width <= 1e-15:
        return 0.5 * (dmin + dmax)
    x = abs((pos - margin) / width)
    if x >= 1:
        return dmax
    if x == 0:
        return dmin
    y = x if power == 1 else (x ** power / mid ** (power - 1) if x <= mid else
                              1 - (1 - x) ** power / (1 - mid) ** (power - 1))
    return dmin + y * (dmax - dmin)


def _KB(m, solref, solimp):
    dmax = min(KMAXIMP, max(KMINIMP, solimp[1]))
    if solref[0] > 0:
        tc = solref[0] if m.opt_disable_refsafe else max(solref[0], 2 * m.opt_timestep)
        return 1 / max(1e-15, dmax * dmax * tc * tc * solref[1] ** 2), 2 / max(1e-15, dmax * tc)
    return -solref[0] / max(1e-15, dmax * dmax), -solref[1] / max(1e-15, dmax)


class Problem:
    """The constraint problem of one state, restated in fp64 from the model, the kinematics of refmath and the oracle's
    contact geometry (dist, pos, frame, geom pair, dim): rows, their weights, aref, and the convex cost

        f(a) = 1/2 (a - a_smooth)' M (a - a_smooth) + s(J a - aref),

    s from MuJoCo's published convex formulation: 1/2 D x^2 for an active one-sided row (x < 0: frictionless contacts,
    pyramidal edges) and a quadratic friction-loss row (Huber beyond R f); per elliptic contact, in the scaled
    coordinates N = mu x_0, T = |(f_j x_j)_j|, zero above the cone (N >= mu T), 1/2 sum_j D_j x_j^2 below the dual cone
    (mu N + T <= 0) and 1/2 Dm (N - mu T)^2 between, Dm = D_0 / (mu^2 (1 + mu^2)).

    Weights.  imp from solimp at pos - margin; R = max(1e-15, (1 - imp) / imp * diagApprox), diagApprox from
    body_invweight0 (translation for rows 0-2, rotation for 3-5; dof_invweight0 for a friction-loss row).  Elliptic:
    R_1 = R_0 / impratio, R_j f_j^2 = R_1 f_0^2 (j >= 1), mu = f_0 sqrt(R_1 / R_0).  Pyramidal: the 2 (condim - 1)
    edges J_n +- f_k J_t,k share R = 2 mu^2 R_0 with mu = f_0 / sqrt(impratio), where R_0 is the first edge's own
    (1 - imp) / imp (tran + f_0^2 tran).  That last rule is transcribed from the implementation, not derived: MuJoCo
    is not vendored, so it is not checked against its source.  aref = -B J v - K imp (pos - margin), K = 0 on elliptic friction rows."""

    def __init__(self, m, qpos, qvel, r, qacc_smooth=None, mocap=None):
        from mujoco_mpc_b200 import refmath
        from mujoco_mpc_b200.mjcf import JNT_HINGE, JNT_SLIDE
        nv = m.nv
        mp, mq = (None, None) if mocap is None or m.nmocap == 0 else (
            np.asarray(mocap, float).reshape(-1, 7)[:, :3], np.asarray(mocap, float).reshape(-1, 7)[:, 3:])
        q = np.array(qpos, float)
        M, _ = refmath.mass_matrix_and_jacobians(m, q, mp, mq)
        kin = refmath.kinematics(m, q, mp, mq)
        self.M = M
        self.a_smooth = np.asarray(r["qacc_smooth"] if qacc_smooth is None else qacc_smooth, float)
        rows = []   # (J, pos, margin, diag, kind, contact, solref, solimp, frictionloss, friction_row)
        if not m.opt_disable_frictionloss:
            for i in range(nv):
                if m.dof_frictionloss[i] > 0:
                    e = np.zeros(nv); e[i] = 1
                    rows.append(dict(J=e, pos=0.0, margin=0.0, diag=float(m.dof_invweight0[i]), kind="floss", id=i,
                                     solref=m.dof_solref[i], solimp=m.dof_solimp[i], floss=float(m.dof_frictionloss[i])))
        # slide / hinge limits: one row per violated side, dist = side (range - q), J = -side on the joint's dof
        assert m.ntendon == 0 or not np.any(m.tendon_limited), "tendon limits are not restated"
        if not m.opt_disable_limit:
            for j in range(m.njnt):
                if not m.jnt_limited[j] or m.jnt_type[j] not in (JNT_SLIDE, JNT_HINGE):
                    continue
                da, qv = int(m.jnt_dofadr[j]), float(q[m.jnt_qposadr[j]])
                for side in (-1, 1):
                    dist = side * (m.jnt_range[j][(side + 1) // 2] - qv)
                    if dist < m.jnt_margin[j]:
                        e = np.zeros(nv); e[da] = -side
                        rows.append(dict(J=e, pos=dist, margin=float(m.jnt_margin[j]), diag=float(m.dof_invweight0[da]),
                                         kind="limit", id=j, solref=m.jnt_solref[j], solimp=m.jnt_solimp[j]))
        self.contacts = []
        pyramidal = m.opt_cone == 0
        for c in range(r["ncon"]):
            g1, g2 = int(r["geom1"][c]), int(r["geom2"][c])
            b1, b2 = int(m.geom_bodyid[g1]), int(m.geom_bodyid[g2])
            pos = r["pos"][c]
            Jp = refmath.body_jacobian(m, kin, b2, pos) - refmath.body_jacobian(m, kin, b1, pos)
            frame = r["frame"][c]
            dim = int(r["dim"][c])
            # parameter mixing (MuJoCo's published rule): the higher-priority geom's parameters; at equal priority the
            # larger condim and friction, and solref / solimp mixed by solmix (the smaller of two direct solrefs)
            if m.geom_priority[g1] != m.geom_priority[g2]:
                gp = g1 if m.geom_priority[g1] > m.geom_priority[g2] else g2
                cdim, solref, solimp, fr3 = m.geom_condim[gp], m.geom_solref[gp], m.geom_solimp[gp], m.geom_friction[gp]
            else:
                cdim = max(m.geom_condim[g1], m.geom_condim[g2])
                w1, w2 = m.geom_solmix[g1], m.geom_solmix[g2]
                mix = (w1 / (w1 + w2) if w1 >= 1e-15 and w2 >= 1e-15 else
                       0.5 if w1 < 1e-15 and w2 < 1e-15 else (0.0 if w1 < 1e-15 else 1.0))
                r1, r2 = np.asarray(m.geom_solref[g1], float), np.asarray(m.geom_solref[g2], float)
                solref = mix * r1 + (1 - mix) * r2 if r1[0] > 0 and r2[0] > 0 else np.minimum(r1, r2)
                solimp = mix * np.asarray(m.geom_solimp[g1], float) + (1 - mix) * np.asarray(m.geom_solimp[g2], float)
                fr3 = np.maximum(m.geom_friction[g1], m.geom_friction[g2])
            assert dim == cdim
            fr3 = np.maximum(fr3, KMINMU)
            fr = np.array([fr3[0], fr3[0], fr3[1], fr3[2], fr3[2]])
            tran = m.body_invweight0[b1][0] + m.body_invweight0[b2][0]
            rot = m.body_invweight0[b1][1] + m.body_invweight0[b2][1]
            Jrow = lambda k: frame[k % 3] @ (Jp[0:3] if k < 3 else Jp[3:6])
            margin = max(m.geom_margin[g1], m.geom_margin[g2]) - max(m.geom_gap[g1], m.geom_gap[g2])
            first = len(rows)
            if pyramidal and dim > 1:
                for k in range(1, dim):
                    for sgn in (1, -1):
                        rows.append(dict(J=Jrow(0) + sgn * fr[k - 1] * Jrow(k), pos=r["dist"][c], margin=margin,
                                         diag=tran + fr[k - 1] ** 2 * (tran if k < 3 else rot), kind="edge",
                                         id=c, solref=solref, solimp=solimp))
            else:
                for k in range(dim):
                    rows.append(dict(J=Jrow(k), pos=r["dist"][c] if k == 0 else 0.0, margin=margin,
                                     diag=rot if k >= 3 else tran, kind="one" if dim == 1 else "cone",
                                     id=c, solref=solref, solimp=solimp, friction_row=k > 0))
            self.contacts.append(dict(adr=first, dim=dim, friction=fr, nrow=len(rows) - first))
        ne = len(rows)
        self.J = np.array([x["J"] for x in rows]).reshape(ne, nv)
        tcode = dict(floss=0, limit=1, one=2, cone=3, edge=5)     # oracle/physics.h CNSTR_*
        self.type = np.array([tcode[x["kind"]] for x in rows], int)
        self.id = np.array([x["id"] for x in rows], int)
        self.kind = [x["kind"] for x in rows]
        self.pos = np.array([x["pos"] for x in rows]); self.margin = np.array([x["margin"] for x in rows])
        self.diag = np.array([x["diag"] for x in rows])
        self.floss = np.array([x.get("floss", 0.0) for x in rows])
        self.imp = np.array([_imp(x["solimp"], x["pos"], x["margin"]) for x in rows])
        KB = np.array([_KB(m, x["solref"], x["solimp"]) for x in rows]).reshape(ne, 2)
        K = np.where([x.get("friction_row", False) or x["kind"] == "floss" for x in rows], 0.0, KB[:, 0])
        self.R = np.maximum(1e-15, (1 - self.imp) / self.imp * self.diag)
        for c in self.contacts:
            a, dim, f = c["adr"], c["dim"], c["friction"]
            if dim == 1:
                c["mu"] = 0.0
                continue
            if pyramidal:
                c["mu"] = f[0] * np.sqrt(1 / max(1e-15, m.opt_impratio))
                self.R[a:a + c["nrow"]] = 2 * c["mu"] ** 2 * self.R[a]
            else:
                self.R[a + 1] = self.R[a] / max(1e-15, m.opt_impratio)
                c["mu"] = f[0] * np.sqrt(self.R[a + 1] / self.R[a])
                for j in range(1, dim - 1):
                    self.R[a + j + 1] = self.R[a + 1] * f[0] ** 2 / f[j] ** 2
        self.D = 1 / self.R
        self.vel = self.J @ np.asarray(qvel, float)
        self.aref = -KB[:, 1] * self.vel - K * self.imp * (self.pos - self.margin)
        self.ne, self.nv = ne, nv

    # per-row cost, force (= -ds/dx) and generalised Hessian of s at x = J a - aref
    def constraint(self, x):
        cost, force, H, zone = 0.0, np.zeros(self.ne), np.zeros((self.ne, self.ne)), [None] * self.ne
        cone_rows = set()
        for c in self.contacts:
            if self.kind[c["adr"]] == "cone":
                a, dim, mu, f = c["adr"], c["dim"], c["mu"], c["friction"]
                cone_rows.update(range(a, a + dim))
                S = np.concatenate([[mu], f[:dim - 1]])
                u = S * x[a:a + dim]
                N, T = u[0], np.linalg.norm(u[1:])
                if N >= mu * T:
                    z = "top"
                elif mu * N + T <= 0:
                    z = "bottom"
                    D = self.D[a:a + dim]
                    cost += 0.5 * np.sum(D * x[a:a + dim] ** 2)
                    force[a:a + dim] = -D * x[a:a + dim]
                    H[a:a + dim, a:a + dim] = np.diag(D)
                else:
                    z = "cone"
                    Dm = self.D[a] / (mu * mu * (1 + mu * mu))
                    NmT = N - mu * T
                    cost += 0.5 * Dm * NmT ** 2
                    g = np.concatenate([[1.0], -mu * u[1:] / T])            # d(N - mu T)/du
                    force[a:a + dim] = -Dm * NmT * g * S
                    Hu = np.outer(g, g)
                    Hu[1:, 1:] -= NmT * mu * (np.eye(dim - 1) / T - np.outer(u[1:], u[1:]) / T ** 3)
                    H[a:a + dim, a:a + dim] = Dm * (S[:, None] * Hu * S[None, :])
                for i in range(a, a + dim):
                    zone[i] = z
        for i in range(self.ne):
            if i in cone_rows:
                continue
            D = self.D[i]
            if self.kind[i] == "floss":
                rf = self.R[i] * self.floss[i]
                if x[i] <= -rf:
                    cost += self.floss[i] * (-0.5 * rf - x[i]); force[i] = self.floss[i]; zone[i] = "linear"
                elif x[i] >= rf:
                    cost += self.floss[i] * (-0.5 * rf + x[i]); force[i] = -self.floss[i]; zone[i] = "linear"
                else:
                    cost += 0.5 * D * x[i] ** 2; force[i] = -D * x[i]; H[i, i] = D; zone[i] = "quadratic"
            elif x[i] < 0:
                cost += 0.5 * D * x[i] ** 2; force[i] = -D * x[i]; H[i, i] = D; zone[i] = "quadratic"
            else:
                zone[i] = "satisfied"
        return cost, force, H, zone

    def cost(self, a):
        d = a - self.a_smooth
        return 0.5 * d @ self.M @ d + self.constraint(self.J @ a - self.aref)[0]

    def grad(self, a):
        return self.M @ (a - self.a_smooth) - self.J.T @ self.constraint(self.J @ a - self.aref)[1]

    def hess(self, a):
        return self.M + self.J.T @ self.constraint(self.J @ a - self.aref)[2] @ self.J

    def force(self, a):
        return self.constraint(self.J @ a - self.aref)[1]

    def zones(self, a):
        return self.constraint(self.J @ a - self.aref)[3]

    def grad_scale(self, a):
        """Magnitude of the terms the gradient is a difference of: |M (a - a_smooth)| + |J' f|."""
        return np.abs(self.M @ (a - self.a_smooth)) + np.abs(self.J.T @ self.force(a))

    def minimise(self, a0=None):
        """An independent minimiser: scipy's trust-region Newton on the restated cost, gradient and Hessian."""
        from scipy.optimize import minimize
        a = self.a_smooth if a0 is None else a0
        for _ in range(3):   # restarted: a stop on an unresolvable cost decrease resets the trust radius
            a = minimize(self.cost, a, jac=self.grad, hess=self.hess, method="trust-exact",
                         options=dict(gtol=1e-13, maxiter=500)).x
        return a


def optimum_starts(p, a_opt, seed):
    """Warm starts around the fp64 optimum a_opt that cost less than a_smooth: perturbations along random directions
    scaled to |a_opt - a_smooth|, at several sizes."""
    rng = np.random.default_rng(seed)
    span = np.linalg.norm(a_opt - p.a_smooth) + 1e-3
    out = []
    c_s = p.cost(p.a_smooth)
    for s in (0.02, 0.1, 0.3, 0.6):
        for _ in range(3):
            d = rng.standard_normal(p.nv)
            a = a_opt + s * span * d / np.linalg.norm(d)
            if p.cost(a) < c_s:
                out.append(a)
                break
    return out
