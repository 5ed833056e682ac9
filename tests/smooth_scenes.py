"""Purpose-built scenes for the smooth dynamics: everything k_forward does before the constraints (k_kinematics,
k_com_pos, k_crb, k_com_vel, the RNE bias of k_smooth_forces) and the position update of k_euler (quat_integrate);
on the oracle side kinematics, com_pos, crb, com_vel, rne and euler of oracle/physics.h.

No scene has a contact (the bodies carry an <inertial> and no geom, and there is no floor),
a spring, damping, friction loss, a limit or an actuator, so that qacc = M^-1 (-qfrc_bias) and the Euler step is the
plain v' = v + h qacc, q' = q (+) h v'.  Each scene lists its cases (name, qpos, qvel, mocap or None for the model's
mocap poses); the comment on each says what it exercises.

Shared by tests/test_smooth_dynamics_cpu.py (an fp64 restatement, pinned to closed forms, against the fp64 oracle) and
tests/test_gpu_smooth_dynamics.py (the device against the fp64 oracle).
"""
import numpy as np

DT = 0.01
QROT = np.array([0.8, 0.2, -0.4, 0.4]) / np.linalg.norm([0.8, 0.2, -0.4, 0.4])
Q2 = np.array([0.3, -0.7, 0.5, 0.4]) / np.linalg.norm([0.3, -0.7, 0.5, 0.4])
# three distinct principal moments and non-zero products: the compiler's body_iquat is far from the identity
TOP_FULLINERTIA = np.array([0.3, 0.2, 0.1, 0.02, -0.01, 0.015])
TOP_INERTIAL = '<inertial mass="2" pos="0.05 -0.03 0.02" fullinertia="0.3 0.2 0.1 0.02 -0.01 0.015"/>'


def principal_axes(full):
    """Columns: the principal axes of a fullinertia (Ixx Iyy Izz Ixy Ixz Iyz) in the body frame."""
    f = full
    I = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
    return np.linalg.eigh(I)[1]


def scene_xml(name, bodies, option=""):
    return f"""
<mujoco model="{name}">
  <compiler angle="radian"/>
  <option timestep="{DT}"{option}/>
  <custom><numeric name="agent_planner" data="0"/><numeric name="agent_horizon" data="0.1"/></custom>
  <worldbody>{bodies}</worldbody>
  {{sensor}}
</mujoco>"""


class Scene:
    """A model (its <worldbody> content) and its cases: (name, qpos, qvel, mocap or None)."""

    def __init__(self, name, bodies, cases, option=""):
        self.name, self.bodies, self.option = name, bodies, option
        self.cases = [(c[0], np.asarray(c[1], float), np.asarray(c[2], float), None if c[3] is None
                       else np.asarray(c[3], float)) for c in cases]

    def text(self):
        return scene_xml(self.name, self.bodies, self.option)

    def compile(self):
        import joint_scenes as JS
        return JS.compile_scene(self.text())


def _rng_cases(prefix, n, nq_parts, nv, seed, vscale=1.0):
    """n random states: nq_parts is a list of 'hinge' / 'slide' / 'ball' / 'free' in joint order."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        q = []
        for p in nq_parts:
            if p in ("hinge", "slide"):
                q.append([rng.uniform(-1.5, 1.5)])
            elif p == "ball":
                u = rng.standard_normal(4); q.append(u / np.linalg.norm(u))
            else:
                u = rng.standard_normal(4)
                q.append(np.concatenate([rng.uniform(-1, 1, 3) + [0, 0, 2], u / np.linalg.norm(u)]))
        out.append((f"{prefix}{i}", np.concatenate(q), vscale * rng.standard_normal(nv), None))
    return out


# ---------------------------------------------------------------------------------------------- free rigid body
def free_top():
    """One free body with anisotropic inertia in a rotated inertial frame (iquat != identity) and ipos != 0."""
    V = principal_axes(TOP_FULLINERTIA)
    lin = np.array([0.3, -0.2, 0.1])
    gen = np.array([3.0, -2.0, 4.0]) / np.linalg.norm([3.0, -2.0, 4.0])
    q = np.concatenate([[0.1, -0.2, 1.0], QROT])
    cases = [(f"spin_principal_{k}", q, np.concatenate([lin, 5.0 * V[:, k]]), None) for k in range(3)]
    cases += [("spin_generic", q, np.concatenate([lin, [3.0, -2.0, 4.0]]), None),
              ("at_rest", q, np.zeros(6), None)]
    # h |omega| of 0.5, 2 and 3.1 rad per step (3.1: a rotation of almost pi in one step)
    cases += [(f"fast_{s}", q, np.concatenate([lin, s / DT * gen]), None) for s in (0.5, 2.0, 3.1)]
    return Scene("free_top", f'<body name="top" pos="0 0 1"><freejoint/>{TOP_INERTIAL}</body>', cases)


# ---------------------------------------------------------------------------------------------- ball pendulum
BALL_PENDULUM = (
    '<body name="bob" pos="0 0 2"><joint name="ball" type="ball" pos="0.03 -0.02 0.15" armature="0.01"/>'
    '<inertial mass="1.5" pos="0.02 0.01 -0.1" fullinertia="0.04 0.03 0.02 0.005 -0.003 0.002"/>'
    '<body name="bob_child" pos="0.05 0 -0.3" quat="0.9 0.1 0.3 -0.2">'
    '<joint name="bob_hinge" type="hinge" axis="0.3 1 0.2" pos="0 0 0.05"/>'
    '<inertial mass="0.7" pos="0.01 0.02 -0.12" diaginertia="0.01 0.008 0.004" quat="0.7 0.5 -0.3 0.4"/>'
    '</body></body>')


def ball_pendulum():
    """A ball joint with a pos offset on a body with anisotropic inertia, a hinge child on a tilted axis below it."""
    cases = [("tilted_at_rest", np.concatenate([QROT, [0.4]]), np.zeros(4), None),
             ("swinging", np.concatenate([Q2, [-0.8]]), [1.5, -2.0, 0.7, 3.0], None),
             ("fast_spin", np.concatenate([QROT, [2.5]]), [40.0, -25.0, 60.0, -30.0], None)]
    return Scene("ball_pendulum", BALL_PENDULUM, cases)


# ---------------------------------------------------------------------------------------------- multi-joint bodies
MULTI_JOINT = (
    '<body name="sled" pos="0.5 0 1.5">'
    '<joint name="sl" type="slide" axis="1 2 0.5"/>'
    '<joint name="h1" type="hinge" axis="0 3 1" pos="0.1 0 0"/>'
    '<joint name="h2" type="hinge" axis="2 -1 1" pos="0 -0.05 0.1" armature="0.02"/>'
    '<inertial mass="1.2" pos="0.03 0.04 -0.05" fullinertia="0.05 0.04 0.03 0.004 0.002 -0.003"/>'
    '<body name="hb" pos="0.2 0.1 -0.2">'
    '<joint name="h3" type="hinge" axis="1 1 0" pos="0 0 0.05"/>'
    '<joint name="bb" type="ball" pos="0.02 0 0"/>'
    '<inertial mass="0.8" pos="0.05 0 -0.1" fullinertia="0.02 0.015 0.01 0.001 -0.002 0.0015"/>'
    '</body></body>')


def multi_joint():
    """One body with slide + hinge + hinge on tilted, non-unit XML axes (with pos offsets); below it one body with
    hinge + ball."""
    cases = [("pose_a", np.concatenate([[0.2, 0.5, -0.7, 0.3], QROT]), [0.4, -1.0, 2.0, 1.5, -0.5, 0.8, 1.2], None),
             ("pose_b", np.concatenate([[-0.3, -2.0, 1.1, -1.4], Q2]), [-1.0, 3.0, -2.5, 4.0, 2.0, -3.0, 1.0], None),
             ("at_rest", np.concatenate([[0.0, 0.3, 0.2, 0.1], QROT]), np.zeros(7), None)]
    return Scene("multi_joint", MULTI_JOINT, cases)


# ---------------------------------------------------------------------------------------------- joint ref
REF_BODIES = (
    '<body name="rh" pos="0 0 1.5"><joint name="rh" type="hinge" axis="1 0.5 0" ref="0.7" pos="0 0 0.05"/>'
    '<inertial mass="1" pos="0 0.2 -0.05" diaginertia="0.02 0.01 0.015" quat="0.9 0.3 0 0.2"/>'
    '<body name="rs" pos="0 0.3 0"><joint name="rs" type="slide" axis="0 1 1" ref="-0.3"/>'
    '<inertial mass="0.5" pos="0.05 0 0" diaginertia="0.004 0.003 0.002"/>'
    '<body name="rh2" pos="0 0.1 0"><joint name="rh2" type="hinge" axis="0 0 1" ref="-1.2"/>'
    '<inertial mass="0.4" pos="0.1 0 0" diaginertia="0.003 0.002 0.002"/>'
    '</body></body></body>')


def joint_ref():
    """Hinge and slide ref != 0 (qpos0 != 0), hinge angles of +-pi and of many turns."""
    v = [2.0, -0.5, 3.0]
    cases = [("at_ref", [0.7, -0.3, -1.2], v, None),
             ("plus_pi", [np.pi, 0.1, -np.pi], v, None),
             ("minus_pi", [-np.pi, 0.4, np.pi], v, None),
             ("forty_rad", [40.3, 0.2, -40.3], v, None),        # about 6.4 turns from ref
             ("forty_rad_fast", [40.3, 0.2, 40.3], [30.0, 2.0, -25.0], None)]
    return Scene("joint_ref", REF_BODIES, cases)


# ---------------------------------------------------------------------------------------------- odd bodies
ODD_CHAIN = (
    '<body name="base" mocap="true" pos="0 0 2.5">'
    '<body name="hung" pos="0 0 -0.1"><joint name="oh1" type="hinge" axis="1 0 0" pos="0 0 0.05"/>'
    '<inertial mass="0.6" pos="0 0.02 -0.1" diaginertia="0.006 0.005 0.002"/>'
    '<body name="welded" pos="0 0.1 -0.2" quat="0.9 0.2 -0.3 0.1">'                     # welded, with mass
    '<inertial mass="0.5" pos="0.03 0 -0.05" fullinertia="0.004 0.003 0.002 0.0005 0 -0.0004"/>'
    '<body name="massless" pos="0.05 0 -0.1" quat="0.8 0 0.6 0">'                      # welded and massless
    '<body name="tip" pos="0 0 -0.1"><joint name="oh2" type="hinge" axis="0 1 0.3"/>'
    '<inertial mass="0.3" pos="0.05 0 -0.05" diaginertia="0.002 0.002 0.001"/>'
    '<body name="ghost" pos="0 0 -0.1"/>'                                               # massless leaf
    '</body></body></body></body></body>')


def odd_chain():
    """A welded body with mass in mid-chain, a massless welded body in mid-chain, a massless leaf (the
    subtreemass < kMinVal branch of k_com_pos), all hanging by hinges from a mocap body."""
    moved = np.concatenate([[0.3, -0.2, 2.2], QROT])
    cases = [("mocap_home", [0.3, -0.6], [1.0, -2.0], None),
             ("mocap_moved", [0.3, -0.6], [1.0, -2.0], moved),
             ("mocap_moved_fast", [-1.2, 2.0], [15.0, -20.0], moved)]
    return Scene("odd_chain", ODD_CHAIN, cases)


# ---------------------------------------------------------------------------------------------- several trees
def forest():
    """Several trees in one model: the free top, the ball pendulum and the multi-joint bodies side by side."""
    bodies = f'<body name="top" pos="0 0 1"><freejoint/>{TOP_INERTIAL}</body>' + BALL_PENDULUM + MULTI_JOINT
    parts = ["free", "ball", "hinge", "slide", "hinge", "hinge", "hinge", "ball"]
    return Scene("forest", bodies, _rng_cases("random_", 3, parts, 6 + 4 + 7, seed=3, vscale=2.0))


# ---------------------------------------------------------------------------------------------- wide level
NWIDE = 42


def wide():
    """A free root with NWIDE hinge children: NWIDE > 32 bodies on one tree level (the second 32-lane chunk of
    k_kinematics, k_com_vel and the RNE), and nv = 6 + NWIDE = 48 in one tree (33 <= nv <= 64)."""
    kids = ""
    for k in range(NWIDE):
        a = 2 * np.pi * k / NWIDE
        c, s = np.cos(a), np.sin(a)
        kids += (f'<body name="w{k}" pos="{0.3 * c:.5f} {0.3 * s:.5f} 0">'
                 f'<joint name="wj{k}" type="hinge" axis="{-s:.5f} {c:.5f} {0.2 * (k % 3 - 1)}" pos="0.01 0 0"/>'
                 f'<inertial mass="{0.05 + 0.01 * (k % 5)}" pos="{0.08 * c:.5f} {0.08 * s:.5f} -0.04" '
                 f'diaginertia="0.0004 0.0003 0.0002"/></body>')
    bodies = f'<body name="hub" pos="0 0 2"><freejoint/>{TOP_INERTIAL}{kids}</body>'
    rng = np.random.default_rng(5)
    q = np.concatenate([[0.1, 0.2, 2.0], QROT, rng.uniform(-1.5, 1.5, NWIDE)])
    v = np.concatenate([[0.2, -0.1, 0.3], [4.0, -3.0, 6.0], 2.0 * rng.standard_normal(NWIDE)])
    return Scene("wide", bodies, [("random", q, v, None), ("at_rest", q, np.zeros(6 + NWIDE), None),
                                  ("fast_hub", q, np.concatenate([v[:3], [40.0, -60.0, 80.0], v[6:]]), None)])


# ---------------------------------------------------------------------------------------------- quaternion edges
QUAT_EDGES = (
    f'<body name="top" pos="0 0 1"><freejoint/>{TOP_INERTIAL}</body>' + BALL_PENDULUM +
    '<body name="handle" mocap="true" pos="1 0 2" quat="1 0 0 0">'
    '<body name="dangle" pos="0 0 -0.1"><joint name="dh" type="hinge" axis="0 1 0"/>'
    '<inertial mass="0.4" pos="0.05 0 -0.1" diaginertia="0.003 0.002 0.001"/></body></body>')


def quat_edges():
    """Non-unit, negative-w and all-zero quaternions in qpos (free body and ball joint) and a non-unit mocap
    quaternion.  MuJoCo normalises a quaternion before it uses it, and the all-zero one to the identity, in the
    kinematics and in the position update alike."""
    lin, w_free, w_ball = [0.3, -0.2, 0.1], [3.0, -2.0, 4.0], [1.5, -2.0, 0.7]
    v = np.concatenate([lin, w_free, w_ball, [1.0], [0.5]])
    v0 = np.concatenate([lin, [0, 0, 0], [0, 0, 0], [1.0], [0.5]])
    mocap = lambda quat: np.concatenate([[1.0, 0.2, 2.1], quat])

    def q(free, ball):
        return np.concatenate([[0.1, -0.2, 1.0], free, ball, [0.4], [0.3]])
    cases = [("non_unit", q(3.7 * QROT, 0.2 * Q2), v, mocap(2.5 * QROT)),
             ("negative_w", q(-QROT, -Q2), v, mocap(-QROT)),
             ("all_zero", q(np.zeros(4), np.zeros(4)), v, None),
             ("all_zero_at_rest", q(np.zeros(4), np.zeros(4)), v0, None),
             # zero angular velocity: the position update still returns the normalised quaternion
             ("non_unit_no_spin", q(3.7 * QROT, 0.2 * Q2), v0, mocap(0.5 * QROT))]
    return Scene("quat_edges", QUAT_EDGES, cases)


# ---------------------------------------------------------------------------------------------- far from the origin
FAR = (f'<body name="top" pos="0 0 1"><freejoint/>{TOP_INERTIAL}'
       '<body name="arm" pos="0.1 0 -0.1"><joint name="fh" type="hinge" axis="0.2 1 0.1" pos="0 0 0.05"/>'
       '<inertial mass="0.5" pos="0.05 0.02 -0.1" diaginertia="0.004 0.003 0.002"/></body></body>')
FAR_X = (1e2, 1e3)


def far():
    """A free body (with a hinged child) at x = 1e2 and 1e3 m, each with its twin translated to the origin: the
    dynamics do not depend on where the body is."""
    v = [0.3, -0.2, 0.1, 3.0, -2.0, 4.0, 2.5]
    base = np.concatenate([[0.1, -0.2, 1.0], QROT, [0.6]])
    cases = [("origin", base, v, None)]
    for x in FAR_X:
        q = base.copy(); q[0] += x
        cases.append((f"x{x:.0e}".replace("+0", ""), q, v, None))
    return Scene("far", FAR, cases)


def far_twin(name):
    """The translation of case `name` of the far scene (0 for the origin twin)."""
    return 0.0 if name == "origin" else float(name[1:])


# ---------------------------------------------------------------------------------------------- closed forms
SLIDE_AXIS = np.array([1.0, -2.0, 3.0]) / np.linalg.norm([1.0, -2.0, 3.0])


def slide_gravity():
    """One body on a tilted slide: qacc = g . axis."""
    body = ('<body name="s" pos="0 0 1" quat="0.9 0.1 0.2 0.3"><joint type="slide" axis="1 -2 3"/>'
            '<inertial mass="0.7" pos="0.1 0.05 0" diaginertia="0.01 0.02 0.03"/></body>')
    return Scene("slide_gravity", body, [("rest", [0.2], [0.0], None), ("moving", [-0.5], [3.0], None)])


PEND = dict(m=0.9, d=0.25, Ixx=0.012, arm=0.03, ref=0.4)


def hinge_pendulum():
    """A hinge about x with its centre of mass at y = d (ref != 0, armature): qacc = -m g d cos(q - ref) /
    (Ixx + m d^2 + armature), whatever the velocity."""
    p = PEND
    body = (f'<body name="p" pos="0 0 1"><joint type="hinge" axis="1 0 0" ref="{p["ref"]}" armature="{p["arm"]}"/>'
            f'<inertial mass="{p["m"]}" pos="0 {p["d"]} 0" diaginertia="{p["Ixx"]} 0.02 0.02"/></body>')
    return Scene("hinge_pendulum", body, [("rest", [1.0], [0.0], None), ("moving", [-2.0], [5.0], None),
                                          ("horizontal", [p["ref"]], [0.0], None)])


DP = dict(m1=1.3, m2=0.8, l1=0.5, c1=0.3, c2=0.2, I1=0.02, I2=0.01)


def double_pendulum():
    """The planar double pendulum without gravity: two hinges about y, link 1 of length l1 with its centre of mass
    at c1, link 2 with its centre of mass at c2, moments I1, I2 about y at the centres of mass."""
    p = DP
    body = (f'<body name="l1" pos="0 0 2"><joint name="t1" type="hinge" axis="0 1 0"/>'
            f'<inertial mass="{p["m1"]}" pos="0 0 {-p["c1"]}" diaginertia="0.03 {p["I1"]} 0.01"/>'
            f'<body name="l2" pos="0 0 {-p["l1"]}"><joint name="t2" type="hinge" axis="0 1 0"/>'
            f'<inertial mass="{p["m2"]}" pos="0 0 {-p["c2"]}" diaginertia="0.02 {p["I2"]} 0.005"/></body></body>')
    cases = [("pose_a", [0.3, 0.9], [1.5, -2.0], None), ("pose_b", [-1.1, 2.5], [-3.0, 4.0], None),
             ("straight", [0.7, 0.0], [2.0, 1.0], None)]
    return Scene("double_pendulum", body, cases, option=' gravity="0 0 0"')


# ---------------------------------------------------------------------------------------------- task models
def extreme_states(m):
    """Airborne extreme states of a model with a free root: (name, qpos, qvel)."""
    rng = np.random.default_rng(17)
    home = m.key_qpos[0].copy()
    home[2] += 2.0                                         # well above the floor: no contact
    nj = m.nv - 6
    out = []
    v = np.zeros(m.nv); v[3:6] = [25.0, -40.0, 30.0]       # fast trunk spin
    out.append(("trunk_spin", home, v))
    v = np.zeros(m.nv); v[:6] = [1.0, -0.5, 0.3, 2.0, -1.0, 1.5]; v[6:] = 20.0 * rng.uniform(-1, 1, nj)
    out.append(("joint_velocities", home, v))
    q = home.copy(); q[3:7] = 2.3 * QROT                # non-unit base quaternion
    out.append(("non_unit_base", q, 0.5 * rng.standard_normal(m.nv)))
    q = home.copy(); q[0] += 1e3                          # far from the origin
    v = 0.5 * rng.standard_normal(m.nv); v[3:6] = [6.0, -4.0, 5.0]
    out.append(("x1e3", q, v))
    return out


def scenes():
    """name -> Scene: every scene above."""
    out = {}
    for f in (free_top, ball_pendulum, multi_joint, joint_ref, odd_chain, forest, wide, quat_edges, far,
              slide_gravity, hinge_pendulum, double_pendulum):
        s = f()
        out[s.name] = s
    return out
