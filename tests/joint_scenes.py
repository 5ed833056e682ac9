"""Purpose-built joint-space scenes: dof friction loss, joint limits, passive forces (springs, damping, armature),
actuation and the <option><flag> switches (csrc/dev_physics.cuh k_make_constraint / k_smooth_forces / k_euler,
oracle/physics.h make_constraint / passive / actuation / euler).

Most scenes are built from independent units: one root body per joint (a slide along world x, a hinge about world z
carrying a sphere at an offset, a ball or a free joint carrying a centred sphere), with contacts switched off.  The
joint-space inertia is then diagonal and known in closed form (slide: m; hinge: 2/5 m r^2 + m d^2; ball and free
rotation: 2/5 m r^2, isotropic so that the gyroscopic term vanishes; plus armature), gravity acts on the free joints'
z dof only, and every dof's constraint problem is one-dimensional: tests/test_oracle_joint_constraints.py solves it in
closed form.  A pose is a (qpos, qvel, ctrl) triple.

The path scenes (hinge chains, 18-dof trees, many limited hinges, the capacity scene) and the mixed scene are only
compared device against oracle (tests/test_gpu_joint_constraints.py).

Shared by tests/test_oracle_joint_constraints.py and tests/test_gpu_joint_constraints.py.
"""
import numpy as np

DT = 0.01
G = 9.81
QROT = np.array([0.8, 0.2, -0.4, 0.4]) / np.linalg.norm([0.8, 0.2, -0.4, 0.4])


class Unit:
    """One root body with one joint.  attrs: extra <joint> attributes; d: sphere offset of a hinge."""

    def __init__(self, kind, attrs="", m=1.0, r=0.1, d=0.0):
        self.kind, self.attrs, self.m, self.r, self.d = kind, attrs, m, r, d

    @property
    def nq(self):
        return {"slide": 1, "hinge": 1, "ball": 4, "free": 7}[self.kind]

    @property
    def nv(self):
        return {"slide": 1, "hinge": 1, "ball": 3, "free": 6}[self.kind]

    def inertia(self):
        """Joint-space inertia of each dof without armature, in closed form."""
        rot = 0.4 * self.m * self.r ** 2
        if self.kind == "slide":
            return np.array([self.m])
        if self.kind == "hinge":
            return np.array([rot + self.m * self.d ** 2])
        if self.kind == "ball":
            return np.full(3, rot)
        return np.array([self.m] * 3 + [rot] * 3)

    def gravity(self):
        """Generalised gravity force on each dof."""
        out = np.zeros(self.nv)
        if self.kind == "free":
            out[2] = -self.m * G
        return out

    def xml(self, k):
        geom = (f'<geom type="sphere" size="{self.r}" mass="{self.m}" pos="{self.d} 0 0" contype="0" '
                f'conaffinity="0"/>')
        axis = {"slide": ' axis="1 0 0"', "hinge": ' axis="0 0 1"'}.get(self.kind, "")
        return (f'<body name="b{k}" pos="0 {0.5 * k} 1"><joint name="j{k}" type="{self.kind}"{axis} {self.attrs}/>'
                f'{geom}</body>')


def scene_xml(name, units=(), bodies="", actuator="", flags="", floor=False, option=""):
    body = "".join(u.xml(k) for k, u in enumerate(units)) + bodies
    fl = f"<flag {flags}/>" if flags else ""
    return f"""
<mujoco model="{name}">
  <compiler angle="radian"/>
  <option timestep="{DT}"{option}>{fl}</option>
  <custom><numeric name="agent_planner" data="0"/><numeric name="agent_horizon" data="0.1"/></custom>
  <worldbody>
    <body name="target" mocap="true" pos="0 0 3"><geom type="sphere" size="0.01" contype="0" conaffinity="0"/></body>
    {'<geom name="floor" type="plane" size="5 5 .1"/>' if floor else ''}
    {body}
  </worldbody>
  <actuator>{actuator}</actuator>
  {{sensor}}
</mujoco>"""


def compile_scene(text):
    """Compile with a particle-copy cost (residual = the state), so that rollouts have a non-trivial return."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.mjcf import compile_xml
    m0 = compile_xml(text.replace("{sensor}", ""))
    dim = m0.nq + m0.nv
    m = compile_xml(text.replace("{sensor}", f'<sensor><user name="State" dim="{dim}" user="0 1 0 1"/></sensor>'))
    m.task_residual_id = T.RESIDUAL_PARTICLE_COPY
    m.task_ids, m.task_state, m.ray_geoms = np.zeros(1, np.int32), np.zeros(1), np.zeros(0, np.int32)
    return m


class Scene:
    """A model (independent units and / or free-form bodies) and its poses: (name, qpos, qvel, ctrl)."""

    def __init__(self, name, units=(), poses=(), actuators=(), flags="", bodies="", floor=False, option=""):
        self.name, self.units, self.actuators = name, list(units), list(actuators)
        self.flags, self.bodies, self.floor, self.option = flags, bodies, floor, option
        self.poses = list(poses)

    def text(self):
        acts = "".join(a.xml() for a in self.actuators)
        return scene_xml(self.name, self.units, self.bodies, acts, self.flags, self.floor, self.option)


class Act:
    """One actuator on joint j{joint}: kind motor / position / velocity / general (affine bias)."""

    def __init__(self, kind, joint, gear=1.0, kp=1.0, kv=0.0, gain=1.0, bias=(0, 0, 0), ctrlrange=None,
                 ctrllimited=None, forcerange=None):
        self.kind, self.joint, self.gear, self.kp, self.kv, self.gain, self.bias = kind, joint, gear, kp, kv, gain, bias
        self.ctrlrange, self.ctrllimited, self.forcerange = ctrlrange, ctrllimited, forcerange

    def xml(self):
        a = f'joint="j{self.joint}" gear="{self.gear}"'
        if self.kind == "position":
            a += f' kp="{self.kp}" kv="{self.kv}"'
        elif self.kind == "velocity":
            a += f' kv="{self.kv}"'
        elif self.kind == "general":
            a += f' gainprm="{self.gain}" biastype="affine" biasprm="{" ".join(str(b) for b in self.bias)}"'
        if self.ctrlrange is not None:
            a += f' ctrlrange="{self.ctrlrange[0]} {self.ctrlrange[1]}"'
        if self.ctrllimited is not None:
            a += f' ctrllimited="{self.ctrllimited}"'
        if self.forcerange is not None:
            a += f' forcerange="{self.forcerange[0]} {self.forcerange[1]}"'
        return f"<{self.kind} {a}/>"

    def force(self, ctrl, q, v):
        """Closed form of the actuator force (before the gear moves it to the joint)."""
        limited = self.ctrllimited == "true" or (self.ctrllimited is None and self.ctrlrange is not None)
        if limited:
            ctrl = min(max(ctrl, self.ctrlrange[0]), self.ctrlrange[1])
        L, V = self.gear * q, self.gear * v
        f = {"motor": lambda: ctrl,
             "position": lambda: self.kp * ctrl - self.kp * L - self.kv * V,
             "velocity": lambda: self.kv * ctrl - self.kv * V,
             "general": lambda: self.gain * ctrl + self.bias[0] + self.bias[1] * L + self.bias[2] * V}[self.kind]()
        if self.forcerange is not None:
            f = min(max(f, self.forcerange[0]), self.forcerange[1])
        return f


# ---------------------------------------------------------------------------------------------- friction loss
_FR_CUSTOM = 'solreffriction="0.05 0.7" solimpfriction="0.8 0.95 0.01 0.5 2"'


def _friction_scene(name, extra="", flags=""):
    """Six units: slide and hinge (default and custom solref / solimp), a ball and two free bodies (weight below and
    above the friction threshold on z), all with frictionloss; `extra` adds to every joint (armature, damping)."""
    units = [Unit("slide", f'frictionloss="0.5" {extra}', m=2.0),
             Unit("slide", f'frictionloss="0.8" {_FR_CUSTOM} {extra}', m=0.7),
             Unit("hinge", f'frictionloss="0.05" {extra}', m=1.5, r=0.05, d=0.3),
             Unit("ball", f'frictionloss="0.02" {_FR_CUSTOM} {extra}', m=3.0, r=0.2),
             Unit("free", f'frictionloss="3" {extra}', m=0.2, r=0.1),      # m g = 1.96 < 3: sticks on z
             Unit("free", f'frictionloss="1" {extra}', m=0.5, r=0.1)]      # m g = 4.9 > 1: slides down
    acts = [Act("motor", 0, ctrlrange=(-10, 10)), Act("motor", 1, ctrlrange=(-10, 10)),
            Act("motor", 2, ctrlrange=(-10, 10))]
    ball = QROT
    free = lambda z: np.concatenate([[0.1, 0.2, z], QROT])

    def pose(name, q, v, u):
        return (name, np.concatenate([np.atleast_1d(x) for x in q]), np.asarray(v, float), np.asarray(u, float))

    q0 = [0.1, -0.2, 0.3, ball, free(1.0), free(1.5)]
    zeros = np.zeros(1 + 1 + 1 + 3 + 6 + 6)
    poses = [
        # at rest, force below the threshold: the quadratic zone (only the regularisation lets the dof move)
        pose("rest_below", q0, zeros, [0.3, -0.5, 0.02]),
        # at rest, force above the threshold, both signs: the linear zone, |force| = frictionloss
        pose("rest_above_pos", q0, zeros, [2.0, 3.0, 0.2]),
        pose("rest_above_neg", q0, zeros, [-2.0, -3.0, -0.2]),
        # moving: aref = -B v decides the zone
        pose("moving", q0, np.concatenate([[0.3, -0.2, 0.5], [0.2, -0.1, 0.3], [0.1, 0.2, -0.1, 0.5, -0.3, 0.2],
                                           [-0.2, 0.1, 0.05, 0.0, 0.4, -0.6]]), [0.1, 0.1, 0.0]),
        pose("moving_slow", q0, np.concatenate([[1e-3, -2e-3, 1e-3], [5e-4, 0, -1e-3], 1e-3 * np.ones(6),
                                                -1e-3 * np.ones(6)]), [0.2, -0.2, 0.01]),
    ]
    return Scene(name, units, poses, acts, flags=flags)


# ---------------------------------------------------------------------------------------------- joint limits
def _limit_units():
    """Slide and hinge limits with every solref / solimp branch (each unit's comment says which)."""
    return [
        Unit("slide", 'range="-0.3 0.4"', m=1.0),                                                   # defaults
        Unit("hinge", 'range="-0.5 0.8" ref="0.3" margin="0.05"', m=2.0, r=0.05, d=0.2),           # ref != 0, margin
        Unit("slide", 'range="-0.05 0.05" margin="0.1"', m=0.5),                                    # both rows always
        Unit("slide", 'range="-0.3 0.4" solreflimit="-2000 -30"', m=1.2),                          # direct K, B
        Unit("hinge", 'range="-0.5 0.5" solreflimit="0.005 1.2"', m=1.0, r=0.05, d=0.1),           # tc < 2 dt
        Unit("slide", 'range="-0.3 0.4" solimplimit="0.5 0.95 0.1 0.5 1"', m=0.8),                 # power 1
        Unit("slide", 'range="-0.3 0.4" solimplimit="0.3 0.97 0.1 0.4 3"', m=0.9),                 # power 3, mid 0.4
        Unit("hinge", 'range="-0.5 0.5" solimplimit="0.9 0.9 0.01 0.5 2" armature="0.05"', m=1.0, r=0.05, d=0.1),
    ]


def _limit_scene(name, flags=""):
    units = _limit_units()
    lo = np.array([-0.3, -0.5, -0.05, -0.3, -0.5, -0.3, -0.3, -0.5])
    hi = np.array([0.4, 0.8, 0.05, 0.4, 0.5, 0.4, 0.4, 0.5])
    margin = np.array([0, 0.05, 0.1, 0, 0, 0, 0, 0])
    n = len(units)
    rng = np.random.default_rng(7)
    v0 = np.zeros(n)
    vm = 0.4 * rng.standard_normal(n)

    def P(name, q, v):
        return (name, np.asarray(q, float), np.asarray(v, float), np.zeros(0))
    # every pose keeps dist - margin at least 5e-3 from zero (module docstring of the GPU test)
    poses = [P("inside", 0.5 * (lo + hi) + 0.01, v0),
             P("inside_margin_lo", lo + 0.5 * margin + np.where(margin > 0, 0, 0.02), v0),
             P("violated_lo", lo - 0.02, v0),
             P("violated_lo_deep", lo - 0.08, v0),
             P("violated_hi", hi + 0.02, v0),
             P("violated_hi_moving", hi + 0.03, vm),
             P("violated_lo_moving_out", lo - 0.03, -np.abs(vm)),
             P("violated_lo_moving_in", lo - 0.01, np.abs(vm) * 3)]
    return Scene(name, units, poses, flags=flags), lo, hi, margin


# ---------------------------------------------------------------------------------------------- passive forces
def _passive_scene(name, flags=""):
    units = [Unit("slide", 'stiffness="40" springref="0.2" ref="-0.1" damping="3" armature="0.2"', m=1.0),
             Unit("hinge", 'stiffness="2" springref="-0.4" ref="0.25" damping="0.5"', m=2.0, r=0.05, d=0.3),
             Unit("slide", 'damping="50" armature="0.1"', m=0.3),           # h b / m = 1.7: the implicit form matters
             Unit("ball", 'damping="0.3" armature="0.01"', m=1.0, r=0.2),
             Unit("free", 'damping="0.2"', m=1.0, r=0.1)]
    v = np.concatenate([[0.5, -1.0, 2.0], [0.3, -0.2, 0.4], [0.1, 0.2, -0.3, 1.0, -0.5, 0.2]])
    q = np.concatenate([[0.5, -0.3, 0.1], QROT, [0, 0, 1, 1, 0, 0, 0]])
    poses = [("spring_damper", q, v, np.zeros(0)), ("at_rest", q, 0 * v, np.zeros(0))]
    return Scene(name, units, poses, flags=flags)


# ---------------------------------------------------------------------------------------------- actuators
def _actuator_scene():
    units = [Unit("slide", "", m=1.0), Unit("slide", 'damping="1"', m=2.0), Unit("hinge", "", m=1.0, r=0.05, d=0.2),
             Unit("slide", "", m=0.5), Unit("slide", "", m=0.8)]
    acts = [Act("motor", 0, gear=-2.5, ctrlrange=(-1, 1)),                                        # negative gear
            Act("position", 1, gear=1.5, kp=30, kv=4, ctrlrange=(-0.5, 0.5)),
            Act("velocity", 2, gear=0.7, kv=6, ctrlrange=(-2, 2)),
            Act("general", 3, gear=2.0, gain=5, bias=(0.3, -7, -1.5), ctrlrange=(-1, 1)),          # all three terms
            Act("motor", 3, gear=-1.0, ctrlrange=(-1, 1), ctrllimited="false"),                   # second on joint 3
            Act("motor", 4, gear=3.0, ctrlrange=(-1, 1), forcerange=(-0.4, 0.6)),                 # forcelimited
            Act("position", 4, gear=1.0, kp=10, ctrlrange=(-1, 1), forcerange=(-2, 1.5))]
    q = np.array([0.3, -0.2, 0.4, 0.25, -0.1])
    v = np.array([0.5, -1.0, 0.8, -0.4, 0.3])
    poses = [("inside_ranges", q, v, np.array([0.4, 0.2, -1.0, 0.5, -0.6, 0.1, 0.3])),
             ("ctrl_out_of_range", q, v, np.array([3.0, -2.0, 5.0, -4.0, 7.5, 2.0, -3.0])),
             ("force_clamped_high", q, v, np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.9, 1.0])),
             ("force_clamped_low", q, v, np.array([0.0, 0.0, 0.0, 0.0, 0.0, -0.9, -1.0]))]
    return Scene("actuators", units, poses, acts)


# ---------------------------------------------------------------------------------------------- scenes
def closed_form_scenes():
    """Scenes of independent units (closed forms exist), name -> Scene."""
    out = {}
    out["friction"] = _friction_scene("friction")
    out["friction_armature_damping"] = _friction_scene("friction_armature_damping", 'armature="0.3" damping="2"')
    out["friction_flag_off"] = _friction_scene("friction_flag_off", flags='frictionloss="disable"')
    for nm, fl in (("limits", ""), ("limits_refsafe_off", 'refsafe="disable"'), ("limits_flag_off", 'limit="disable"')):
        out[nm] = _limit_scene(nm, flags=fl)[0]
    out["passive"] = _passive_scene("passive")
    out["passive_eulerdamp_off"] = _passive_scene("passive_eulerdamp_off", 'eulerdamp="disable"')
    out["actuators"] = _actuator_scene()
    return out



# ---------------------------------------------------------------------------------------------- flags
def flag_scene(flag, iterations=None):
    """Friction loss + limits + damping + a floor contact in one model, with `flag` disabled (or nothing: None);
    iterations caps the Newton solve."""
    units = [Unit("slide", 'frictionloss="0.5" range="-0.3 0.4" damping="20"', m=1.0),
             Unit("hinge", 'frictionloss="0.05" range="-0.5 0.5" solreflimit="0.005 1" damping="0.5"', m=1.0, r=0.05,
                  d=0.2)]
    bodies = ('<body name="ball" pos="0 -1 0.1"><freejoint/><geom type="sphere" size="0.1" mass="1"/></body>')
    acts = [Act("motor", 0, ctrlrange=(-10, 10))]
    fl = f'{flag}="disable"' if flag else ""
    return Scene(f"flag_{flag}", units, [], acts, flags=fl, bodies=bodies, floor=True,
                 option=f' iterations="{iterations}"' if iterations is not None else "")


FLAGS = ("frictionloss", "limit", "eulerdamp", "refsafe", "warmstart")


def flag_pose():
    # slide violated below and moving; hinge violated above (tc < 2 dt: refsafe matters); ball 2 mm into the floor
    q = np.concatenate([[-0.32, 0.52], [0, -1, 0.098, 1, 0, 0, 0]])
    v = np.concatenate([[0.4, -0.3], [0.2, 0.1, -0.2, 0.5, 0.3, -0.1]])
    return q, v, np.array([0.2])


# ---------------------------------------------------------------------------------------------- path scenes
def hinge_chain(n, attrs='frictionloss="0.1" damping="0.2" armature="0.01"'):
    """n hinges in one chain, axes alternating y / x, capsule links hanging down."""
    body = ""
    for k in range(n):
        ax = "0 1 0" if k % 2 == 0 else "1 0 0"
        body += (f'<body name="c{k}" pos="0 0 -0.1"><joint name="h{k}" type="hinge" axis="{ax}" {attrs}/>'
                 f'<geom type="capsule" fromto="0 0 0 0 0 -0.1" size="0.02" contype="0" conaffinity="0"/>')
    return f'<body name="root" pos="0 0 4">{body}{"</body>" * n}</body>'


def branches(nb, nper, attrs='frictionloss="0.1" damping="0.2" armature="0.01" range="-0.6 0.6"'):
    """nb chains of nper hinges each, hanging from a fixed base."""
    out = ""
    for b in range(nb):
        body = ""
        for k in range(nper):
            ax = "0 1 0" if k % 2 == 0 else "1 0 0"
            body += (f'<body name="c{b}_{k}" pos="0 0 -0.1"><joint name="h{b}_{k}" type="hinge" axis="{ax}" {attrs}/>'
                     f'<geom type="capsule" fromto="0 0 0 0 0 -0.1" size="0.02" contype="0" conaffinity="0"/>')
        out += f'<body name="base{b}" pos="{0.5 * b} 0 4">{body}{"</body>" * nper}</body>'
    return out


def independent_hinges(n, attrs):
    return "".join(f'<body name="i{k}" pos="{0.3 * k} 0 2"><joint name="h{k}" type="hinge" axis="0 0 1" {attrs}/>'
                   f'<geom type="sphere" size="0.05" pos="0.1 0 0" mass="1" contype="0" conaffinity="0"/></body>'
                   for k in range(n))


def path_scenes():
    """name -> (Scene, what the test asserts about the host-side model)."""
    lim = 'range="-0.4 0.4" frictionloss="0.05"'
    motor = lambda j: [ActNamed("motor", j, ctrlrange=(-1, 1))]
    return {
        # nv != 18, friction loss on every dof: generic Hessian, jt_force / row_dot; cached line search (<= 32 items)
        "chain10_floss": Scene("chain10_floss", bodies=hinge_chain(10), actuators=motor("h0")),
        # 34 friction rows: more than 32 work items, the uncached line search k_ls_eval
        "chain34_floss": Scene("chain34_floss", bodies=hinge_chain(34), actuators=motor("h0")),
        # 40 limited hinges: the joint-limit compaction runs a second 32-lane chunk
        "hinges40_limits": Scene("hinges40_limits", bodies=independent_hinges(40, 'range="-0.4 0.4"'),
                                 actuators=motor("h0")),
        # nv = 18: one chain (nhpair 171, the NQ = 6 Hessian) and three 6-hinge branches (nhpair 63, NQ = 4)
        "chain18": Scene("chain18", bodies=hinge_chain(18, 'frictionloss="0.1" damping="0.2" armature="0.01" '
                                                            'range="-0.6 0.6"'), actuators=motor("h0")),
        "branches3x6": Scene("branches3x6", bodies=branches(3, 6), actuators=motor("h0_0")),
        # capacity: 32 friction + 64 limit rows fill the 96-row buffer exactly; 34 + 68 = 102 rows do not fit
        "capacity_fits": Scene("capacity_fits", bodies=independent_hinges(32, lim + ' margin="0.5"'),
                               actuators=motor("h0")),
        "capacity_overflow": Scene("capacity_overflow", bodies=independent_hinges(34, lim + ' margin="0.5"'),
                                   actuators=motor("h0")),
    }


def mixed_scene(narrow=False, condim=3, joint_rows=True, cone="pyramidal", margin=0.0, legs=None):
    """Friction loss, limits and floor contacts in one model: limited, friction-loss legs on a free body.
    Three legs with hip ranges of +-0.5; narrow: six legs with ranges of +-0.05, so that six standing legs give
    6 friction + 6 limit + 24 contact rows (pyramidal condim 3: 4 rows per contact), more than 32 line-search work
    items.  legs overrides the number of legs; joint_rows=False drops the friction loss and the limits (contacts
    only); margin is the legs' geom margin
    (an elliptic contact's friction rows then sit at pos - margin = -margin, where only K = 0 keeps aref = -B v)."""
    n, rng = (6, "-0.05 0.05") if narrow else (3, "-0.5 0.5")
    n = legs or n
    jr = f'range="{rng}" frictionloss="0.3" margin="0.02"' if joint_rows else ""
    legs = "".join(
        f'<body name="leg{k}" pos="{0.15 * np.cos(2 * np.pi * k / n):.4f} {0.15 * np.sin(2 * np.pi * k / n):.4f} 0">'
        f'<joint name="hip{k}" type="hinge" axis="{-np.sin(2 * np.pi * k / n):.4f} {np.cos(2 * np.pi * k / n):.4f} 0" '
        f'{jr} damping="0.5" armature="0.01"/>'
        f'<geom type="capsule" fromto="0 0 0 0 0 -0.15" size="0.02" mass="0.2" condim="{condim}" '
        f'friction="0.8 0.05 0.02" margin="{margin}"/></body>' for k in range(n))
    bodies = f'<body name="torso" pos="0 0 0.2"><freejoint/><geom type="box" size="0.15 0.15 0.03" mass="2"/>{legs}</body>'
    return Scene("mixed", bodies=bodies, floor=True, option=f' cone="{cone}"',
                 actuators=[ActNamed("motor", f"hip{k}", gear=2.0, ctrlrange=(-1, 1)) for k in range(n)])


class ActNamed(Act):
    """An actuator on a joint given by name."""

    def xml(self):
        return super().xml().replace(f'joint="j{self.joint}"', f'joint="{self.joint}"')


def nhpair(m):
    """Lower-triangle nonzeros of the tree-sparse mass matrix: each dof with all its ancestors."""
    n = 0
    for i in range(m.nv):
        j = i
        while j >= 0:
            n += 1
            j = int(m.dof_parentid[j])
    return n
