"""Purpose-built states and task snapshots for the task residuals (csrc/dev_task.cuh k_residual,
k_residual_quadruped and the ground ray-cast ground_height; oracle/residuals.h).

A case is one residual evaluation: (model, qpos, qvel, ctrl, mocap, time, task_state, parameters) and flags naming the
edge it sits on.  Cases whose value jumps at a threshold that fp32 cannot place where fp64 does (the |StepHeight| < 1e-6
cut, the edge of a ray target, the Flip posture switches, a Humanoid Track frame boundary, sub_quat at an angle of pi,
the Walk turn-rate threshold) carry `sides`: variants of the case a hair to either side of the threshold.  The device
must then equal fp64 evaluated at the case or at one of its sides, row by row.

Quadruped cases are placed with the home keyframe's joint angles and a trunk pose chosen so that the feet sit over the
terrain piece under test: the floor plane (z = -0.01), the tilted `ramp` box, the `hill` sphere, the movable mocap
`box` (mocap 1) and, in a model variant, a ball above the floor.  shifted(case, t0) moves a Quadruped case to absolute clock time t0: its time and every absolute time
of the task state (mode start, phase start time and the phase start, which the reset makes equal to the time).

Shared by tests/test_residuals_cpu.py and tests/test_gpu_residuals.py.
"""
import math

import numpy as np

CLOCK_SHIFTS = (0.0, 1e2, 1e4, 1e6)
# row groups of the Quadruped residual (42 rows: nu = 12)
QUAD_GROUPS = dict(upright=(0, 3), height=(3, 4), position=(4, 7), gait=(7, 11), balance=(11, 13), effort=(13, 25),
                   posture=(25, 37), yaw=(37, 39), angmom=(39, 42))

_MODELS = {}
BALL_CENTER, BALL_RADIUS = (1.0, 0.0, 0.1), 0.3


def model(name):
    """The built-in task model `name`, or a Quadruped variant with contacts disabled: "quadruped_nocontact", for poses
    far below the floor (whose contacts would overflow the contact buffer and raise the step's warning for that
    reason), and "quadruped_ball", whose `hill` sphere is a ball of radius BALL_RADIUS centred at BALL_CENTER, above the
    floor, so that a down-ray can pass it near its tangent and the hit is the nearest one."""
    if name not in _MODELS:
        from mujoco_mpc_b200 import models
        if name in ("quadruped_nocontact", "quadruped_ball"):
            from mujoco_mpc_b200.mjcf import compile_xml
            base = model("quadruped")
            text = models.quadruped_flat_xml().replace('impratio="10"/>', 'impratio="10"><flag contact="disable"/></option>')
            if name == "quadruped_ball":
                hill = '<geom name="hill" class="prop" pos="6 6 -5.5" size="6" type="sphere"/>'
                assert hill in text
                text = text.replace(hill, '<geom name="hill" class="prop" pos="%g %g %g" size="%g" type="sphere"/>'
                                    % (*BALL_CENTER, BALL_RADIUS))
            m = compile_xml(text)
            for k in ("task_residual_id", "task_ids", "task_state", "task_name", "opt_timestep", "ray_geoms"):
                m[k] = base[k]
        else:
            m = models.load(name)
        _MODELS[name] = m
    return _MODELS[name]


class Case:
    def __init__(self, name, model_name, qpos, qvel, ctrl, mocap, time, task_state, parameters, flags=(), sides=()):
        self.name, self.model_name = name, model_name
        self.qpos, self.qvel, self.ctrl = np.asarray(qpos, float), np.asarray(qvel, float), np.asarray(ctrl, float)
        self.mocap, self.time = np.asarray(mocap, float), float(time)
        self.task_state, self.parameters = np.asarray(task_state, float), np.asarray(parameters, float)
        self.flags = set(flags)
        self.sides = list(sides)      # dicts of fields that replace the case's to make one side of a threshold
        self.t0 = 0.0                 # the clock shift of shifted()

    @property
    def m(self):
        return model(self.model_name)

    def replace(self, **kw):
        c = Case(self.name, self.model_name, self.qpos, self.qvel, self.ctrl, self.mocap, self.time, self.task_state,
                 self.parameters, self.flags, self.sides)
        c.t0 = self.t0
        for k, v in kw.items():
            setattr(c, k, v if k in ("sides", "flags", "name", "t0") else np.asarray(v, float) if k != "time" else float(v))
        return c

    def side_cases(self):
        return [self.replace(**s, sides=[]) for s in self.sides]

    def rounded(self):
        """The inputs the device receives, rounded to fp32 and upcast (the time is relative to the case's clock shift,
        which stays exact: shifted() adds it in double)."""
        f = lambda a: np.asarray(a, np.float32).astype(float)
        t0 = self.t0
        return self.replace(qpos=f(self.qpos), qvel=f(self.qvel), ctrl=f(self.ctrl), mocap=f(self.mocap),
                            time=t0 + float(np.float32(self.time - t0)),
                            sides=[{**s, **{k: f(v) for k, v in s.items() if k in ("qpos", "mocap")}} for s in self.sides])


# ---------------------------------------------------------------------------------------------- Quadruped placement
def quad_mocap(m, goal=(0.3, 0.0, 0.26), box=(-2.5, 0.0, 0.0), box_quat=(1, 0, 0, 0)):
    bq = np.asarray(box_quat, float) / np.linalg.norm(box_quat)
    return np.concatenate([goal, [1, 0, 0, 0], box, bq])


def foot_offsets(m):
    """World offsets of the four foot geoms (FL, HL, FR, HR: task_ids order) from the trunk at the home pose."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.refmath import kinematics
    q = np.asarray(m.key_qpos[0], float).copy()
    q[:3] = 0
    kin = kinematics(m, q)
    out = []
    for f in range(4):
        g = int(m.task_ids[T.QI_FOOT_GEOM + f])
        b = m.geom_bodyid[g]
        out.append(kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g])
    return np.array(out)


def quad_qpos(m, x, y, z, quat=(1, 0, 0, 0), joints=None):
    q = np.asarray(m.key_qpos[0], float).copy()
    q[:3] = (x, y, z)
    q[3:7] = np.asarray(quat, float) / np.linalg.norm(quat)
    if joints is not None:
        q[7:] = joints
    return q


def quat_about(axis, angle):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([[math.cos(angle / 2)], math.sin(angle / 2) * a])


def step_height64(phase, footphase, duty):
    """StepHeight (quadruped.cc) in double."""
    angle = math.fmod(phase + math.pi - footphase, 2 * math.pi) - math.pi
    value = 0.0
    if duty < 1:
        angle *= 0.5 / (1 - duty)
        value = math.cos(max(-math.pi / 2, min(math.pi / 2, angle)))
    return 0.0 if abs(value) < 1e-6 else value


def quadruped_cases():
    from mujoco_mpc_b200 import task as T
    m = model("quadruped")
    pn = [p[len("residual_"):] for p in m.task_parameter_names]
    P0 = np.asarray(m.task_parameters, float)
    S0 = np.asarray(m.task_state, float)
    rng = np.random.default_rng(11)
    nu = m.nu

    def params(**kw):
        p = P0.copy()
        names = dict(gait="select_Gait", biped="select_Biped type", cadence="Cadence", amp="Amplitude",
                     duty="Duty ratio", speed="Walk speed", turn="Walk turn", flip="select_Flip dir",
                     heading="Heading", arm="Arm posture")
        for k, v in kw.items():
            p[pn.index(names[k])] = v
        return p

    def state(mode=0, gait=0, cadence=2.0, mode_start=0.0, phase_start=0.0, heading=(0.4, 0.2), position=(0.1, -0.2, 0.26),
              speed=0.0, angvel=0.0, ground=0.0, orientation=(1, 0, 0, 0)):
        s = S0.copy()
        s[T.QS_MODE], s[T.QS_GAIT] = mode, gait
        s[T.QS_MODE_START_TIME] = mode_start
        s[T.QS_PHASE_START] = s[T.QS_PHASE_START_TIME] = phase_start      # the reset (and a mode switch) sets both
        s[T.QS_PHASE_VELOCITY] = 2 * math.pi * cadence
        s[T.QS_POSITION:T.QS_POSITION + 3] = position
        s[T.QS_HEADING:T.QS_HEADING + 2] = heading
        s[T.QS_SPEED], s[T.QS_ANGVEL], s[T.QS_GROUND] = speed, angvel, ground
        s[T.QS_ORIENTATION:T.QS_ORIENTATION + 4] = orientation
        return s

    qv = 0.3 * rng.standard_normal(m.nv)
    ctrl = np.clip(0.6 * rng.standard_normal(nu), -1.2, 1.2)
    ctrl[0], ctrl[5] = 1.7, -1.4                                    # outside ctrlrange: the force uses the clamp
    foot = foot_offsets(m)
    z0 = 0.02 - foot[:, 2].min() - 0.01                             # lowest foot 1 cm below its rest height
    out = []

    def add(name, qpos=None, time=0.37, ts=None, prm=None, mocap=None, flags=(), sides=(), qvel=qv, u=ctrl):
        out.append(Case(name, "quadruped", quad_qpos(m, 0.05, -0.03, z0 + 0.004) if qpos is None else qpos, qvel, u,
                        quad_mocap(m) if mocap is None else mocap, time, state() if ts is None else ts,
                        P0 if prm is None else prm, flags, sides))

    tilt = quat_about((0.3, 1, 0.2), 0.15)
    # ---- modes
    add("quadruped", qpos=quad_qpos(m, 0.05, -0.03, z0 + 0.004, tilt))
    for bt in (0, 1):
        add(f"biped_type{bt}", qpos=quad_qpos(m, 0.05, -0.03, 0.45, quat_about((0, 1, 0), (-1 if bt else 1) * 1.2)),
            ts=state(mode=1), prm=params(biped=bt, arm=0.4))
    add("walk_straight", ts=state(mode=2, speed=0.7, angvel=0.0), prm=params(speed=0.7))
    add("walk_turning", ts=state(mode=2, speed=0.7, angvel=0.8, mode_start=0.1), prm=params(turn=0.8))
    add("walk_turn_below_threshold", ts=state(mode=2, speed=0.7, angvel=0.0099))
    add("walk_turn_negative", ts=state(mode=2, speed=0.7, angvel=-0.5))
    # just under the 0.01 threshold in double is 0.01f in fp32, on the other side of fabsf(x) < 0.01f
    add("walk_turn_at_threshold", ts=state(mode=2, speed=0.7, angvel=0.01 - 1e-10), flags=("discontinuous",),
        sides=[dict(task_state=state(mode=2, speed=0.7, angvel=0.01))])
    add("walk_zero_heading", ts=state(mode=2, speed=0.7, angvel=0.0, heading=(0.0, 0.0)))
    add("scramble", ts=state(mode=3), prm=params(gait=1), mocap=quad_mocap(m, goal=(0.9, 0.4, 0.35)))
    for fd in (0, 1):
        add(f"flip_dir{fd}", ts=state(mode=4, mode_start=0.2), prm=params(flip=fd), time=0.2 + 0.33,
            qpos=quad_qpos(m, 0.05, -0.03, 0.5, quat_about((0, 1, 0), 0.7)))
    # ---- gaits and duty ratios (gait rows: times spread over the cycle so that every foot is in the air somewhere)
    for g in range(5):
        for k, t in enumerate((0.05, 0.18, 0.29, 0.41)):
            add(f"gait{g}_t{k}", ts=state(gait=g), prm=params(gait=g, amp=0.08, duty=0.3), time=t)
    for duty in (0.0, 0.3, 0.99, 1.0):
        add(f"duty{duty}", ts=state(gait=1), prm=params(gait=1, amp=0.08, duty=duty), time=0.23)
    add("amplitude0", ts=state(gait=1), prm=params(gait=1, amp=0.0, duty=0.3), time=0.23)
    # the |StepHeight| < 1e-6 cut: foot 0 of gait 0 with duty 0 at cos(angle) = 1e-6 (phase + pi = 2 pi + 2e-6)
    t_cut = (math.pi + 2e-6) / (4 * math.pi)
    add("step_height_cut", ts=state(gait=0), prm=params(gait=0, amp=0.08, duty=0.0), time=t_cut,
        flags=("discontinuous",), sides=[dict(time=t_cut - 2e-6), dict(time=t_cut + 2e-6)])
    # ---- Flip clock: mode times before, at and after each segment boundary
    S = S0
    bounds = dict(crouch=S[T.QS_CROUCH_TIME], jump=S[T.QS_JUMP_TIME], land=S[T.QS_JUMP_TIME] + S[T.QS_FLIGHT_TIME],
                  end=S[T.QS_JUMP_TIME] + S[T.QS_FLIGHT_TIME] + S[T.QS_LAND_TIME])
    ms = 0.3
    for bname, b in bounds.items():
        for tag, dt in (("before", -2e-3), ("at", 0.0), ("after", 2e-3)):
            t = ms + b + dt
            kw = {}
            if tag == "at":
                kw = dict(flags=("discontinuous",), sides=[dict(time=t - 1e-5), dict(time=t + 1e-5)])
            add(f"flip_{bname}_{tag}", ts=state(mode=4, mode_start=ms, ground=0.02), prm=params(flip=1), time=t,
                qpos=quad_qpos(m, 0.0, 0.0, 0.45, quat_about((0, 1, 0), 1.0)), **kw)
    # ---- terrain: feet over the ramp, the hill, the mocap box (moved and rotated), grazing the box edge
    ramp_c = m.geom_pos[list(m.geom_names).index("ramp")]
    ramp_top = lambda x, y: ramp_c[2] + (0.5 - math.sin(0.2) * (x - ramp_c[0])) / math.cos(0.2)   # rough: placement only
    add("ramp", qpos=quad_qpos(m, 3.0, 2.4, ramp_top(3.0, 2.4) + z0 + 0.02), ts=state(gait=1),
        prm=params(gait=1, amp=0.08, duty=0.3), time=0.18)
    add("ramp_tilted_body", qpos=quad_qpos(m, 2.2, 2.9, ramp_top(2.2, 2.9) + z0 + 0.03, quat_about((0, 1, 0), -0.2)),
        ts=state(gait=3), prm=params(gait=3, amp=0.08, duty=0.3), time=0.29)
    add("hill_top", qpos=quad_qpos(m, 6.0, 6.1, 0.5 + z0 + 0.02), ts=state(gait=1), prm=params(gait=1, amp=0.08, duty=0.3),
        time=0.18)
    add("hill_slope", qpos=quad_qpos(m, 7.5, 6.4, 6 * math.cos(math.asin(1.55 / 6)) - 5.5 + z0 + 0.05), ts=state(gait=2),
        prm=params(gait=2, amp=0.08, duty=0.3), time=0.11)
    # the hill's rim, where its cap meets the floor (foot 0 over the cap, 1.2 mm above the floor plane)
    add("hill_rim", qpos=quad_qpos(m, 6.0 - 2.418 - foot[0, 0], 6.0 - foot[0, 1], z0 + 0.01), ts=state(gait=0),
        prm=params(gait=0, amp=0.08, duty=0.3), time=0.1)
    # foot 0's down-ray passing a ball above the floor 1e-3 r inside its tangent (a hit near the equator) and 1e-3 r
    # outside (a miss: the floor).  At the tangent itself the hit height is cz + sqrt(det) / |v| with det a difference
    # of rounded squares, so one ulp of det moves it by ~1e-4 m in fp32: no bar can pin that, these two bracket it.
    for tag, d in (("inside", 1 - 1e-3), ("outside", 1 + 1e-3)):
        x = BALL_CENTER[0] - d * BALL_RADIUS - foot[0, 0]
        out.append(Case(f"ball_near_tangent_{tag}", "quadruped_ball", quad_qpos(m, x, BALL_CENTER[1] - foot[0, 1], z0 + 0.11),
                        qv, ctrl, quad_mocap(m), 0.1, state(gait=0), params(gait=0, amp=0.08, duty=0.3)))
    add("box_top", qpos=quad_qpos(m, -2.5, 0.1, 0.3 + z0 + 0.02), ts=state(gait=1), prm=params(gait=1, amp=0.08, duty=0.3),
        time=0.18)
    mb = quad_mocap(m, box=(0.4, -0.3, -0.1), box_quat=quat_about((0.2, 0.1, 1.0), 0.6))
    add("box_moved_rotated", qpos=quad_qpos(m, 0.3, -0.2, 0.2 + z0 + 0.05), mocap=mb, ts=state(gait=4),
        prm=params(gait=4, amp=0.08, duty=0.3), time=0.33)
    # front-left foot exactly above the box's edge x = -1.5 (box moved so that the edge is under it); sides move the box
    xe = 0.2 + foot[0, 0]
    box_at = lambda dx: quad_mocap(m, box=(xe - 1.0 + dx, 0.0, 0.0))
    add("box_edge", qpos=quad_qpos(m, 0.2, 0.0, 0.3 + z0 + 0.02), mocap=box_at(0.0), ts=state(gait=0),
        prm=params(gait=0, amp=0.08, duty=0.3), time=0.1, flags=("discontinuous", "ray_edge"),
        sides=[dict(mocap=box_at(-1e-5)), dict(mocap=box_at(1e-5))])
    # ---- Scramble: a foot directly under the goal (zero-length normalize3 of the goal offset)
    g = np.array([0.4 + foot[0, 0], -0.1 + foot[0, 1], 0.3])
    add("scramble_foot_under_goal", qpos=quad_qpos(m, 0.4, -0.1, z0 + 0.01), mocap=quad_mocap(m, goal=g),
        ts=state(mode=3, gait=0), prm=params(gait=0, amp=0.08, duty=0.3), time=0.1)
    # ---- nothing below the feet: every ray misses, the warning must be set
    out.append(Case("warning_below_floor", "quadruped_nocontact", quad_qpos(m, 0.0, 0.0, -1.0), qv, ctrl, quad_mocap(m),
                    0.18, state(gait=1), params(gait=1, amp=0.08, duty=0.3), flags=("warning",)))
    return out


def shifted(case, t0):
    """The Quadruped case at absolute clock time t0: time, mode start, phase start time and phase start moved by t0."""
    from mujoco_mpc_b200 import task as T
    s = case.task_state.copy()
    for i in (T.QS_MODE_START_TIME, T.QS_PHASE_START_TIME, T.QS_PHASE_START):
        s[i] += t0
    sides = []
    for d in case.sides:
        d = dict(d)
        if "time" in d:
            d["time"] += t0
        if "task_state" in d:
            d["task_state"] = shifted(case.replace(task_state=d["task_state"], sides=[]), t0).task_state
        sides.append(d)
    return case.replace(time=case.time + t0, task_state=s, sides=sides, t0=t0, name=f"{case.name}@{t0:g}")


# ---------------------------------------------------------------------------------------------- other residuals
def other_cases():
    from mujoco_mpc_b200 import task as T
    out = []
    rng = np.random.default_rng(5)
    # Cartpole at small pole angles (cos(q) - 1 cancels)
    m = model("cartpole")
    for a in (0.0, 1e-4, 3e-3, 0.2):
        out.append(Case(f"cartpole_{a:g}", "cartpole", [0.3, a], [0.1, -0.4], [0.5], [], 0.2, m.task_state,
                        m.task_parameters))
    # Humanoid Stand
    m = model("humanoid")
    q = np.asarray(m.qpos0, float).copy(); q[7:] += 0.1 * rng.standard_normal(m.nq - 7)
    out.append(Case("humanoid_stand", "humanoid", q, 0.4 * rng.standard_normal(m.nv), rng.uniform(-1, 1, m.nu), [], 0.3,
                    m.task_state, m.task_parameters))
    # Humanoid Track: every clip; before the reference time, on a frame, on the clip's last frame and past it
    m = model("humanoid_track")
    mocap = np.concatenate([np.asarray(m.key_mpos[0]).reshape(-1, 3), np.tile([1.0, 0, 0, 0], (m.nmocap, 1))], 1).reshape(-1)
    ref = 0.25
    for clip, length in enumerate(T.TRACK_MOTION_LENGTHS):
        start = sum(T.TRACK_MOTION_LENGTHS[:clip])
        q = np.asarray(m.key_qpos[start + 3], float).copy(); q[2] += 0.5
        v, u = 0.3 * rng.standard_normal(m.nv), rng.uniform(-1, 1, m.nu)
        ts = np.array([float(clip), ref])
        times = dict(before=ref - 0.1, inside=ref + 0.0123 + 0.031 * clip, frame=ref + 7 / 30.0,
                     last=ref + (length - 1) / 30.0, past=ref + length / 30.0 + 1.0)
        for tag, t in times.items():
            kw = {}
            if tag in ("frame", "last"):
                kw = dict(flags=("discontinuous",), sides=[dict(time=t - 1e-6), dict(time=t + 1e-6)])
            out.append(Case(f"track_clip{clip}_{tag}", "humanoid_track", q, v, u, mocap, t, ts, m.task_parameters, **kw))
    # Shadow Reorient: the goal's ball joint (qpos 0:4) against the cube's free joint quaternion (qpos 7:11)
    m = model("shadow_reorient")
    q0 = np.asarray(m.key_qpos[0], float).copy()
    cube = q0[7:11] / np.linalg.norm(q0[7:11])
    v, u = 0.2 * rng.standard_normal(m.nv), rng.uniform(-0.5, 0.5, m.nu)

    def qmul(a, b):
        w1, x1, y1, z1 = a; w2, x2, y2, z2 = b
        return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                         w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])

    def goal(qg):
        q = q0.copy(); q[0:4] = qg
        return q
    axis = np.array([0.3, -0.5, 0.8])
    out.append(Case("shadow_goal_is_cube", "shadow_reorient", goal(cube), v, u, [], 0.1, m.task_state, m.task_parameters))
    out.append(Case("shadow_goal_minus_cube", "shadow_reorient", goal(-cube), v, u, [], 0.1, m.task_state,
                    m.task_parameters))
    out.append(Case("shadow_goal_unnormalised", "shadow_reorient", goal(1.7 * qmul(cube, quat_about(axis, 0.9))), v, u, [],
                    0.1, m.task_state, m.task_parameters))
    out.append(Case("shadow_goal_near_pi", "shadow_reorient", goal(qmul(cube, quat_about(axis, math.pi - 1e-3))), v, u, [],
                    0.1, m.task_state, m.task_parameters))
    out.append(Case("shadow_goal_at_pi", "shadow_reorient", goal(qmul(cube, quat_about(axis, math.pi))), v, u, [], 0.1,
                    m.task_state, m.task_parameters, flags=("discontinuous",),
                    sides=[dict(qpos=goal(qmul(cube, quat_about(axis, math.pi + d)))) for d in (-1e-4, 1e-4)]))
    return out
