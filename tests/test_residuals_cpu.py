"""The fp64 oracle's task residuals (oracle/residuals.h) pinned to an independent restatement.

The Quadruped residual (mjpc/tasks/quadruped/quadruped.cc Residual) is restated here in numpy from its formulas, on
refmath's kinematics and Jacobians (world-frame Jacobians, not the oracle's composite recursion): foot geom and head
site positions from the body frames, the torso subtree's centre of mass and linear velocity from masses and Jacobians,
actuator forces from the gain and bias parameters with the control clamped, and the ground under each foot from
closed-form geometry (the floor plane's height, the height of a box face under the query point, a sphere's cap height)
instead of a ray-cast.  It is compared with oracle.forward_debug on every case of tests/residual_scenes.py.  The Flip
trajectory's closed forms (continuity, the leap height and angle) are checked on the task-state block the reset makes.
"""
import math

import numpy as np
import pytest

import residual_scenes as RS


@pytest.fixture(scope="module")
def oracles(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    cache = {}

    def get(name):
        if name not in cache:
            m = RS.model(name)
            cache[name] = oracle_lib.Oracle(to_blob(m), m, 64)
        return cache[name]
    return get


def oracle_residual(o, c):
    o.set_task(parameters=c.parameters, task_state=c.task_state)
    r = o.forward_debug(c.qpos, c.qvel, c.ctrl, c.mocap, time=c.time)
    return r["residual"][: c.m.task_num_residual], r["warning"]


# ---------------------------------------------------------------------------------------------- numpy restatement
def _qmul(a, b):
    w1, x1, y1, z1 = a; w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def _rotvec_diff(qa, qb):
    """The rotation vector v with qb * exp(v) = qa, angle in (-pi, pi] (mju_subQuat)."""
    qd = _qmul(qb * [1, -1, -1, -1], qa)
    s = np.linalg.norm(qd[1:])
    axis = qd[1:] / s if s >= 1e-15 else np.array([1.0, 0, 0])
    angle = 2 * math.atan2(s, qd[0])
    if angle > math.pi:
        angle -= 2 * math.pi
    return axis * angle


def _quat2mat(q):
    from mujoco_mpc_b200.mjcf import quat2mat
    return quat2mat(np.asarray(q, float) / np.linalg.norm(q))


def ground_height(m, kin, mocap_pos, mocap_quat, query):
    """Height of the highest surface of a ray geom at or below `query` on the vertical through it (None: none):
    a plane's height at (x, y), the face of a box facing up whose footprint holds (x, y), a sphere's upper cap."""
    x, y, qz = query
    hits = []
    for g in m.ray_geoms:
        b = m.geom_bodyid[g]
        if m.body_mocapid[b] >= 0:
            k = m.body_mocapid[b]
            bp, bR = mocap_pos[k], _quat2mat(mocap_quat[k])
        else:
            bp, bR = kin["xpos"][b], kin["xmat"][b]
        c = bp + bR @ m.geom_pos[g]
        R = bR @ _quat2mat(m.geom_quat[g])
        size, t = m.geom_size[g], m.geom_type[g]
        if t == 0:                                    # plane: n . (p - c) = 0
            n = R[:, 2]
            h = c[2] - (n[0] * (x - c[0]) + n[1] * (y - c[1])) / n[2]
            local = R.T @ (np.array([x, y, h]) - c)
            if all(size[i] <= 0 or abs(local[i]) <= size[i] for i in (0, 1)):
                hits.append(h)
        elif t == 2:                                  # sphere
            d2 = (x - c[0]) ** 2 + (y - c[1]) ** 2
            if d2 <= size[0] ** 2:
                hits.append(c[2] + math.sqrt(size[0] ** 2 - d2))
        elif t == 6:                                  # box: every face whose outward normal points up
            for i in range(3):
                for s in (-1, 1):
                    n = s * R[:, i]
                    if n[2] <= 1e-12:
                        continue
                    h = c[2] + (size[i] - n[0] * (x - c[0]) - n[1] * (y - c[1])) / n[2]
                    local = R.T @ (np.array([x, y, h]) - c)
                    if all(abs(local[j]) <= size[j] * (1 + 1e-12) for j in range(3) if j != i):
                        hits.append(h)
    hits = [h for h in hits if h <= qz]
    return max(hits) if hits else None


def flip_height(S, t):
    from mujoco_mpc_b200 import task as T
    jump, flight, land = S[T.QS_JUMP_TIME], S[T.QS_FLIGHT_TIME], S[T.QS_LAND_TIME]
    if t >= jump + flight + land:
        return 0.25 + S[T.QS_GROUND]
    if t < jump:
        h = 0.25 + t * S[T.QS_CROUCH_VEL] + 0.5 * t * t * S[T.QS_JUMP_ACC]
    elif t < jump + flight:
        t -= jump
        h = 0.5 + S[T.QS_JUMP_VEL] * t - 0.5 * 9.81 * t * t
    else:
        t -= jump + flight
        h = 0.5 - S[T.QS_JUMP_VEL] * t + 0.5 * S[T.QS_LAND_ACC] * t * t
    return h + S[T.QS_GROUND]


def flip_angle(S, t):
    from mujoco_mpc_b200 import task as T
    jump, flight, land, crouch = S[T.QS_JUMP_TIME], S[T.QS_FLIGHT_TIME], S[T.QS_LAND_TIME], S[T.QS_CROUCH_TIME]
    if t >= jump + flight + land:
        return 2 * math.pi
    if crouch <= t < jump:
        t -= crouch
        return 0.5 * S[T.QS_JUMP_ROT_ACC] * t * t + S[T.QS_JUMP_ROT_VEL] * t
    if jump <= t < jump + flight:
        return math.pi / 2 + S[T.QS_FLIGHT_ROT_VEL] * (t - jump)
    if t >= jump + flight:
        t -= jump + flight
        return 1.75 * math.pi + S[T.QS_FLIGHT_ROT_VEL] * t - 0.5 * S[T.QS_LAND_ROT_ACC] * t * t
    return 0.0


def flip_quat(S, t, flip_dir):
    from mujoco_mpc_b200 import task as T
    a = flip_angle(S, t)
    q = np.array([math.cos(a / 2), 0, (1 if flip_dir else -1) * math.sin(a / 2), 0])
    return _qmul(S[T.QS_ORIENTATION:T.QS_ORIENTATION + 4], q)


GAIT_PHASE = ((0, 0, 0, 0), (0, 0.75, 0.5, 0.25), (0, 0.5, 0.5, 0), (0, 0.33, 0.33, 0.66), (0, 0.4, 0.05, 0.35))


def quadruped_residual(c):
    """(residual, warning) of the Quadruped task at case c, restated in numpy."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.refmath import body_jacobian, kinematics
    m, S, I, prm = c.m, c.task_state, c.m.task_ids, c.parameters
    param = lambda qi: prm[I[qi]]
    mp = c.mocap.reshape(-1, 7)
    kin = kinematics(m, c.qpos, mp[:, :3], mp[:, 3:])
    mode, biped_type = int(S[T.QS_MODE]), int(param(T.QI_PARAM_BIPED_TYPE))
    torso = I[T.QI_TORSO_BODY]
    feet = []
    for f in range(4):
        g = I[T.QI_FOOT_GEOM + f]; b = m.geom_bodyid[g]
        feet.append(kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g])
    feet = np.array(feet)                                              # FL, HL, FR, HR
    avg = (0.5 * (feet[0] + feet[2]) if biped_type else 0.5 * (feet[1] + feet[3])) if mode == 1 else feet.mean(0)
    sub = [b for b in range(m.nbody) if _in_subtree(m, b, torso)]
    mass = sum(m.body_mass[b] for b in sub)
    com = sum(m.body_mass[b] * kin["xipos"][b] for b in sub) / mass
    comvel = sum(m.body_mass[b] * body_jacobian(m, kin, b, kin["xipos"][b])[:3] @ c.qvel for b in sub) / mass
    xmat = kin["xmat"][torso]
    goal = mp[I[T.QI_GOAL_MOCAP], :3]
    mode_time = c.time - S[T.QS_MODE_START_TIME]
    r = np.zeros(m.task_num_residual)
    # upright
    if mode == 4:
        r[0:3] = _rotvec_diff(kin["xquat"][torso], flip_quat(S, mode_time, int(param(T.QI_PARAM_FLIP_DIR))))
    else:
        r[0] = xmat[2, 0] - (-1 if biped_type else 1) if mode == 1 else xmat[2, 2] - 1
    # height
    hgoal = 0.6 if mode == 1 else 0.25
    torso_z = kin["xipos"][torso][2]
    r[3] = 0.0 if mode == 3 else torso_z - flip_height(S, mode_time) if mode == 4 else torso_z - avg[2] - hgoal
    # position
    s = I[T.QI_HEAD_SITE]
    head = kin["xpos"][m.site_bodyid[s]] + kin["xmat"][m.site_bodyid[s]] @ m.site_pos[s]
    target = goal.copy()
    if mode == 2:
        heading, position = S[T.QS_HEADING:T.QS_HEADING + 2], S[T.QS_POSITION:T.QS_POSITION + 3]
        if abs(S[T.QS_ANGVEL]) < 0.01:
            n = np.linalg.norm(heading)
            fw = heading / n if n >= 1e-15 else np.array([1.0, 0])
            target[:2] = position[:2] + heading + mode_time * S[T.QS_SPEED] * fw
        else:
            a = mode_time * S[T.QS_ANGVEL]
            target[:2] = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]) @ heading + position[:2]
    r[4], r[5] = head[0] - target[0], head[1] - target[1]
    r[6] = 2 * (head[2] - target[2]) if mode == 3 else 0.0
    # gait
    warning = False
    phase = S[T.QS_PHASE_START] + (c.time - S[T.QS_PHASE_START_TIME]) * S[T.QS_PHASE_VELOCITY]
    gait = 2 if mode == 1 else int(S[T.QS_GAIT])
    for f in range(4):
        if mode == 1 and ((not biped_type and f in (0, 2)) or (biped_type and f in (1, 3))):
            continue
        step = param(T.QI_PARAM_AMPLITUDE) * RS.step_height64(phase, 2 * math.pi * GAIT_PHASE[gait][f],
                                                              param(T.QI_PARAM_DUTY))
        query = feet[f].copy()
        if mode == 3:
            tg = goal - feet[f]; tg[2] = 0
            n = np.linalg.norm(tg)
            query += 0.15 * (tg / n if n >= 1e-15 else np.array([1.0, 0, 0]))
        gh = ground_height(m, kin, mp[:, :3], mp[:, 3:], query + [0, 0, 0.5])
        if gh is None:
            warning, gh = True, 0.0
        hd = feet[f][2] - (gh + 0.02 + step)
        if mode == 3:
            hd = min(0.0, hd)
        r[7 + f] = hd if step else 0.0
    # balance
    fall = math.sqrt(2 * hgoal / 9.81)
    r[11:13] = com[:2] + comvel[:2] * fall - avg[:2]
    # effort: actuator force from gain and bias, control clamped to ctrlrange
    nu = m.nu
    for i in range(nu):
        u = c.ctrl[i]
        lo, hi = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)[i]
        u = min(max(u, lo), hi)
        j = np.atleast_2d(np.asarray(m.actuator_trnid).T).T[i, 0]
        gear = np.asarray(m.actuator_gear, float).reshape(nu, -1)[i, 0]
        length, vel = gear * c.qpos[m.jnt_qposadr[j]], gear * c.qvel[m.jnt_dofadr[j]]
        gp = np.asarray(m.actuator_gainprm, float).reshape(nu, -1)[i]
        bp = np.asarray(m.actuator_biasprm, float).reshape(nu, -1)[i]
        r[13 + i] = 2e-2 * (gp[0] * u + bp[0] + bp[1] * length + bp[2] * vel)
    # posture
    home = np.asarray(m.key_qpos, float)[I[T.QI_KEY_HOME]]
    post = c.qpos[7:] - home[7:]
    if mode == 4:
        if mode_time < S[T.QS_CROUCH_TIME]:
            post = c.qpos[7:] - np.asarray(m.key_qpos, float)[I[T.QI_KEY_CROUCH]][7:]
        elif mode_time < S[T.QS_JUMP_TIME] + S[T.QS_FLIGHT_TIME]:
            post = 0 * post
    post = post * np.tile([2.0, 1.0, 1.0], 4)
    if mode == 1:
        base = 6 if biped_type else 0
        post[base:base + 6] *= param(T.QI_PARAM_ARM_POSTURE)
    r[25:37] = post
    # yaw and angular momentum
    th = np.array([xmat[0, 0], xmat[1, 0]])
    if mode == 1:
        hs = 1 if biped_type else -1
        th = hs * np.array([xmat[0, 2], xmat[1, 2]])
    n = np.linalg.norm(th)
    th = th / n if n >= 1e-15 else np.array([1.0, 0])
    hg = param(T.QI_PARAM_HEADING)
    r[37], r[38] = th[0] - math.cos(hg), th[1] - math.sin(hg)
    r[39:42] = comvel
    return r, warning


def _in_subtree(m, b, root):
    while b > 0:
        if b == root:
            return True
        b = m.body_parentid[b]
    return False


# ---------------------------------------------------------------------------------------------- tests
def _cases():
    out = []
    for c in RS.quadruped_cases():
        out += [c, RS.shifted(c, 1e2)]
    return out


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c.name)
def test_quadruped_residual_against_numpy(case, oracles):
    o = oracles(case.model_name)
    r64, warn = oracle_residual(o, case)
    mine, mine_warn = quadruped_residual(case)
    assert bool(warn) == mine_warn == ("warning" in case.flags)
    err = np.abs(r64 - mine)
    if "discontinuous" in case.flags:
        # on the threshold the two double evaluations may fall either side: row by row, one side must agree
        for side in case.side_cases():
            err = np.minimum(err, np.abs(r64 - quadruped_residual(side)[0]))
            err = np.minimum(err, np.abs(oracle_residual(o, side)[0] - mine))
    assert err.max() < 1e-9, (case.name, int(err.argmax()), err.max())


def test_terrain_cases_stand_on_their_terrain():
    """Each terrain case's feet find the surface it is named for, at the closed-form heights (so that the gait rows of
    the comparison above measure that surface's ray-cast)."""
    from mujoco_mpc_b200 import task as T
    from mujoco_mpc_b200.refmath import kinematics
    cases = {c.name: c for c in RS.quadruped_cases()}
    m = RS.model("quadruped")
    ramp = list(m.geom_names).index("ramp")
    Rr = _quat2mat(m.geom_quat[ramp]); cr = m.geom_pos[ramp]
    for name, expect in (("ramp", "ramp"), ("ramp_tilted_body", "ramp"), ("hill_top", "hill"), ("hill_slope", "hill"),
                         ("box_top", "box"), ("box_moved_rotated", "box"), ("quadruped", "floor")):
        c = cases[name]
        mp = c.mocap.reshape(-1, 7)
        kin = kinematics(m, c.qpos, mp[:, :3], mp[:, 3:])
        for f in range(4):
            g = m.task_ids[T.QI_FOOT_GEOM + f]; b = m.geom_bodyid[g]
            p = kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g]
            h = ground_height(m, kin, mp[:, :3], mp[:, 3:], p + [0, 0, 0.5])
            if expect == "floor":
                assert abs(h + 0.01) < 1e-12
            elif expect == "hill":
                d2 = (p[0] - 6) ** 2 + (p[1] - 6) ** 2
                assert abs(h - (-5.5 + math.sqrt(36 - d2))) < 1e-12 and h > 0
            elif expect == "ramp":
                # the top face: n . (x - c) = 0.5 with n the ramp's local z axis
                n = Rr[:, 2]
                assert abs(n @ (np.array([p[0], p[1], h]) - cr) - 0.5) < 1e-12 and h > 0
            else:
                assert h > 0.05 and abs(h - p[2]) < 0.1, (name, f, h, p)
    # foot 0 beside the ball: its cap height 1e-3 r inside the tangent, the floor 1e-3 r outside; the other feet on the floor
    for tag in ("inside", "outside"):
        c = cases["ball_near_tangent_" + tag]
        mb, mp = c.m, c.mocap.reshape(-1, 7)
        kin = kinematics(mb, c.qpos, mp[:, :3], mp[:, 3:])
        for f in range(4):
            g = mb.task_ids[T.QI_FOOT_GEOM + f]; b = mb.geom_bodyid[g]
            p = kin["xpos"][b] + kin["xmat"][b] @ mb.geom_pos[g]
            h = ground_height(mb, kin, mp[:, :3], mp[:, 3:], p + [0, 0, 0.5])
            d = math.hypot(p[0] - RS.BALL_CENTER[0], p[1] - RS.BALL_CENTER[1])
            if f == 0 and tag == "inside":
                assert abs(d / RS.BALL_RADIUS - (1 - 1e-3)) < 1e-9
                assert abs(h - (RS.BALL_CENTER[2] + math.sqrt(RS.BALL_RADIUS ** 2 - d * d))) < 1e-12 and h > 0.1
            else:
                assert d > RS.BALL_RADIUS and abs(h + 0.01) < 1e-12, (tag, f, d, h)


def test_flip_trajectory_closed_forms(oracles):
    """The designed Flip trajectory (QuadrupedFlat::ResetLocked): height and angle continuous at every segment
    boundary, the leap height 0.5 and angle pi / 2 at `jump`, 0.25 plus the ground after landing and 2 pi at the end;
    with the torso placed exactly on it, the upright and height rows are zero."""
    from mujoco_mpc_b200 import task as T
    S = np.asarray(RS.model("quadruped").task_state, float).copy()
    S[T.QS_GROUND] = 0.03
    jump, flight, land, crouch = S[T.QS_JUMP_TIME], S[T.QS_FLIGHT_TIME], S[T.QS_LAND_TIME], S[T.QS_CROUCH_TIME]
    eps = 1e-9
    for b in (jump, jump + flight, jump + flight + land):
        assert abs(flip_height(S, b - eps) - flip_height(S, b)) < 1e-7, b
        assert abs(flip_angle(S, b - eps) - flip_angle(S, b)) < 1e-7, b
    assert abs(flip_angle(S, crouch - eps) - flip_angle(S, crouch)) < 1e-7
    assert abs(flip_height(S, jump) - (0.5 + S[T.QS_GROUND])) < 1e-12
    assert abs(flip_angle(S, jump) - math.pi / 2) < 1e-12
    assert abs(flip_height(S, jump + flight + land) - (0.25 + S[T.QS_GROUND])) < 1e-12
    assert abs(flip_angle(S, jump + flight + land - eps) - 2 * math.pi) < 1e-7
    # the torso on the trajectory: upright and height rows vanish
    c0 = next(c for c in RS.quadruped_cases() if c.name == "flip_dir1")
    m = c0.m
    o = oracles("quadruped")
    torso = m.task_ids[T.QI_TORSO_BODY]
    S[T.QS_MODE] = 4
    S[T.QS_ORIENTATION:T.QS_ORIENTATION + 4] = RS.quat_about((0, 0, 1), 0.4)
    ms = 0.2
    for t in np.linspace(0, jump + flight + land + 0.1, 23):
        for fd in (0, 1):
            q = c0.qpos.copy()
            quat = flip_quat(S, t, fd)
            q[3:7] = quat
            q[0:3] = [0.1, 0.0, flip_height(S, t) - (_quat2mat(quat) @ m.body_ipos[torso])[2]]
            prm = c0.parameters.copy(); prm[m.task_ids[T.QI_PARAM_FLIP_DIR]] = fd
            c = c0.replace(qpos=q, time=ms + t, task_state=np.r_[S[:1], ms, S[2:]], parameters=prm)
            r, _ = oracle_residual(o, c)
            assert np.abs(r[0:4]).max() < 1e-9, (t, fd, r[0:4])
