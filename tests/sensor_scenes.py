"""Purpose-built scenes for the frame, subtree, ball-joint, actuator and tendon sensors, the shipped models with those
sensors added (copies made here, the shipped models stay as they are), and an independent numpy restatement of the
sensors on the kinematics of mujoco_mpc_b200.refmath.  Shared by tests/test_sensors_cpu.py and tests/test_gpu_sensors.py.

The restatement (sensors_np) forms velocities from world-frame Jacobians times qvel (refmath.body_jacobian), the
subtree quantities from per-body sums, and frame rotations from quaternion products: a formulation independent of the
sensor oracle's com-based motion vectors and of the kernels'.
"""
import numpy as np

from mujoco_mpc_b200 import models
from mujoco_mpc_b200.mjcf import (JNT_BALL, OBJ_BODY, OBJ_GEOM, OBJ_SITE, OBJ_XBODY, SENS_ACTUATORFRC,
                                  SENS_ACTUATORPOS, SENS_ACTUATORVEL, SENS_BALLANGVEL, SENS_BALLQUAT, SENS_FRAMEANGVEL,
                                  SENS_FRAMELINVEL, SENS_FRAMEPOS, SENS_FRAMEQUAT, SENS_FRAMEXAXIS, SENS_FRAMEYAXIS,
                                  SENS_FRAMEZAXIS, SENS_JOINTACTUATORFRC, SENS_JOINTPOS, SENS_JOINTVEL, SENS_SUBTREEANGMOM, SENS_SUBTREECOM,
                                  SENS_SUBTREELINVEL, SENS_TENDONPOS, SENS_TENDONVEL, compile_xml, quat2mat, quat_mul)
from mujoco_mpc_b200.refmath import body_jacobian, kinematics

# world rotations the scenes are built in: (w, x, y, z), not normalised
ROTATIONS = ((1, 0, 0, 0), (0.7071068, 0, 0, 0.7071068), (0.5, 0.5, -0.5, 0.5), (0.9, 0.3, -0.2, 0.25))


def _rot(quat):
    q = np.asarray(quat, float)
    return q / np.linalg.norm(q)


def _fmt(v):
    return " ".join("%.10g" % x for x in v)


def _world(quat, pos, local_quat=(1, 0, 0, 0)):
    """gravity, the rotated position of pos and the rotated orientation local_quat, for a scene rotated by quat"""
    q = _rot(quat)
    R = quat2mat(q)
    return _fmt(R @ np.array([0, 0, -9.81])), _fmt(R @ np.asarray(pos, float)), _fmt(quat_mul(q, _rot(local_quat)))


def free_body_xml(rot=ROTATIONS[0], timestep=0.002):
    """(a) A free-floating asymmetric body: off-centre sites with their own orientation, a geom with its own quat, an
    inertial frame rotated against the body frame.  Sensors 0-3 are an IMU (framepos, framequat, gyro, accelerometer
    of one site), the sensor kinds of the reference's quadrotor."""
    g, p, q = _world(rot, (0.1, -0.2, 0.5), (0.96, 0.1, -0.2, 0.15))
    return f"""
<mujoco model="free body">
  <option timestep="{timestep}" gravity="{g}"><flag contact="disable"/></option>
  <worldbody>
    <body name="body" pos="{p}" quat="{q}">
      <freejoint name="free"/>
      <inertial pos="0.02 -0.01 0.03" quat="0.9 0.2 -0.3 0.1" mass="1.3" diaginertia="0.02 0.035 0.05"/>
      <geom name="shell" type="box" size="0.06 0.04 0.02" pos="0.01 0.02 -0.01" quat="0.8 0.1 0.5 -0.2" mass="0"/>
      <site name="imu" pos="0.05 -0.03 0.02" quat="0.7 0.3 -0.2 0.6"/>
      <site name="corner" pos="-0.04 0.06 -0.01"/>
    </body>
  </worldbody>
  <sensor>
    <framepos name="imu_pos" objtype="site" objname="imu"/>
    <framequat name="imu_quat" objtype="site" objname="imu"/>
    <gyro name="imu_gyro" site="imu"/>
    <accelerometer name="imu_acc" site="imu"/>
    <framequat objtype="body" objname="body"/><framequat objtype="xbody" objname="body"/>
    <framequat objtype="geom" objname="shell"/>
    <framexaxis objtype="site" objname="imu"/><frameyaxis objtype="body" objname="body"/>
    <framezaxis objtype="geom" objname="shell"/><framexaxis objtype="xbody" objname="body"/>
    <framelinvel objtype="site" objname="corner"/><framelinvel objtype="body" objname="body"/>
    <frameangvel objtype="geom" objname="shell"/><frameangvel objtype="xbody" objname="body"/>
    <framelinacc objtype="site" objname="imu"/><framelinacc objtype="xbody" objname="body"/>
    <framelinacc objtype="geom" objname="shell"/><framelinacc objtype="body" objname="body"/>
    <frameangacc objtype="body" objname="body"/>
    <subtreecom body="body"/><subtreelinvel body="body"/><subtreeangmom body="body"/>
  </sensor>
</mujoco>"""


def ball_chain_xml(rot=ROTATIONS[0], timestep=0.002):
    """(b) A free base carrying a ball joint and two hinges."""
    g, p, q = _world(rot, (0, 0, 1), (0.95, 0.05, 0.2, -0.1))
    return f"""
<mujoco model="ball chain">
  <option timestep="{timestep}" gravity="{g}"><flag contact="disable"/></option>
  <worldbody>
    <body name="base" pos="{p}" quat="{q}">
      <freejoint/>
      <geom name="base" type="box" size="0.1 0.05 0.03" mass="2"/>
      <body name="arm" pos="0.1 0 0">
        <joint name="ball" type="ball" damping="0.02"/>
        <geom name="arm" type="capsule" fromto="0 0 0 0.2 0 0" size="0.02" mass="0.5"/>
        <body name="fore" pos="0.2 0 0">
          <joint name="h1" type="hinge" axis="0 1 0" damping="0.01"/>
          <geom name="fore" type="capsule" fromto="0 0 0 0 0 -0.15" size="0.015" mass="0.3"/>
          <body name="hand" pos="0 0 -0.15">
            <joint name="h2" type="hinge" axis="1 0 0.3" damping="0.01"/>
            <geom name="hand" type="sphere" size="0.03" pos="0.01 0 0" mass="0.1"/>
            <site name="tip" pos="0 0.02 -0.01" quat="0.8 0 0.6 0"/>
          </body>
        </body>
      </body>
    </body>
  </worldbody>
  <sensor>
    <ballquat joint="ball"/><ballangvel joint="ball"/>
    <subtreecom body="base"/><subtreelinvel body="base"/><subtreeangmom body="base"/>
    <subtreeangmom body="arm"/><subtreecom body="fore"/>
    <framelinacc objtype="site" objname="tip"/><frameangacc objtype="body" objname="hand"/>
    <framequat objtype="body" objname="fore"/><frameangvel objtype="xbody" objname="hand"/>
    <framelinvel objtype="geom" objname="hand"/><framezaxis objtype="site" objname="tip"/>
    <jointpos joint="h1"/><jointvel joint="h2"/>
  </sensor>
</mujoco>"""


def tendon_pair_xml(rot=ROTATIONS[0], timestep=0.002):
    """(c) Two hinges coupled by a fixed tendon with a tendon-transmission position actuator, and a slide driven only
    by a motor with gear 2.5 whose force limit binds for |ctrl| > 0.4."""
    g, p, q = _world(rot, (0, 0, 0.5))
    return f"""
<mujoco model="tendon pair">
  <option timestep="{timestep}" gravity="{g}"><flag contact="disable"/></option>
  <worldbody>
    <body name="base" pos="{p}" quat="{q}">
      <body name="l1">
        <joint name="j1" type="hinge" axis="0 1 0" damping="0.1"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.02" mass="0.4"/>
        <body name="l2" pos="0.2 0 0">
          <joint name="j2" type="hinge" axis="0 1 0" damping="0.1"/>
          <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.02" mass="0.2"/>
          <site name="tip" pos="0.2 0 0"/>
        </body>
      </body>
      <body name="cart" pos="0 0.3 0">
        <joint name="j3" type="slide" axis="1 0 0" damping="0.5"/>
        <geom type="sphere" size="0.03" mass="0.3"/>
      </body>
    </body>
  </worldbody>
  <tendon>
    <fixed name="couple"><joint joint="j1" coef="0.7"/><joint joint="j2" coef="-0.4"/></fixed>
  </tendon>
  <actuator>
    <position name="tpos" tendon="couple" kp="3" ctrllimited="true" ctrlrange="-1 1"/>
    <motor name="m3" joint="j3" gear="2.5" ctrllimited="true" ctrlrange="-1 1" forcelimited="true"
           forcerange="-0.4 0.4"/>
  </actuator>
  <sensor>
    <actuatorpos actuator="tpos"/><actuatorvel actuator="tpos"/><actuatorpos actuator="m3"/>
    <actuatorvel actuator="m3"/><actuatorfrc actuator="tpos"/><actuatorfrc actuator="m3"/>
    <jointactuatorfrc joint="j3"/><jointactuatorfrc joint="j1"/>
    <tendonpos tendon="couple"/><tendonvel tendon="couple"/>
    <framepos objtype="site" objname="tip"/><jointpos joint="j1"/><jointpos joint="j2"/><jointpos joint="j3"/>
  </sensor>
</mujoco>"""


def imu_body(rot=ROTATIONS[0], timestep=0.005):
    """scene (a) as a filtering model: the estimators measure its IMU (sensors 0-3) at the given timestep"""
    custom = """<custom><numeric name="estimator_sensor_start" data="0"/><numeric name="estimator_number_sensor" data="4"/>
  <numeric name="estimator_timestep" data="%g"/></custom>""" % timestep
    return compile_xml(free_body_xml(rot, timestep).replace("<worldbody>", custom + "\n  <worldbody>", 1))


def imu_plant(m, T=120):
    """An fp64 oracle flight of the IMU body (imu_body) from a seeded state at its estimator timestep: states
    [T + 1][nq + nv], the IMU readings of each with seeded Gaussian noise of std 1e-3, and the (zero) controls"""
    from estimator_backends import simulate
    x0 = random_states(m, 1, seed=8, scale=0.1)[0]
    x0[m.nq:] *= 0.5
    return simulate(m, x0[:m.nq], x0[m.nq:], T + 1, timestep=0.005, start=0, count=4, noise=1e-3, seed=9)


SCENES = {"free_body": free_body_xml, "ball_chain": ball_chain_xml, "tendon_pair": tendon_pair_xml}


def scene(name, rot=ROTATIONS[0], timestep=0.002):
    return compile_xml(SCENES[name](rot, timestep))


# ------------------------------------------------------------------------------------- shipped models, augmented
QUADRUPED_SENSORS = """
    <framequat objtype="body" objname="trunk"/><framequat objtype="site" objname="head"/>
    <framelinvel objtype="site" objname="head"/><frameangvel objtype="xbody" objname="trunk"/>
    <framelinacc objtype="site" objname="FR"/><frameangacc objtype="body" objname="trunk"/>
    <framexaxis objtype="geom" objname="FR"/><framezaxis objtype="xbody" objname="trunk"/>
    <subtreeangmom body="trunk"/><subtreeangmom body="FR_thigh"/><subtreecom body="RL_calf"/>
    <actuatorpos actuator="FR_hip"/><actuatorvel actuator="FR_thigh"/><actuatorfrc actuator="RL_calf"/>
    <jointactuatorfrc joint="FR_calf_joint"/>
"""
HUMANOID_SENSORS = """
    <framequat objtype="body" objname="torso"/><framelinvel objtype="site" objname="tracking[head]"/>
    <frameangvel objtype="body" objname="pelvis"/><framelinacc objtype="site" objname="foot_right"/>
    <frameangacc objtype="xbody" objname="shin_left"/><frameyaxis objtype="geom" objname="foot1_left"/>
    <subtreeangmom body="torso"/><subtreelinvel body="thigh_left"/>
    <tendonpos tendon="hamstring_right"/><tendonvel tendon="hamstring_left"/>
    <actuatorpos actuator="knee_right"/><actuatorvel actuator="hip_y_left"/><actuatorfrc actuator="elbow_left"/>
    <jointactuatorfrc joint="knee_left"/>
"""
HAND_SENSORS = """
    <framelinvel objtype="body" objname="cube"/><frameangvel objtype="body" objname="cube"/>
    <framelinacc objtype="body" objname="cube"/><frameangacc objtype="geom" objname="cube"/>
    <framexaxis objtype="xbody" objname="cube"/><ballquat joint="goal_ball"/><ballangvel joint="goal_ball"/>
    <actuatorpos actuator="rh_A_FFJ0"/><actuatorvel actuator="rh_A_FFJ0"/><actuatorpos actuator="rh_A_THJ1"/>
    <tendonpos tendon="rh_LFJ0"/><tendonvel tendon="rh_MFJ0"/><actuatorfrc actuator="rh_A_WRJ1"/>
    <jointactuatorfrc joint="rh_THJ2"/><subtreeangmom body="rh_palm"/>
"""
HAND_FILTER_SENSORS = """
    <framepos name="f_cube_pos" objtype="body" objname="cube"/><framequat name="f_cube_quat" objtype="body" objname="cube"/>
    <framelinvel name="f_cube_linvel" objtype="body" objname="cube"/>
    <frameangvel name="f_cube_angvel" objtype="body" objname="cube"/>
""" + "".join('<jointpos joint="rh_%s"/>' % j for j in (
    "WRJ2", "WRJ1", "FFJ4", "FFJ3", "FFJ2", "FFJ1", "MFJ4", "MFJ3", "MFJ2", "MFJ1", "RFJ4", "RFJ3", "RFJ2", "RFJ1",
    "LFJ5", "LFJ4", "LFJ3", "LFJ2", "LFJ1", "THJ5", "THJ4", "THJ3", "THJ2", "THJ1"))
AUGMENTED = {"quadruped": ("quadruped_flat_xml", QUADRUPED_SENSORS), "humanoid_track": ("humanoid_track_xml", HUMANOID_SENSORS),
             "shadow_reorient": ("shadow_reorient_xml", HAND_SENSORS)}


def load_augmented(name, monkeypatch, extra=None, **kw):
    """models.load(name) with sensors appended to a copy of its MJCF; returns (model, index of the first added
    sensor, number added).  The shipped XML function is replaced for the duration of the test only."""
    fn, sensors = AUGMENTED[name]
    sensors = sensors if extra is None else extra
    orig = getattr(models, fn)

    def patched(*a, **k):
        x = orig(*a, **k).replace('<joint type="ball" damping="0.01"/>', '<joint name="goal_ball" type="ball" damping="0.01"/>')
        i = x.rindex("</sensor>")
        return x[:i] + sensors + x[i:]
    base = models.load(name, **kw)
    monkeypatch.setattr(models, fn, patched)
    m = models.load(name, **kw)
    monkeypatch.setattr(models, fn, orig)
    return m, base.nsensor, m.nsensor - base.nsensor


# ------------------------------------------------------------------------------------------ numpy restatement
def _frame(m, kin, ot, oid):
    """position, quaternion and body of a frame sensor's object"""
    if ot == OBJ_SITE:
        b = m.site_bodyid[oid]
        return kin["xpos"][b] + kin["xmat"][b] @ m.site_pos[oid], quat_mul(kin["xquat"][b], m.site_quat[oid]), b
    if ot == OBJ_GEOM:
        b = m.geom_bodyid[oid]
        return kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[oid], quat_mul(kin["xquat"][b], m.geom_quat[oid]), b
    if ot == OBJ_XBODY:
        return kin["xpos"][oid], kin["xquat"][oid], oid
    assert ot == OBJ_BODY
    return kin["xipos"][oid], quat_mul(kin["xquat"][oid], m.body_iquat[oid]), oid


def _subtree(m, body):
    out = []
    for j in range(body, m.nbody):
        k = j
        while k > body:
            k = m.body_parentid[k]
        if k == body:
            out.append(j)
    return out


def sensors_np(m, qpos, qvel, start, n, actuator_force=None, qfrc_actuator=None):
    """Sensors [start, start + n) of one state in fp64 without acceleration: every type of this module's scenes except
    framelinacc / frameangacc / accelerometer / gyro (checked against physical laws instead).  actuatorfrc and
    jointactuatorfrc read the given actuator_force / qfrc_actuator."""
    qpos, qvel = np.asarray(qpos, float), np.asarray(qvel, float)
    kin = kinematics(m, qpos)
    out = []

    def vel(b, point):
        J = body_jacobian(m, kin, b, point)
        return J[0:3] @ qvel, J[3:6] @ qvel

    def tendon(t, v):
        a, e = m.tendon_adr[t], m.tendon_adr[t] + m.tendon_num[t]
        return sum(m.wrap_coef[w] * (qvel[m.wrap_dof[w]] if v else qpos[m.wrap_qposadr[w]]) for w in range(a, e))

    for i in range(start, start + n):
        t, ot, oid = int(m.sensor_type[i]), int(m.sensor_objtype[i]), int(m.sensor_objid[i])
        if t == SENS_JOINTPOS:
            out.append([qpos[m.jnt_qposadr[oid]]])
        elif t == SENS_JOINTVEL:
            out.append([qvel[m.jnt_dofadr[oid]]])
        elif t in (SENS_FRAMEPOS, SENS_FRAMEQUAT, SENS_FRAMEXAXIS, SENS_FRAMEYAXIS, SENS_FRAMEZAXIS, SENS_FRAMELINVEL,
                   SENS_FRAMEANGVEL):
            p, q, b = _frame(m, kin, ot, oid)
            if t == SENS_FRAMEPOS:
                out.append(p)
            elif t == SENS_FRAMEQUAT:
                out.append(q)
            elif t in (SENS_FRAMEXAXIS, SENS_FRAMEYAXIS, SENS_FRAMEZAXIS):
                out.append(quat2mat(q / np.linalg.norm(q))[:, t - SENS_FRAMEXAXIS])
            else:
                lin, ang = vel(b, p)
                out.append(lin if t == SENS_FRAMELINVEL else ang)
        elif t in (SENS_SUBTREECOM, SENS_SUBTREELINVEL, SENS_SUBTREEANGMOM):
            js = _subtree(m, oid)
            mass = np.array([m.body_mass[j] for j in js])
            com = sum(mass[k] * kin["xipos"][j] for k, j in enumerate(js)) / mass.sum()
            v = [vel(j, kin["xipos"][j]) for j in js]
            vcom = sum(mass[k] * v[k][0] for k in range(len(js))) / mass.sum()
            if t == SENS_SUBTREECOM:
                out.append(com)
            elif t == SENS_SUBTREELINVEL:
                out.append(vcom)
            else:
                L = np.zeros(3)
                for k, j in enumerate(js):
                    R = kin["ximat"][j]
                    L += R @ np.diag(m.body_inertia[j]) @ R.T @ v[k][1]
                    L += np.cross(kin["xipos"][j] - com, mass[k] * (v[k][0] - vcom))
                out.append(L)
        elif t == SENS_BALLQUAT:
            assert m.jnt_type[oid] == JNT_BALL
            a = m.jnt_qposadr[oid]
            out.append(qpos[a:a + 4] / np.linalg.norm(qpos[a:a + 4]))
        elif t == SENS_BALLANGVEL:
            out.append(qvel[m.jnt_dofadr[oid]:m.jnt_dofadr[oid] + 3])
        elif t in (SENS_ACTUATORPOS, SENS_ACTUATORVEL):
            v = t == SENS_ACTUATORVEL
            j = m.actuator_trnid[oid]
            x = tendon(j, v) if m.actuator_trntype[oid] == 1 else (qvel[m.jnt_dofadr[j]] if v else qpos[m.jnt_qposadr[j]])
            out.append([m.actuator_gear[oid] * x])
        elif t in (SENS_TENDONPOS, SENS_TENDONVEL):
            out.append([tendon(oid, t == SENS_TENDONVEL)])
        elif t == SENS_ACTUATORFRC:
            out.append([actuator_force[oid]])
        elif t == SENS_JOINTACTUATORFRC:
            out.append([qfrc_actuator[m.jnt_dofadr[oid]]])
        else:
            raise NotImplementedError("sensor %d (type %d) is not restated here" % (i, t))
    return np.concatenate([np.asarray(o, float) for o in out]) if out else np.zeros(0)


def random_states(m, k, seed=0, scale=0.3):
    """k states near qpos0 with normalised free / ball quaternions and random velocities"""
    rng = np.random.default_rng(seed)
    X = np.array([np.concatenate([m.qpos0 + scale * rng.normal(size=m.nq), rng.normal(size=m.nv)]) for _ in range(k)])
    for j in range(m.njnt):
        a = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == 0 else 0)
        if m.jnt_type[j] in (0, JNT_BALL):
            X[:, a:a + 4] /= np.linalg.norm(X[:, a:a + 4], axis=1)[:, None]
    return X
