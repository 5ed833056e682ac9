"""The CPU oracle as a sigma-point backend of mujoco_mpc_b200.estimator.Unscented, and the reference's estimator test
scenes (mjpc/test/estimator/unscented_test.cc).  Shared by tests/test_estimator_cpu.py and tests/test_gpu_estimator.py.

The oracle backend steps the sigma points and evaluates their sensors, touch included, on the CPU oracle through
sensor_oracle (fp64, or fp32 as the yardstick of device bars).  sensors_fp64 restates jointpos / jointvel / framepos in
numpy on the kinematics of mujoco_mpc_b200.refmath (a formulation independent of the oracle's and the kernels'), to
cross-check the sensor oracle.
"""
import os

import numpy as np

from mujoco_mpc_b200.blob import to_blob
from mujoco_mpc_b200.mjcf import (OBJ_BODY, OBJ_GEOM, OBJ_SITE, OBJ_XBODY, SENS_FRAMEPOS, SENS_JOINTPOS,
                                  SENS_JOINTVEL, compile_xml, quat2mat)
from mujoco_mpc_b200.refmath import kinematics

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_estimator_model(name):
    """The reference's estimator test models, verbatim fixtures: "particle1d" (task1D.xml), "box3drot" (task3Drot.xml)."""
    f = {"particle1d": "estimator_particle_task1D.xml", "box3drot": "estimator_box_task3Drot.xml"}[name]
    return compile_xml(path=os.path.join(GOLDEN, f))


def mocap_vector(m, mocap_pos=None, mocap_quat=None):
    if m.nmocap == 0:
        return np.zeros(0)
    p = m.mocap_pos0 if mocap_pos is None else mocap_pos
    q = m.mocap_quat0 if mocap_quat is None else mocap_quat
    return np.concatenate([np.concatenate([p[i], q[i]]) for i in range(m.nmocap)])


def sensors_fp64(m, qpos, qvel, start, n, mocap=None):
    """jointpos / jointvel / framepos sensors [start, start + n) of one state, fp64."""
    mp = mq = None
    if m.nmocap and mocap is not None:
        mc = np.asarray(mocap, float).reshape(m.nmocap, 7)
        mp, mq = mc[:, :3], mc[:, 3:]
    kin = None
    out = []
    for i in range(start, start + n):
        t, ot, oid = int(m.sensor_type[i]), int(m.sensor_objtype[i]), int(m.sensor_objid[i])
        if t == SENS_JOINTPOS:
            out.append([qpos[m.jnt_qposadr[oid]]])
        elif t == SENS_JOINTVEL:
            out.append([qvel[m.jnt_dofadr[oid]]])
        elif t == SENS_FRAMEPOS:
            if kin is None:
                kin = kinematics(m, qpos, mp, mq)
            if ot == OBJ_SITE:
                b = m.site_bodyid[oid]
                out.append(kin["xpos"][b] + kin["xmat"][b] @ m.site_pos[oid])
            elif ot == OBJ_GEOM:
                b = m.geom_bodyid[oid]
                out.append(kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[oid])
            elif ot == OBJ_XBODY:
                out.append(kin["xpos"][oid])
            else:
                assert ot == OBJ_BODY
                out.append(kin["xipos"][oid])
        else:
            raise NotImplementedError("sensor %d: the oracle backend evaluates jointpos, jointvel and framepos" % i)
    return np.concatenate(out) if out else np.zeros(0)


def sensor_oracle(m, timestep=None, precision=64):
    import sensor_oracle as so
    so.build()
    mm = type(m)(m)
    if timestep is not None:
        mm["opt_timestep"] = float(timestep)
    return so.SensorOracle(to_blob(mm), mm, precision)


class OracleSigmaBackend:
    """The sigma points stepped by the CPU oracle with their measurement sensors (sensor_oracle)."""

    def __init__(self, m, sensor_start, nsensor, timestep, precision=64, nthreads=None):
        self.m = m
        self.o = sensor_oracle(m, timestep, precision)
        self.start, self.n = sensor_start, nsensor

    def step_sensors(self, states, ctrl, mocap, time, warmstart):
        m = self.m
        x = np.asarray(states, float)
        B, nq = x.shape[0], m.nq
        r = self.o.step(x[:, :nq], x[:, nq:], np.tile(ctrl, (B, 1)), mocap, np.full(B, time), self.start, self.n,
                        warmstart=warmstart)
        nxt = np.concatenate([r["next_qpos"], r["next_qvel"]], axis=1)
        return nxt, r["sensordata"], r["qacc"], int(np.count_nonzero(r["warning"]))


def simulate(m, qpos0, qvel0, T, timestep=None, ctrl=None, precision=64, start=0, count=None, noise=0.0, seed=0):
    """The reference's test Simulation (test/simulation.cc:55-70) on the oracle: states [T][nq+nv], the sensors
    [start, start + count) of each state before its step [T][dim] (plus seeded Gaussian noise of std `noise`) and the
    controls [T][nu]; ctrl is None (zeros), an array [nu] or a function (t, state) -> ctrl.  The warm start carries over
    from step to step as in one mjData."""
    o = sensor_oracle(m, timestep, precision)
    h = m.opt_timestep if timestep is None else timestep
    count = m.nsensor - start if count is None else count
    rng = np.random.default_rng(seed)
    mc = mocap_vector(m)
    q, v = np.array(qpos0, float), np.array(qvel0, float)
    warm = np.zeros(m.nv)
    X, Y, U = [], [], []
    for t in range(T):
        x = np.concatenate([q, v])
        u = np.zeros(m.nu) if ctrl is None else (ctrl(t, x) if callable(ctrl) else np.asarray(ctrl, float))
        r = o.step(q[None], v[None], u[None], mc, np.array([t * h]), start, count, warmstart=warm[None])
        X.append(x); U.append(u)
        Y.append(r["sensordata"][0] + (noise * rng.normal(size=r["sensordata"].shape[1]) if noise else 0.0))
        q, v, warm = r["next_qpos"][0], r["next_qvel"][0], r["qacc"][0]
    return np.array(X), np.array(Y), np.array(U)


def quat_error(m, qa, qb):
    """mju_subQuat of a ball-joint model's single quaternion (the Box3Drot test's position error)."""
    from mujoco_mpc_b200.estimator import quat_sub
    return quat_sub(qa[:4], qb[:4])


def box_corner_closed_form(m, qpos):
    """Site positions of the Box3Drot corners: body at (0, 0, 0.25) rotated by the ball quaternion."""
    R = quat2mat(np.asarray(qpos[:4]) / np.linalg.norm(qpos[:4]))
    return np.concatenate([np.array([0, 0, 0.25]) + R @ m.site_pos[s] for s in range(m.nsite)])


# purpose-built scenes: every framepos object type (offset geom, inertial and site frames on a hinged body), and a ball
# on a plane with touch zones that contain the contact point, are hit by the normal ray, are missed by it, belong to
# another body, and are not spheres
FRAMES_XML = """
<mujoco model="frames">
  <option><flag contact="disable"/></option>
  <worldbody>
    <body name="arm" pos="0.1 0.2 0.3" quat="0.9 0.1 0.3 0.2">
      <joint name="hinge" type="hinge" axis="0.3 1 0.2"/>
      <inertial pos="0.05 -0.02 0.01" mass="1" diaginertia="0.01 0.02 0.03"/>
      <geom name="link" type="capsule" size="0.02 0.1" pos="0.1 0.03 -0.02" quat="1 0 1 0" mass="0"/>
      <site name="tip" pos="0.2 0.01 0.04"/>
      <body name="forearm" pos="0.2 0 0">
        <joint name="slide" type="slide" axis="1 0 0.5"/>
        <inertial pos="0.03 0.01 0" mass="0.5" diaginertia="0.01 0.01 0.01"/>
      </body>
    </body>
  </worldbody>
  <sensor>
    <framepos objtype="site" objname="tip"/><framepos objtype="body" objname="arm"/>
    <framepos objtype="xbody" objname="arm"/><framepos objtype="geom" objname="link"/>
    <framepos objtype="body" objname="forearm"/><jointpos joint="hinge"/><jointvel joint="slide"/>
  </sensor>
</mujoco>"""

TOUCH_XML = """
<mujoco model="touch scene">
  <option timestep="0.002" cone="{cone}"/>
  <worldbody>
    <geom name="floor" type="plane" size="1 1 .1"/>
    <body name="other" mocap="true" pos="0.3 0 0.3">
      <site name="other" type="sphere" size="1"/>
    </body>
    <body name="ball" pos="0 0 0.05">
      <freejoint/>
      <geom name="ball" type="sphere" size="0.05" mass="1"/>
      <site name="inside" type="sphere" size="0.08"/>
      <site name="ray" type="sphere" size="0.01"/>
      <site name="miss" type="sphere" size="0.01" pos="0.03 0 0"/>
      <site name="boxzone" type="box" size="0.01 0.01 0.01"/>
    </body>
  </worldbody>
  <sensor>
    <touch site="inside"/><touch site="ray"/><touch site="miss"/><touch site="other"/><touch site="boxzone"/>
  </sensor>
</mujoco>"""


def settle(step, m, n, h, x=None):
    """n steps of step(x, warmstart, time) -> dict(next_qpos, next_qvel, qacc) from x (default qpos0, zero qvel);
    returns the final state and warm start."""
    x = np.concatenate([m.qpos0, np.zeros(m.nv)]) if x is None else np.array(x, float)
    w = np.zeros((1, m.nv))
    for t in range(n):
        r = step(x, w, t * h)
        x = np.concatenate([r["next_qpos"][0], r["next_qvel"][0]]).astype(float) if "next_qpos" in r else \
            r["next_states"][0].astype(float)
        w = r["qacc"]
    return x, w
