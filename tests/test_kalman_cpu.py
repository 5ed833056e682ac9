"""The IMU sensors (accelerometer, velocimeter, gyro) on the sensor oracle and the Kalman filter on the fp64 / fp32
oracle (no GPU).

The sensor oracle's IMU sensors are checked against an independent restatement on mujoco_mpc_b200.refmath kinematics:
from a random state (q0, v0) with the oracle's qacc, the path q(t) = q0 (+) (v0 t + 1/2 qacc t^2) moves every site with
the velocity J(q(t)) qdot(t) (body_jacobian), and the world acceleration of the site is that velocity differenced in
time.  gyro and velocimeter are the rotated velocities (bar 1e-12); the accelerometer is the differenced acceleration
minus gravity, rotated into the site frame, with the error of a centred difference at h = 1e-5, below 1e-7 here (bar 1e-6).

The filter test is the reference's own (mjpc/test/estimator/kalman_test.cc) on its verbatim task_imu model: qpos0 0.25,
T = 200, covariance and both noises 1e-5, noise-free measurements, epsilon 1e-6 one-sided; after update_measurement at
step t the qpos and qvel error norms against the simulation's state t are within 1e-4, ground impact included.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import OracleSigmaBackend, mocap_vector, sensor_oracle, simulate  # noqa: E402
from quadruped_filtering import plant, run_filter  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.estimator import (KALMAN_CENTERED, KALMAN_EPSILON, EstimatorError, Kalman,  # noqa: E402
                                       integrate_pos, measured_range)
from mujoco_mpc_b200.mjcf import (OBJ_SITE, SENS_ACCELEROMETER, SENS_GYRO, SENS_VELOCIMETER, compile_xml,  # noqa: E402
                                  quat2mat)
from mujoco_mpc_b200.refmath import body_jacobian, kinematics  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_task_imu():
    """The reference's Kalman test model (estimator/particle/task_imu.xml, verbatim): jointpos + accelerometer."""
    return compile_xml(path=os.path.join(GOLDEN, "estimator_particle_task_imu.xml"))


# purpose-built scenes without contacts: a hinge / slide / hinge chain with offset joints and rotated sites, and a free
# body carrying a hinged pendulum (the site's body is not its tree's root, so subtree_com[root] is not its own com)
IMU_CHAIN_XML = """
<mujoco model="imu chain">
  <option><flag contact="disable"/></option>
  <worldbody>
    <body name="arm" pos="0.1 0.2 0.3" quat="0.9 0.1 0.3 0.2">
      <joint name="hinge" type="hinge" axis="0.3 1 0.2" pos="0.01 -0.02 0.03" damping="0.05"/>
      <inertial pos="0.05 -0.02 0.01" mass="1" diaginertia="0.01 0.02 0.03"/>
      <site name="arm_imu" pos="0.2 0.01 0.04" quat="0.8 0.3 -0.2 0.4"/>
      <body name="forearm" pos="0.2 0 0" quat="0.7 0 0.7 0.1">
        <joint name="slide" type="slide" axis="1 0 0.5"/>
        <joint name="wrist" type="hinge" axis="0 0.6 0.8" pos="0.03 0 0"/>
        <inertial pos="0.03 0.01 0" mass="0.5" diaginertia="0.01 0.01 0.01"/>
        <site name="hand_imu" pos="0.1 -0.03 0.02" quat="0.5 0.5 -0.5 0.5"/>
      </body>
    </body>
  </worldbody>
  <sensor>
    <gyro site="arm_imu"/><velocimeter site="arm_imu"/><accelerometer site="arm_imu"/>
    <gyro site="hand_imu"/><velocimeter site="hand_imu"/><accelerometer site="hand_imu"/>
  </sensor>
</mujoco>"""

IMU_FREE_XML = """
<mujoco model="imu free body">
  <option><flag contact="disable"/></option>
  <worldbody>
    <body name="torso" pos="0 0 1">
      <freejoint/>
      <inertial pos="0.02 -0.01 0.03" mass="2" diaginertia="0.05 0.04 0.03"/>
      <site name="torso_imu" pos="0.05 0.1 -0.02" quat="0.7 0.1 0.7 0.1"/>
      <body name="pendulum" pos="0.1 0 -0.1">
        <joint name="swing" type="hinge" axis="0 1 0.3"/>
        <inertial pos="0 0 -0.15" mass="0.7" diaginertia="0.01 0.01 0.002"/>
        <site name="bob_imu" pos="0.02 0 -0.3" quat="0.9 -0.3 0.1 0.2"/>
      </body>
    </body>
  </worldbody>
  <sensor>
    <accelerometer site="torso_imu"/><gyro site="torso_imu"/><velocimeter site="torso_imu"/>
    <accelerometer site="bob_imu"/><gyro site="bob_imu"/><velocimeter site="bob_imu"/>
  </sensor>
</mujoco>"""


def test_imu_tags_parse_as_site_sensors():
    m = compile_xml(IMU_CHAIN_XML)
    assert list(m.sensor_type) == [SENS_GYRO, SENS_VELOCIMETER, SENS_ACCELEROMETER] * 2
    assert (SENS_ACCELEROMETER, SENS_VELOCIMETER, SENS_GYRO) == (10, 11, 12)
    assert list(m.sensor_objtype) == [OBJ_SITE] * 6 and list(m.sensor_dim) == [3] * 6
    assert list(m.sensor_objid) == [m.site_names.index("arm_imu")] * 3 + [m.site_names.index("hand_imu")] * 3
    assert measured_range(m, 0, 6) == 18
    p = load_task_imu()
    assert list(p.sensor_type) == [2, SENS_ACCELEROMETER] and p.sensor_objid[1] == p.site_names.index("center")
    assert measured_range(p, 0, 2) == 4


def _site_motion(m, q, v, s):
    """World angular / linear velocity of site s and its rotation, from refmath kinematics and body_jacobian."""
    kin = kinematics(m, q)
    b = m.site_bodyid[s]
    p = kin["xpos"][b] + kin["xmat"][b] @ m.site_pos[s]
    J = body_jacobian(m, kin, b, p)
    R = kin["xmat"][b] @ quat2mat(m.site_quat[s] / np.linalg.norm(m.site_quat[s]))
    return J[3:] @ v, J[:3] @ v, R


def imu_restated(m, q0, v0, qacc, h=1e-5):
    """gyro / velocimeter / accelerometer of every sensor of m along q(t) = q0 (+) (v0 t + qacc t^2 / 2)."""
    def at(t):
        return integrate_pos(m, q0, v0 * t + 0.5 * qacc * t * t, 1.0), v0 + qacc * t
    out = []
    for i in range(m.nsensor):
        s = int(m.sensor_objid[i])
        w, v, R = _site_motion(m, q0, v0, s)
        if m.sensor_type[i] == SENS_GYRO:
            out.append(R.T @ w)
        elif m.sensor_type[i] == SENS_VELOCIMETER:
            out.append(R.T @ v)
        else:
            acc = (_site_motion(m, *at(h), s)[1] - _site_motion(m, *at(-h), s)[1]) / (2 * h)
            out.append(R.T @ (acc - m.opt_gravity))
    return np.concatenate(out)


@pytest.mark.parametrize("scene", ["chain", "free"])
def test_imu_sensor_oracle_against_restatement(scene):
    m = compile_xml(IMU_CHAIN_XML if scene == "chain" else IMU_FREE_XML)
    o = sensor_oracle(m)
    rng = np.random.default_rng(11)
    acc = np.array([m.sensor_type[i] == SENS_ACCELEROMETER for i in range(m.nsensor) for _ in range(3)])
    for _ in range(6):
        q = m.qpos0 + 0.4 * rng.normal(size=m.nq)
        if scene == "free":
            q[3:7] /= np.linalg.norm(q[3:7])
        v = 2.0 * rng.normal(size=m.nv)
        u = rng.normal(size=m.nu)
        r = o.step(q[None], v[None], u[None], mocap_vector(m), [0.0], 0, m.nsensor)
        y, ref = r["sensordata"][0], imu_restated(m, q, v, r["qacc"][0])
        assert np.max(np.abs(y[~acc] - ref[~acc])) < 1e-12, np.abs(y - ref)[~acc].max()
        assert np.max(np.abs(y[acc] - ref[acc])) < 1e-6, np.abs(y - ref)[acc].max()
        assert np.abs(y[acc]).max() > 1e-2             # the readings are not trivially zero


def test_accelerometer_closed_forms():
    """task_imu: the particle in free fall reads 0; at rest on the plane it reads (0, 0, |g|)."""
    m = load_task_imu()
    g = np.linalg.norm(m.opt_gravity)
    X, Y, _ = simulate(m, [0.25], [0.0], 3000)
    assert np.max(np.abs(Y[0][1:])) < 1e-12 and Y[0][0] == 0.25
    assert abs(X[-1, 1]) < 1e-8
    assert np.max(np.abs(Y[-1][1:] - [0.0, 0.0, g])) < 1e-6 * g, Y[-1]


def reference_kalman_test(m, backend, epsilon=1e-6, centered=False, T=200):
    """kalman_test.cc: the errors after update_measurement at every step t against the simulation's state t."""
    X, Y, U = simulate(m, [0.25], [0.0], T)
    f = Kalman(m, backend, epsilon=epsilon, centered=centered)
    assert f.nsensordata == m.nsensordata and f.timestep == m.opt_timestep
    f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
    ep, ev = [], []
    for t in range(T):
        f.update_measurement(U[t], Y[t])
        ep.append(np.linalg.norm(f.state[:m.nq] - X[t, :m.nq]))
        ev.append(np.linalg.norm(f.state[m.nq:] - X[t, m.nq:]))
        assert np.array_equal(f.covariance, f.covariance.T)
        f.update_prediction()
    assert f.time == pytest.approx(T * m.opt_timestep) and f.warnings == 0
    # the particle hits the ground inside the window
    assert X[:, 0].min() < 0.011 and X[:, 1].max() > 0
    return np.array(ep), np.array(ev)


def test_reference_kalman_test_on_fp64_oracle():
    m = load_task_imu()
    ep, ev = reference_kalman_test(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts))
    assert ep.max() <= 1e-4 and ev.max() <= 1e-4, (ep.max(), ev.max())


@pytest.mark.parametrize("settings", ["reference", "engine"])
def test_reference_kalman_test_on_fp32_oracle(settings):
    """The same test with fp32 steps: with the reference's 1e-6 one-sided and with the engine default, the filter still
    holds the reference's 1e-4 (the bar tests/test_gpu_kalman.py holds the engine filters to)."""
    m = load_task_imu()
    kw = dict(epsilon=1e-6, centered=False) if settings == "reference" else \
        dict(epsilon=KALMAN_EPSILON, centered=KALMAN_CENTERED)
    ep, ev = reference_kalman_test(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=32), **kw)
    assert ep.max() <= 1e-4 and ev.max() <= 1e-4, (ep.max(), ev.max())


def test_sensor_covariance_failure_leaves_state_untouched():
    m = load_task_imu()
    f = Kalman(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts))
    f.reset(state=[0.25, 0.0], time=0.3)
    f.set_noise(sensor=np.full(f.nsensordata, -1.0))   # indefinite: C P C' + R cannot be factored
    before = (f.state.copy(), f.covariance.copy(), f.time)
    with pytest.raises(EstimatorError, match="sensor covariance factorisation"):
        f.update(np.zeros(m.nu), [0.25, 0.0, 0.0, 0.0])
    assert np.array_equal(f.state, before[0]) and np.array_equal(f.covariance, before[1]) and f.time == before[2]


def test_kalman_quadruped_filtering_on_the_oracles():
    """The Quadruped scenario (tests/quadruped_filtering.py) with the Kalman filter's steps on the fp64 and on the fp32
    oracle at the engine's finite differences.  The covariance stays exactly symmetric and positive definite, and no
    step warns.  Linearised through making and breaking contacts, the Kalman filter follows the plant far more loosely
    than the Unscented filter (RMS qpos about 9e-3 against 2e-3), and its errors move by 10-20 % between fp64 and fp32
    steps (fp64 8.6e-3 / 1.24, fp32 9.5e-3 / 1.48 for qpos / qvel): tests/test_gpu_kalman.py holds the engine filters
    to the fp32-oracle filter's errors + 5 % + that spread."""
    m = models.load("quadruped")
    X, Y, U = plant(m)
    res = {}
    for prec in (64, 32):
        f = Kalman(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=prec))
        assert f.nstates == 73
        res[prec] = run_filter(m, f, X, Y, U, mocap_vector(m))
        print("Kalman quadruped fp%d oracle: RMS qpos %.4g qvel %.4g, min eigenvalue %.3g" %
              (prec, res[prec][0], res[prec][1], res[prec][3]))
        assert res[prec][2] == 0.0 and res[prec][3] > 0 and f.warnings == 0
    assert res[64][0] < 2e-2 and res[32][0] < 2e-2, res     # the estimate follows the plant to a couple of cm / rad
