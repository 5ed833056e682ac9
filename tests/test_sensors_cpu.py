"""CPU: the frame, subtree, ball-joint, actuator and tendon sensors of the fp64 sensor oracle against closed forms,
physical laws and the numpy restatement of tests/sensor_scenes.py; and the loader's refusals of frame sensors it does
not implement.

Bars.  The restatement and the oracle compute the same fp64 quantities by different formulas (Jacobians times qvel
against com-based motion vectors), so they agree to the rounding of a few dozen fp64 operations: 1e-12.  The free-flight
laws hold at each state up to fp64 rounding (1e-9), and the momentum's change per Euler step is g dt to 1e-4 (second-order terms); the
angular momentum about the com, whose drift is the integrator's: first order in the timestep, so halving the timestep
halves it (ratio within 0.4 .. 0.6, the pattern of tests/test_oracle_invariants.py).
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import sensor_oracle  # noqa: E402
from sensor_scenes import ROTATIONS, random_states, scene, sensors_np  # noqa: E402

from mujoco_mpc_b200.mjcf import compile_xml, quat2mat  # noqa: E402


def _step(o, m, x, u=None, t=0.0, start=0, count=None):
    count = m.nsensor - start if count is None else count
    u = np.zeros((len(x), m.nu)) if u is None else np.atleast_2d(u)
    return o.step(x[:, :m.nq], x[:, m.nq:], u, np.zeros(0), np.full(len(x), t), start, count)


def _slices(m):
    return [slice(int(m.sensor_adr[i]), int(m.sensor_adr[i] + m.sensor_dim[i])) for i in range(m.nsensor)]


def _tendon_pair_forces(m, x, u):
    """tendon_pair's actuator forces by hand: position actuator kp (ctrl - length), motor ctrl clamped to +-0.4;
    qfrc_actuator = gear coef force per wrap / gear force on the slide"""
    q, v = x[:m.nq], x[m.nq:]
    kp, length = 3.0, 0.7 * q[0] - 0.4 * q[1]
    f = np.array([kp * (np.clip(u[0], -1, 1) - length), np.clip(np.clip(u[1], -1, 1), -0.4, 0.4)])
    qfrc = np.array([0.7 * f[0], -0.4 * f[0], 2.5 * f[1]])
    return f, qfrc


@pytest.mark.parametrize("name", ["free_body", "ball_chain", "tendon_pair"])
@pytest.mark.parametrize("rot", range(len(ROTATIONS)))
def test_oracle_against_the_numpy_restatement(name, rot):
    m = scene(name, ROTATIONS[rot])
    o = sensor_oracle(m)
    X = random_states(m, 5, seed=rot)
    U = np.random.default_rng(rot).uniform(-1, 1, size=(len(X), m.nu))
    y = _step(o, m, X, U)["sensordata"]
    skip = {10, 12, 17, 18}          # accelerometer, gyro, framelinacc, frameangacc: the physical-law tests below
    for b, x in enumerate(X):
        f, qfrc = _tendon_pair_forces(m, x, U[b]) if name == "tendon_pair" else (None, None)
        for i, s in enumerate(_slices(m)):
            if int(m.sensor_type[i]) in skip:
                continue
            ref = sensors_np(m, x[:m.nq], x[m.nq:], i, 1, f, qfrc)
            assert np.max(np.abs(y[b, s] - ref)) < 1e-12, (i, int(m.sensor_type[i]), y[b, s], ref)


def test_free_xbody_framequat_and_frame_axes():
    """A free body's xbody framequat is its normalised free-joint quaternion; every frame's x / y / z axis is the
    matching column of the matrix of that frame's framequat."""
    m = scene("free_body", ROTATIONS[3])
    X = random_states(m, 4, seed=1)
    X[:, 3:7] *= 1.7                              # an unnormalised joint quaternion
    y = _step(sensor_oracle(m), m, X)["sensordata"]
    sl = _slices(m)
    for b, x in enumerate(X):
        assert np.max(np.abs(y[b, sl[5]] - x[3:7] / np.linalg.norm(x[3:7]))) < 1e-15
        # framexaxis site imu (7) / frameyaxis body (8) / framezaxis geom (9) / framexaxis xbody (10), with the
        # framequat of the same object: site 1, body 4, geom 6, xbody 5
        for ax, quat, col in ((7, 1, 0), (8, 4, 1), (9, 6, 2), (10, 5, 0)):
            R = quat2mat(y[b, sl[quat]] / np.linalg.norm(y[b, sl[quat]]))
            assert np.max(np.abs(y[b, sl[ax]] - R[:, col])) < 1e-12, (ax, y[b, sl[ax]], R[:, col])


def test_actuator_and_tendon_closed_forms():
    """actuatorpos = gear q, tendonpos = sum coef q, with their velocities; actuatorfrc is the clamped force, and on
    the slide driven only by the motor jointactuatorfrc is gear times that force."""
    m = scene("tendon_pair")
    X = random_states(m, 6, seed=2)
    U = np.array([[0.3, 0.9], [-0.5, -0.7], [0.1, 0.2], [1.5, -2.0], [0.0, 0.41], [-1.0, 0.39]])
    y = _step(sensor_oracle(m), m, X, U)["sensordata"]
    for b, x in enumerate(X):
        q, v = x[:m.nq], x[m.nq:]
        L, Lv = 0.7 * q[0] - 0.4 * q[1], 0.7 * v[0] - 0.4 * v[1]
        f = [3.0 * (np.clip(U[b, 0], -1, 1) - L), np.clip(np.clip(U[b, 1], -1, 1), -0.4, 0.4)]
        want = [L, Lv, 2.5 * q[2], 2.5 * v[2], f[0], f[1], 2.5 * f[1], 0.7 * f[0], L, Lv]
        assert np.max(np.abs(y[b, :10] - want)) < 1e-12, (y[b, :10], want)
    assert abs(y[0, 5]) == 0.4 and abs(y[1, 5]) == 0.4 and abs(y[2, 5]) == pytest.approx(0.2)   # the limit binds


def _fly(m, steps, seed=0):
    """fp64 oracle free flight from a random state: (states, sensordata)"""
    o = sensor_oracle(m)
    x = random_states(m, 1, seed=seed)
    X, Y = [], []
    w = np.zeros((1, m.nv))
    for t in range(steps):
        r = o.step(x[:, :m.nq], x[:, m.nq:], np.zeros((1, m.nu)), np.zeros(0), [t * m.opt_timestep], 0, m.nsensor,
                   warmstart=w)
        X.append(x[0]); Y.append(r["sensordata"][0])
        x, w = np.concatenate([r["next_qpos"], r["next_qvel"]], 1), r["qacc"]
    return np.array(X), np.array(Y)


@pytest.mark.parametrize("rot", [0, 3])
def test_free_flight_laws(rot):
    """A free body in flight.  MuJoCo's com-based acceleration carries the gravity offset (cacc of the world is
    [0, -gravity]), so framelinacc is the classical acceleration of the frame's point minus g: 0 at the centre of mass
    (free fall) and alpha x r + w x (w x r) at a point r from it, with frameangacc = alpha given by Euler's equations
    I alpha = -w x I w (the asymmetric inertia makes it non-zero).  subtreelinvel is the total momentum over the mass
    and changes by g dt per step."""
    m = scene("free_body", ROTATIONS[rot])
    g, h = np.asarray(m.opt_gravity, float), m.opt_timestep
    X, Y = _fly(m, 200)
    sl = _slices(m)
    com = Y[:, sl[20]]
    for k in range(0, len(Y), 10):
        w, alpha = Y[k, sl[14]], Y[k, sl[19]]        # frameangvel of the xbody, frameangacc of the inertial frame
        R = quat2mat(Y[k, sl[4]] / np.linalg.norm(Y[k, sl[4]]))
        I = R @ np.diag(m.body_inertia[1]) @ R.T
        assert np.linalg.norm(alpha) > 1e-2
        assert np.max(np.abs(I @ alpha + np.cross(w, I @ w))) < 1e-9
        assert np.max(np.abs(Y[k, sl[18]])) < 1e-9   # framelinacc of the inertial frame: free fall
        # framelinacc of the site (its framepos is sensor 0), of the xbody and of the geom
        xb = X[k, :3]
        geom = m.geom_bodyid[0]
        for i, p in ((15, Y[k, sl[0]]), (16, xb), (17, None)):
            if p is None:
                Rb = quat2mat(X[k, 3:7] / np.linalg.norm(X[k, 3:7]))
                p = xb + Rb @ m.geom_pos[0]
            r = p - com[k]
            want = np.cross(alpha, r) + np.cross(w, np.cross(w, r))
            assert np.max(np.abs(Y[k, sl[i]] - want)) < 1e-9, (i, Y[k, sl[i]], want)
        assert geom == 1
    # the accelerometer of the IMU site reads its framelinacc rotated into the site frame
    Rs = np.array([quat2mat(q / np.linalg.norm(q)) for q in Y[:, sl[1]]])
    assert np.max(np.abs(np.einsum("kji,kj->ki", Rs, Y[:, sl[15]]) - Y[:, sl[3]])) < 1e-9
    vcom = Y[:, sl[21]]
    mom = np.array([m.body_mass[1] * Y[k, sl[12]] for k in range(len(Y))])   # framelinvel of the inertial frame
    assert np.max(np.abs(vcom - mom / m.body_mass[1])) < 1e-12
    # the Euler step integrates the free joint's frame origin, not the com, so the com velocity changes by g dt up to
    # terms of second order in dt (w and the origin-to-com offset change within the step)
    assert np.max(np.abs(np.diff(vcom, axis=0) - g * h)) < 1e-4 * 9.81 * h


def test_ballquat_has_unit_norm():
    m = scene("ball_chain", ROTATIONS[2])
    X = random_states(m, 8, seed=3)
    a = m.jnt_qposadr[m.jnt_names.index("ball")]
    X[:, a:a + 4] *= np.linspace(0.5, 2.0, 8)[:, None]
    y = _step(sensor_oracle(m), m, X)["sensordata"]
    assert np.max(np.abs(np.linalg.norm(y[:, :4], axis=1) - 1)) < 1e-15


@pytest.mark.parametrize("name,body,adr", [("free_body", 1, 70), ("ball_chain", 1, 13)])
def test_subtree_angular_momentum_is_conserved(name, body, adr):
    """In free flight the angular momentum about the subtree com is conserved; the Euler step's drift halves with the
    timestep."""
    drift = []
    for h in (2e-3, 1e-3):
        m = compile_xml(__import__("sensor_scenes").SCENES[name](ROTATIONS[1], h))
        _, Y = _fly(m, int(round(0.2 / h)), seed=4)
        L = Y[:, adr:adr + 3]
        assert np.linalg.norm(L[0]) > 1e-3
        drift.append(np.linalg.norm(L[-1] - L[0]) / np.linalg.norm(L[0]))
    assert drift[0] < 0.05 and 0.4 < drift[1] / drift[0] < 0.6, drift


@pytest.mark.parametrize("attr", ['reftype="body" refname="b"', 'refname="b"'])
def test_loader_refuses_reference_frames(attr):
    xml = """<mujoco><worldbody><body name="b"><freejoint/><geom size="0.1"/><site name="s"/></body></worldbody>
      <sensor><framequat objtype="site" objname="s" %s/></sensor></mujoco>""" % attr
    with pytest.raises(ValueError, match="reftype / refname"):
        compile_xml(xml)


def test_loader_refuses_camera_frames():
    xml = """<mujoco><worldbody><body name="b"><freejoint/><geom size="0.1"/><camera name="c"/></body></worldbody>
      <sensor><framelinvel objtype="camera" objname="c"/></sensor></mujoco>"""
    with pytest.raises(ValueError, match="camera"):
        compile_xml(xml)
