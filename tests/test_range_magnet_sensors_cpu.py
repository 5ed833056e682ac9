"""CPU: the magnetometer and rangefinder of the loader and the fp64 sensor oracle, against closed forms and an
independent numpy restatement.  The scenes here are shared with tests/test_gpu_range_magnet_sensors.py.

Bars.  Closed forms and the oracle are fp64 evaluations of the same geometry, with the probe's pose written to the
MJCF in 12 digits: 1e-10 (distances of order 1).  The numpy
restatement finds each ray's first crossing of an implicit surface by sampling and bisection, a formulation independent
of the oracle's quadratics, and is converged to 1e-10.
"""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import sensor_oracle  # noqa: E402
from sensor_scenes import ROTATIONS  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.blob import from_blob, to_blob  # noqa: E402
from mujoco_mpc_b200.mjcf import (GEOM_BOX, GEOM_CAPSULE, GEOM_CYLINDER, GEOM_ELLIPSOID, GEOM_PLANE,  # noqa: E402
                                  GEOM_SPHERE, SENS_MAGNETOMETER, SENS_MEASURED, SENS_RANGEFINDER, SENS_TENDONVEL,
                                  axisangle2quat, compile_xml, quat2mat, quat_mul)

MAGNETIC = (0.12, -0.41, 0.23)


def _fmt(v):
    return " ".join("%.12g" % x for x in v)


def probe_xml(geoms, pos=(0, 0, 1), quat=(1, 0, 0, 0), magnetic=MAGNETIC, assets="", extra_sites="", extra_sensors=""):
    """A free probe body (its own sphere geom of radius 0.05 around the eye site, which the rangefinder must skip) at
    pos / quat among `geoms`; sensors: rangefinder and magnetometer of the eye, then a user sensor (its address shows
    where the sensors after a magnetometer start)."""
    mag = "" if magnetic is None else ' magnetic="%s"' % _fmt(magnetic)
    return f"""
<mujoco model="range probe">
  <option timestep="0.002" gravity="0 0 0"{mag}><flag contact="disable"/></option>
  <asset>{assets}</asset>
  <worldbody>
    {geoms}
    <body name="probe" pos="{_fmt(pos)}" quat="{_fmt(quat)}">
      <freejoint/>
      <geom name="shell" type="sphere" size="0.05" mass="0.5"/>
      <site name="eye"/>
      {extra_sites}
    </body>
  </worldbody>
  <sensor>
    <rangefinder name="range" site="eye"/>
    <magnetometer name="mag" site="eye"/>
    {extra_sensors}
    <user name="after" dim="2"/>
  </sensor>
</mujoco>"""


def down(theta=0.0):
    """the probe's quaternion whose z axis is -z tilted by theta towards -y"""
    return axisangle2quat([1, 0, 0], math.pi - theta)


def read(m, x=None, precision=64):
    """(rangefinder, magnetometer) of the probe's state x (default: qpos0 at rest) from the sensor oracle"""
    o = sensor_oracle(m, precision=precision)
    x = np.concatenate([m.qpos0, np.zeros(m.nv)])[None] if x is None else np.atleast_2d(x)
    # every sensor but the last, the user sensor
    y = o.step(x[:, :m.nq], x[:, m.nq:], np.zeros((len(x), m.nu)), np.zeros(0), np.zeros(len(x)), 0, m.nsensor - 1)
    return y["sensordata"]


# --------------------------------------------------------------------------------------- the room of random states
ROOM_GEOMS = """
    <geom name="floor" type="plane" size="0 0 1"/>
    <geom name="deck" type="plane" pos="1.6 0.2 0.35" size="0.4 0.3 0.1" euler="0 0 20"/>
    <geom name="ball" type="sphere" pos="0.8 0.6 0.4" size="0.25"/>
    <geom name="crate" type="box" pos="-0.7 0.5 0.3" size="0.2 0.15 0.3" euler="10 -15 30"/>
    <geom name="pipe" type="capsule" fromto="-0.6 -0.6 0.4 0.2 -0.9 0.6" size="0.12"/>
    <geom name="drum" type="cylinder" pos="0.7 -0.6 0.3" size="0.2 0.25" euler="25 5 0"/>
    <geom name="egg" type="ellipsoid" pos="0 1.0 0.5" size="0.3 0.2 0.15" euler="0 30 45"/>
    <geom name="ghost" type="box" pos="0 0 0.45" size="0.3 0.3 0.05" rgba="1 0 0 0"/>
    <geom name="glass" type="sphere" pos="-0.3 -0.2 0.6" size="0.15" material="clear"/>
"""
ROOM_ASSETS = '<material name="clear" rgba="1 1 1 0"/><material name="paint" rgba="0.2 0.3 0.4 1"/>'
# rangefinders along other directions of the probe, and a site of a second body on the probe's chain would be a
# world geom: these sites look down, sideways and up
ROOM_SITES = """
      <site name="side" pos="0.02 0 0" zaxis="1 0.3 -0.6"/>
      <site name="back" pos="0 -0.03 0.01" zaxis="-0.4 -1 -0.5"/>
      <site name="up" zaxis="0.1 0.2 1"/>
"""
ROOM_SENSORS = """
    <rangefinder name="side" site="side"/><rangefinder name="back" site="back"/><rangefinder name="up" site="up"/>
    <magnetometer name="mag_side" site="side"/>
"""


def room(rot=ROTATIONS[0]):
    """the probe among every geom type, an alpha-0 box and a sphere whose material's alpha is 0"""
    return compile_xml(probe_xml(ROOM_GEOMS, pos=(0.1, 0.05, 1.1), quat=down(0.3), assets=ROOM_ASSETS,
                                 extra_sites=ROOM_SITES, extra_sensors=ROOM_SENSORS))


def room_states(m, k, seed=0):
    """k poses of the probe over the room, looking mostly down, with random velocities"""
    rng = np.random.default_rng(seed)
    X = np.zeros((k, m.nq + m.nv))
    for i in range(k):
        X[i, :3] = [rng.uniform(-1.2, 1.9), rng.uniform(-1.0, 1.2), rng.uniform(0.75, 1.6)]
        q = quat_mul(down(rng.uniform(-0.9, 0.9)), axisangle2quat(rng.normal(size=3), rng.uniform(0, 0.8)))
        X[i, 3:7] = q / np.linalg.norm(q)
        X[i, 7:] = rng.normal(size=m.nv)
    return X


# ------------------------------------------------------------------------------------------- numpy restatement
def _implicit(m, g, p):
    """f(p) < 0 inside geom g, > 0 outside, for points p [n][3] in the geom's frame"""
    t, s = int(m.geom_type[g]), m.geom_size[g]
    if t == GEOM_SPHERE:
        return np.linalg.norm(p, axis=1) - s[0]
    if t == GEOM_ELLIPSOID:
        return np.sum((p / s) ** 2, axis=1) - 1
    if t == GEOM_BOX:
        return np.max(np.abs(p) - s, axis=1)
    if t == GEOM_CAPSULE:
        z = np.clip(p[:, 2], -s[1], s[1])
        return np.linalg.norm(p - np.stack([0 * z, 0 * z, z], 1), axis=1) - s[0]
    if t == GEOM_CYLINDER:
        return np.maximum(np.hypot(p[:, 0], p[:, 1]) - s[0], np.abs(p[:, 2]) - s[1])
    raise NotImplementedError(t)


def _geom_pose(m, kin, g):
    b = m.geom_bodyid[g]
    return kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g], kin["xmat"][b] @ quat2mat(m.geom_quat[g])


def ray_np(m, kin, g, pnt, vec, tmax=6.0, step=1e-3):
    """first crossing of geom g's surface by pnt + t vec: a plane analytically (front face, extent), a solid by sampling
    its implicit function and bisecting the first sign change"""
    c, R = _geom_pose(m, kin, g)
    lp, lv = R.T @ (pnt - c), R.T @ vec
    if int(m.geom_type[g]) == GEOM_PLANE:
        if lv[2] >= 0:
            return -1.0
        t = -lp[2] / lv[2]
        x = lp + t * lv
        s = m.geom_size[g]
        return t if (s[0] <= 0 or abs(x[0]) <= s[0]) and (s[1] <= 0 or abs(x[1]) <= s[1]) else -1.0
    ts = np.arange(0, tmax, step)
    f = _implicit(m, g, lp[None] + ts[:, None] * lv[None])
    change = np.nonzero(np.sign(f[1:]) != np.sign(f[0]))[0]
    if change.size == 0:
        return -1.0
    a, b = ts[change[0]], ts[change[0] + 1]
    fa = f[change[0]]
    for _ in range(60):
        mid = 0.5 * (a + b)
        fm = _implicit(m, g, (lp + mid * lv)[None])[0]
        if np.sign(fm) == np.sign(fa):
            a = mid
        else:
            b = mid
    return 0.5 * (a + b)


def range_np(m, qpos, site):
    """mj_ray of the rangefinder at `site`: every geom not of the site's body with alpha != 0"""
    from mujoco_mpc_b200.refmath import kinematics
    kin = kinematics(m, np.asarray(qpos, float))
    b = m.site_bodyid[site]
    R = kin["xmat"][b] @ quat2mat(m.site_quat[site])
    pnt = kin["xpos"][b] + kin["xmat"][b] @ m.site_pos[site]
    hits = [ray_np(m, kin, g, pnt, R[:, 2]) for g in range(m.ngeom) if m.geom_bodyid[g] != b and m.geom_alpha[g] != 0]
    hits = [h for h in hits if h >= 0]
    return min(hits) if hits else -1.0


def magnet_np(m, qpos, site):
    from mujoco_mpc_b200.refmath import kinematics
    kin = kinematics(m, np.asarray(qpos, float))
    b = m.site_bodyid[site]
    return (kin["xmat"][b] @ quat2mat(m.site_quat[site])).T @ m.opt_magnetic


# ----------------------------------------------------------------------------------------------------- loader
def test_codes_dimensions_and_addresses():
    assert (SENS_MAGNETOMETER, SENS_RANGEFINDER) == (SENS_TENDONVEL + 1, SENS_TENDONVEL + 2)
    assert SENS_MAGNETOMETER in SENS_MEASURED and SENS_RANGEFINDER in SENS_MEASURED
    m = compile_xml(probe_xml("", extra_sensors='<magnetometer site="eye"/><framepos objtype="site" objname="eye"/>'))
    assert list(m.sensor_type[:4]) == [SENS_RANGEFINDER, SENS_MAGNETOMETER, SENS_MAGNETOMETER, 1]
    # MuJoCo's addresses: rangefinder 1, magnetometer 3, so the user sensor after them starts at 1 + 3 + 3 + 3
    assert list(m.sensor_dim) == [1, 3, 3, 3, 2] and list(m.sensor_adr) == [0, 1, 4, 7, 10] and m.nsensordata == 12
    site = m.site_names.index("eye")
    assert list(m.sensor_objtype[:3]) == [3, 3, 3] and list(m.sensor_objid[:3]) == [site] * 3


def test_magnetic_option_and_alpha():
    m = compile_xml(probe_xml("", magnetic=None))
    assert np.array_equal(m.opt_magnetic, [0, -0.5, 0])
    m = compile_xml(probe_xml("", magnetic=(1, 2, 3)))
    assert np.array_equal(m.opt_magnetic, [1, 2, 3])
    m = room()
    alpha = dict(zip(m.geom_names, m.geom_alpha))
    assert alpha["ghost"] == 0 and alpha["glass"] == 0 and alpha["floor"] == 1 and alpha["shell"] == 1
    b = from_blob(to_blob(m))
    assert np.array_equal(b["opt_magnetic"], MAGNETIC) and np.array_equal(b["geom_alpha"], m.geom_alpha)


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track", "shadow_reorient", "cartpole", "particle"])
def test_shipped_blobs_gain_no_entry(name):
    b = from_blob(to_blob(models.load(name)))
    assert "opt_magnetic" not in b and "geom_alpha" not in b


# ------------------------------------------------------------------------------------------ oracle, closed forms
@pytest.mark.parametrize("rot", range(len(ROTATIONS)))
@pytest.mark.parametrize("magnetic", [None, MAGNETIC])
def test_magnetometer_is_the_field_in_the_site_frame(rot, magnetic):
    q = np.asarray(ROTATIONS[rot], float)
    q /= np.linalg.norm(q)
    site_quat = axisangle2quat([0.3, -0.5, 0.8], 0.7)
    m = compile_xml(probe_xml("", quat=q, magnetic=magnetic,
                              extra_sites='<site name="tilted" quat="%s"/>' % _fmt(site_quat),
                              extra_sensors='<magnetometer site="tilted"/>'))
    B = np.array([0, -0.5, 0] if magnetic is None else magnetic)
    y = read(m)[0]
    assert np.max(np.abs(y[1:4] - quat2mat(q).T @ B)) < 1e-10
    assert np.max(np.abs(y[4:7] - quat2mat(quat_mul(q, site_quat)).T @ B)) < 1e-10


@pytest.mark.parametrize("theta", [0.0, 0.3, 0.9, 1.3])
def test_plane_reads_height_over_cos(theta):
    h = 0.8
    m = compile_xml(probe_xml('<geom type="plane" size="0 0 1"/>', pos=(0.3, -0.2, h), quat=down(theta)))
    assert abs(read(m)[0, 0] - h / math.cos(theta)) < 1e-10
    # pointing up, away from the front face; and from behind the plane, pointing at its back face
    m = compile_xml(probe_xml('<geom type="plane" size="0 0 1"/>', pos=(0.3, -0.2, h), quat=down(math.pi - theta)))
    assert read(m)[0, 0] == -1
    m = compile_xml(probe_xml('<geom type="plane" size="0 0 1"/>', pos=(0.3, -0.2, -h), quat=down(math.pi - theta)))
    assert read(m)[0, 0] == -1


def test_finite_plane_is_missed_outside_its_extent():
    xml = '<geom type="plane" pos="0 0 0.2" size="0.5 0.3 0.1"/>'
    for x, y, hit in ((0.4, 0.2, True), (0.6, 0.0, False), (0.0, 0.35, False), (-0.45, -0.25, True)):
        r = read(compile_xml(probe_xml(xml, pos=(x, y, 1.0), quat=down())))[0, 0]
        assert (r == -1) if not hit else abs(r - 0.8) < 1e-10, (x, y, r)


# (geom xml, probe position, the distance down from it)
H = 1.5
CLOSED_FORMS = {
    "sphere": ('<geom type="sphere" pos="0.1 0.2 0.3" size="0.25"/>', (0.1, 0.2, H), H - 0.3 - 0.25),
    "sphere_offset": ('<geom type="sphere" pos="0 0 0.3" size="0.25"/>', (0.15, 0, H), H - 0.3 - math.sqrt(0.25 ** 2 - 0.15 ** 2)),
    "box": ('<geom type="box" pos="0 0 0.2" size="0.3 0.2 0.1"/>', (0.25, -0.15, H), H - 0.3),
    "box_turned": ('<geom type="box" pos="0 0 0.4" size="0.3 0.2 0.1" euler="0 0 40"/>', (0.05, 0.05, H), H - 0.5),
    "capsule_side": ('<geom type="capsule" fromto="-0.4 0 0.3 0.4 0 0.3" size="0.1"/>', (0.2, 0.05, H),
                     H - 0.3 - math.sqrt(0.01 - 0.0025)),
    "capsule_cap": ('<geom type="capsule" fromto="0 0 0.1 0 0 0.5" size="0.1"/>', (0, 0, H), H - 0.6),
    "capsule_cap_offset": ('<geom type="capsule" fromto="0 0 0.1 0 0 0.5" size="0.1"/>', (0.06, 0, H),
                           H - 0.5 - math.sqrt(0.01 - 0.0036)),
    "capsule_lying_cap": ('<geom type="capsule" pos="0 0 0.3" size="0.1 0.2" euler="90 0 0"/>', (0, 0.25, H),
                          H - 0.3 - math.sqrt(0.01 - 0.0025)),
    "cylinder_side": ('<geom type="cylinder" fromto="-0.4 0 0.3 0.4 0 0.3" size="0.1"/>', (0.35, 0.06, H),
                      H - 0.3 - math.sqrt(0.01 - 0.0036)),
    "cylinder_end": ('<geom type="cylinder" pos="0 0 0.2" size="0.15 0.2"/>', (0.1, -0.05, H), H - 0.4),
    "ellipsoid": ('<geom type="ellipsoid" pos="0 0 0.3" size="0.3 0.2 0.15"/>', (0.2, 0, H),
                  H - 0.3 - 0.15 * math.sqrt(1 - (0.2 / 0.3) ** 2)),
    "ellipsoid_turned": ('<geom type="ellipsoid" pos="0 0 0.3" size="0.3 0.2 0.15" euler="90 0 0"/>', (0, 0, H), H - 0.5),
}


@pytest.mark.parametrize("case", sorted(CLOSED_FORMS))
def test_known_distances(case):
    xml, pos, dist = CLOSED_FORMS[case]
    m = compile_xml(probe_xml(xml, pos=pos, quat=down()))
    assert abs(read(m)[0, 0] - dist) < 1e-10, (read(m)[0, 0], dist)


def test_ray_starting_inside_reads_the_exit():
    m = compile_xml(probe_xml('<geom type="sphere" pos="0 0 0.9" size="0.3"/>', pos=(0, 0, 1.0), quat=down()))
    assert abs(read(m)[0, 0] - 0.4) < 1e-10


def test_nearest_of_several_and_skips():
    geoms = """<geom type="plane" size="0 0 1"/><geom type="sphere" pos="0 0 0.4" size="0.2"/>
               <geom type="box" pos="0.02 0 0.9" size="0.1 0.1 0.1"/>"""
    m = compile_xml(probe_xml(geoms, pos=(0, 0, 1.5), quat=down()))
    assert abs(read(m)[0, 0] - 0.5) < 1e-10                      # the box's top at 1.0
    # the box made invisible (geom rgba, then a material's) leaves the sphere's top at 0.6
    for vis in ('rgba="1 1 1 0"', 'material="clear"'):
        g = geoms.replace('size="0.1 0.1 0.1"', 'size="0.1 0.1 0.1" %s' % vis)
        m = compile_xml(probe_xml(g, pos=(0, 0, 1.5), quat=down(), assets='<material name="clear" rgba="1 1 1 0"/>'))
        assert abs(read(m)[0, 0] - 0.9) < 1e-10, vis
    # a material with alpha > 0 wins over a geom rgba with alpha 0: the box is hit again
    g = geoms.replace('size="0.1 0.1 0.1"', 'size="0.1 0.1 0.1" rgba="1 1 1 0" material="paint"')
    m = compile_xml(probe_xml(g, pos=(0, 0, 1.5), quat=down(), assets='<material name="paint" rgba="1 1 1 1"/>'))
    assert abs(read(m)[0, 0] - 0.5) < 1e-10
    # the probe's own shell (radius 0.05 around the eye) is never hit; with nothing else the ray misses
    m = compile_xml(probe_xml("", pos=(0, 0, 1.5), quat=down()))
    assert read(m)[0, 0] == -1


# -------------------------------------------------------------------------------- oracle against the restatement
def test_room_against_the_numpy_restatement():
    m = room()
    sites = [int(m.sensor_objid[i]) for i in range(m.nsensor) if m.sensor_type[i] == SENS_RANGEFINDER]
    mags = [int(m.sensor_objid[i]) for i in range(m.nsensor) if m.sensor_type[i] == SENS_MAGNETOMETER]
    X = room_states(m, 24, seed=3)
    Y = read(m, X)
    ri = [int(m.sensor_adr[i]) for i in range(m.nsensor) if m.sensor_type[i] == SENS_RANGEFINDER]
    mi = [int(m.sensor_adr[i]) for i in range(m.nsensor) if m.sensor_type[i] == SENS_MAGNETOMETER]
    hits = 0
    for b, x in enumerate(X):
        for a, s in zip(ri, sites):
            ref = range_np(m, x[:m.nq], s)
            assert abs(Y[b, a] - ref) < 1e-9, (b, s, Y[b, a], ref)
            hits += ref >= 0
        for a, s in zip(mi, mags):
            assert np.max(np.abs(Y[b, a:a + 3] - magnet_np(m, x[:m.nq], s))) < 1e-10
    assert hits >= len(X) * 2, hits    # most rays hit something


def test_oracle_refuses_a_hfield():
    m = compile_xml(probe_xml('<geom type="hfield" size="1 1 0.1"/>'))
    with pytest.raises(ValueError, match="not evaluated"):
        read(m)


# ------------------------------------------------------------------------------ the IMU body with its third sensor
def imu_nav(timestep=0.005):
    """sensor_scenes.imu_body's free body over a floor (contact off), with a magnetometer on its IMU site and a
    rangefinder on a site that looks straight down at the body's initial pose.  Sensors: 0 magnetometer, 1 framepos
    of the xbody (the body origin, whose position does not depend on the orientation), 2 gyro, 3 accelerometer,
    4 rangefinder; [0, 4) measures the heading, [1, 4) does not; [2, 5) measures the height, [2, 4) does not."""
    from sensor_scenes import free_body_xml
    xml = free_body_xml(ROTATIONS[0], timestep)
    m0 = compile_xml(xml)
    R = quat2mat(m0.qpos0[3:7])
    eye = '<site name="eye" zaxis="%s"/>' % _fmt(R.T @ np.array([0, 0, -1.0]))
    xml = xml.replace('<site name="corner"', eye + '\n      <site name="corner"', 1)
    xml = xml.replace("<worldbody>", """<custom><numeric name="estimator_timestep" data="%g"/></custom>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1"/>""" % timestep, 1)
    i, j = xml.index("<sensor>"), xml.index("</sensor>")
    return compile_xml(xml[:i] + """<sensor>
    <magnetometer site="imu"/><framepos objtype="xbody" objname="body"/><gyro site="imu"/>
    <accelerometer site="imu"/><rangefinder site="eye"/>
  """ + xml[j:])


def yaw_error(q_est, q_true):
    """the rotation about the world z axis that takes the true orientation to the estimate"""
    E = quat2mat(q_est / np.linalg.norm(q_est)) @ quat2mat(q_true).T
    return abs(math.atan2(E[1, 0] - E[0, 1], E[0, 0] + E[1, 1]))


def nav_flight(m, T):
    """an fp64 oracle flight of imu_nav from a seeded state: states [T + 1], every sensor's readings with Gaussian
    noise of std 1e-3"""
    from estimator_backends import simulate
    rng = np.random.default_rng(5)
    v0 = np.concatenate([0.1 * rng.normal(size=3), 0.4 * rng.normal(size=3)])
    return simulate(m, m.qpos0, v0, T + 1, timestep=0.005, start=0, count=5, noise=1e-3, seed=6)


def nav_start(m, x, what):
    """the filter's initial state and covariance: the true state with a 0.5 rad yaw error ("heading") or a 0.3 m height
    error ("height"), and a covariance that admits it"""
    x = x.copy()
    P = 1e-6 * np.eye(2 * m.nv)
    if what == "heading":
        x[3:7] = quat_mul(axisangle2quat([0, 0, 1], 0.5), x[3:7])
        P[5, 5] = 0.25
    else:
        x[2] += 0.3
        P[2, 2] = 0.09
    return x, P


NAV = {("heading", True): (0, 4), ("heading", False): (1, 3), ("height", True): (2, 3), ("height", False): (2, 2)}


def nav_columns(m, what, measured):
    """the filter's sensor range (start, count) and its sensordata columns [a, e)"""
    s, n = NAV[(what, measured)]
    return s, n, int(m.sensor_adr[s]), int(m.sensor_adr[s + n - 1] + m.sensor_dim[s + n - 1])


def nav_error(m, x, x_true, what):
    return yaw_error(x[3:7], x_true[3:7]) if what == "heading" else abs(x[2] - x_true[2])


# the error after the last of NAV_T updates: below the first bar when the sensor is measured, above the second when not
NAV_T = 60
NAV_BARS = {"heading": (0.02, 0.4), "height": (0.01, 0.25)}


@pytest.mark.parametrize("kind", ["kalman", "unscented"])
@pytest.mark.parametrize("what", ["heading", "height"])
def test_oracle_filters_observe_heading_and_height(kind, what):
    """The Python filters on the fp64 sensor oracle: with the magnetometer the yaw error falls, with the rangefinder the
    height error falls, and without them neither does."""
    from estimator_backends import OracleSigmaBackend
    from mujoco_mpc_b200.estimator import Kalman, Unscented
    m = imu_nav()
    T = NAV_T
    X, Y, U = nav_flight(m, T)
    F = Kalman if kind == "kalman" else Unscented
    for measured in (True, False):
        s, n, a, e = nav_columns(m, what, measured)
        f = F(m, lambda s_, n_, ts: OracleSigmaBackend(m, s_, n_, ts, 64), sensor_start=s, nsensor=n)
        x0, P0 = nav_start(m, X[0], what)
        f.reset(state=x0)
        f.covariance = P0
        f.set_noise(process=np.full(2 * m.nv, 1e-8), sensor=np.full(e - a, 1e-6))
        for t in range(T):
            f.update(U[t], Y[t][a:e], np.zeros(0))
        err = nav_error(m, f.state, X[T], what)
        print("%s %s, %s: final error %.3g" % (kind, what, "measured" if measured else "not measured", err))
        assert err < NAV_BARS[what][0] if measured else err > NAV_BARS[what][1], (measured, err)
