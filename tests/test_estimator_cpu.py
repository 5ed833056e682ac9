"""Measurement sensors, the model description they need and the Unscented filter on the fp64 oracle (no GPU).

The filter tests are the reference's own (mjpc/test/estimator/unscented_test.cc, Particle1D and Box3Drot) on their
verbatim models: covariance, process and sensor noise 1e-5, noise-free measurements, and the filtered state at step t
against the simulation at t + 1 within 1e-4 (norm of the position error, quaternion difference for the box).
"""
import hashlib
import struct
import sys
import os

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from estimator_backends import (OracleSigmaBackend, box_corner_closed_form, load_estimator_model, quat_error,  # noqa: E402
                                sensors_fp64, simulate)

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200 import task as T  # noqa: E402
from mujoco_mpc_b200.blob import from_blob, to_blob  # noqa: E402
from mujoco_mpc_b200.estimator import EstimatorError, Unscented, measured_range, quaternion_mean  # noqa: E402
from mujoco_mpc_b200.mjcf import GEOM_SPHERE, SENS_JOINTVEL, SENS_TOUCH, compile_xml  # noqa: E402

# sha256 of each shipped model's blob before the sensor / site entries existed
PARENT_BLOB_SHA256 = {
    "particle": "f645f6d5860e22618cb582d7eed1ec9c6425bcefa0403a5915bc4270bea022e4",
    "particle_copy": "3b892689888e636e1cdbc7c9fec08e1c9a5b10ef49287cd0433c65852ba56068",
    "cartpole": "f3fd2d8adbf1171b3d51908aebc041a565f730d36f0514b204c5422b48dbc87e",
    "quadruped": "6802ca294cf132d5fadfc3977af85d644c9cf59f556337ba2bbf9567b7a11986",
    "humanoid": "34f75c02cd3eaa3227adbd3b2e2de521403743170ad176b972fd3741560295d1",
    "humanoid_track": "23f83159b96d8bf8586c9eda38c18d4dcbaa7e9a28039e8d7833829c3a3a919a",
    "shadow_reorient": "1a3a1f24de0b3df58701c338d911904aaba71d53da886281ff4d13f928fcfd73",
}
NEW_ENTRIES = {"nsensor", "sensor_type", "sensor_objtype", "sensor_objid", "sensor_dim", "sensor_adr", "site_type",
               "site_size", "sensor_cutoff"}


def _without(blob, drop):
    """Re-serialise a blob without the entries in `drop` (same layout rules as blob.to_blob)."""
    _, n = struct.unpack_from("<ii", blob, 8)
    kept = []
    for i in range(n):
        name, dt, cnt, off = struct.unpack_from("<40siiq", blob, 16 + 56 * i)
        if name.rstrip(b"\0").decode() not in drop:
            kept.append((name, dt, cnt, blob[off:off + cnt * (8 if dt else 4)]))
    off = 16 + 56 * len(kept)
    table, payload = bytearray(), bytearray()
    for name, dt, cnt, raw in kept:
        pad = (-len(raw)) % 8
        table += struct.pack("<40siiq", name, dt, cnt, off)
        payload += raw + b"\0" * pad
        off += len(raw) + pad
    return blob[:8] + struct.pack("<ii", 1, len(kept)) + bytes(table) + bytes(payload)


@pytest.mark.parametrize("name", sorted(PARENT_BLOB_SHA256))
def test_shipped_blobs_unchanged_apart_from_sensor_entries(name):
    blob = to_blob(models.load(name))
    assert NEW_ENTRIES <= set(from_blob(blob))
    assert hashlib.sha256(_without(blob, NEW_ENTRIES)).hexdigest() == PARENT_BLOB_SHA256[name]


def test_sensor_and_site_description():
    m = models.load("quadruped")
    b = from_blob(to_blob(m))
    assert int(b["nsensor"][0]) == m.nsensor == len(b["sensor_type"])
    # the reference's 21 estimator sensors: 5 framepos, 12 jointpos, 4 touch on the foot sites (sphere, r 0.015)
    s0, n = int(m.numeric["estimator_sensor_start"][0]), int(m.numeric["estimator_number_sensor"][0])
    assert (s0, n) == (9, 21) and float(m.numeric["estimator_timestep"][0]) == 0.005
    assert list(b["sensor_type"][s0:s0 + n]) == [1] * 5 + [2] * 12 + [SENS_TOUCH] * 4
    assert measured_range(m, s0, n) == 5 * 3 + 12 + 4
    for i in range(s0 + 17, s0 + 21):
        site = int(b["sensor_objid"][i])
        assert b["site_type"][site] == GEOM_SPHERE and b["site_size"][3 * site] == pytest.approx(0.015)
    c = models.load("cartpole")
    assert (int(c.numeric["estimator_sensor_start"][0]), int(c.numeric["estimator_number_sensor"][0])) == (4, 2)
    assert measured_range(c, 4, 2) == 2
    p = load_estimator_model("particle1d")
    assert list(p.sensor_type) == [2, SENS_JOINTVEL]


def test_measured_range_refusals():
    m = models.load("quadruped")
    with pytest.raises(EstimatorError, match="not a measured sensor"):
        measured_range(m, 0, 10)            # user sensors (cost terms)
    with pytest.raises(EstimatorError, match="outside"):
        measured_range(m, 9, m.nsensor)
    xml = open(os.path.join(os.path.dirname(__file__), "golden", "estimator_particle_task1D.xml")).read()
    mc = compile_xml(xml.replace('<jointvel name="vel_z" joint="root_z" />',
                                 '<jointvel name="vel_z" joint="root_z" cutoff="1"/>'))
    with pytest.raises(EstimatorError, match="cutoff"):
        measured_range(mc, 0, 2)


def test_model_without_cost_terms_has_no_residual(oracle_lib):
    for name in ("particle1d", "box3drot"):
        m = load_estimator_model(name)
        assert m.task_num_term == 0 and m.task_residual_id == T.RESIDUAL_NONE
    # and it steps on the oracle (the reference's Particle1D falls freely)
    m = load_estimator_model("particle1d")
    X, _, _ = simulate(m, [0.25], [0.0], 3)
    h = m.opt_timestep
    assert X[1, 1] == pytest.approx(-9.81 * h, rel=1e-12) and X[2, 0] == pytest.approx(0.25 - 3 * 9.81 * h * h, rel=1e-12)


def test_oracle_sensors_against_closed_forms():
    rng = np.random.default_rng(7)
    p = load_estimator_model("particle1d")
    for _ in range(5):
        q, v = rng.normal(size=1), rng.normal(size=1)
        assert np.array_equal(sensors_fp64(p, q, v, 0, 2), np.array([q[0], v[0]]))
    b = load_estimator_model("box3drot")
    for _ in range(5):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        y = sensors_fp64(b, q, np.zeros(3), 0, 8)
        assert np.max(np.abs(y - box_corner_closed_form(b, q))) < 1e-12


def test_quaternion_mean_against_eigh():
    """quaternion_mean runs the Jacobi rotations of the C++ filter's PrincipalEigenVector4; LAPACK's eigh is the
    independent yardstick."""
    rng = np.random.default_rng(3)
    q0 = rng.normal(size=4)
    q0 /= np.linalg.norm(q0)
    Q = q0 + 0.05 * rng.normal(size=(13, 4))
    Q /= np.linalg.norm(Q, axis=1)[:, None]
    Q[::2] *= -1                                          # q and -q are one rotation
    w = np.full(13, 1 / 12.0)
    w[-1] = 2.0                                           # the covariance weight of the nominal point (alpha 1, beta 2)
    K = sum(4 * w[i] * np.outer(Q[i], Q[i]) for i in range(13)) - w.sum() * np.eye(4)
    vals, vecs = np.linalg.eigh(K)
    ref = vecs[:, -1] * np.sign(vecs[:, -1] @ Q[-1])
    assert np.max(np.abs(quaternion_mean(Q, w, Q[-1]) - ref)) < 1e-10
    # rotations q0 exp(+-v_i / 2), symmetric about q0: the mean is q0
    from mujoco_mpc_b200.estimator import quat_integrate
    d = 0.1 * rng.normal(size=(6, 3))
    Qs = np.array([quat_integrate(q0, v, s) for s in (1.0, -1.0) for v in d] + [q0])
    assert np.max(np.abs(quaternion_mean(Qs, np.ones(13), q0) - q0)) < 1e-10


def _run_reference_test(name, backend_factory, q0, v0, T):
    """unscented_test.cc: filter T - 1 noise-free measurements; returns the max position / velocity errors."""
    m = load_estimator_model(name)
    X, Y, _ = simulate(m, m.qpos0 if q0 is None else q0, v0, T)
    f = Unscented(m, backend_factory(m))
    assert f.nsensordata == m.nsensordata and f.timestep == m.opt_timestep
    assert (f.weight_mean0, f.weight_covariance0) == (0.0, 2.0)
    f.reset(state=X[0], covariance_scale=1e-5, process_scale=1e-5, sensor_scale=1e-5)
    ep, ev = [], []
    for t in range(T - 1):
        f.update(np.zeros(m.nu), Y[t])
        if name == "box3drot":
            ep.append(np.linalg.norm(quat_error(m, f.state[:m.nq], X[t + 1, :m.nq])))
        else:
            ep.append(np.linalg.norm(f.state[:m.nq] - X[t + 1, :m.nq]))
        ev.append(np.linalg.norm(f.state[m.nq:] - X[t + 1, m.nq:]))
        assert np.allclose(f.covariance, f.covariance.T)
    assert f.time == pytest.approx((T - 1) * m.opt_timestep)
    return max(ep), max(ev)


CASES = [("particle1d", [0.25], [0.0], 5), ("box3drot", None, [1.0, -0.75, 1.25], 100)]


@pytest.mark.parametrize("name,q0,v0,T", CASES)
def test_reference_unscented_tests_on_fp64_oracle(name, q0, v0, T):
    ep, ev = _run_reference_test(name, lambda m: (lambda s, n, ts: OracleSigmaBackend(m, s, n, ts)),
                                 None if q0 is None else np.array(q0), np.array(v0), T)
    assert ep <= 1e-4 and ev <= 1e-4, (ep, ev)


def test_factorisation_failure_leaves_state_untouched():
    m = load_estimator_model("particle1d")
    f = Unscented(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts))
    f.reset(state=[0.25, 0.0])
    f.covariance = -np.eye(2)
    before = (f.state.copy(), f.covariance.copy(), f.time)
    with pytest.raises(EstimatorError, match="covariance factorisation"):
        f.update(np.zeros(1), [0.25, 0.0])
    assert np.array_equal(f.state, before[0]) and np.array_equal(f.covariance, before[1]) and f.time == before[2]
    # an indefinite sensor noise makes the sensor covariance indefinite: the second factor fails
    f.reset(state=[0.25, 0.0])
    f.noise_sensor[:] = -1.0
    before = (f.state.copy(), f.covariance.copy(), f.time)
    with pytest.raises(EstimatorError, match="sensor covariance factorisation"):
        f.update(np.zeros(1), [0.25, 0.0])
    assert np.array_equal(f.state, before[0]) and np.array_equal(f.covariance, before[1]) and f.time == before[2]


# ------------------------------------------------------------------------------------ sensors on the CPU oracle
from estimator_backends import FRAMES_XML, TOUCH_XML, settle, sensor_oracle  # noqa: E402
from quadruped_filtering import plant, run_filter  # noqa: E402


def test_sensor_oracle_against_numpy_restatement():
    """jointpos / jointvel / framepos of the sensor oracle (fp64, oracle kinematics) against sensors_fp64 (refmath
    kinematics): every framepos object type, at random states of a purpose-built scene and of the Humanoid (body
    framepos) and the Quadruped (site framepos, jointpos)."""
    from mujoco_mpc_b200.mjcf import SENS_FRAMEPOS
    rng = np.random.default_rng(2)
    fr = compile_xml(FRAMES_XML)
    assert {int(t) for t in fr.sensor_objtype[fr.sensor_type == SENS_FRAMEPOS]} == {0, 1, 2, 3}
    for m, start, count in ((fr, 0, fr.nsensor), (models.load("humanoid"), 5, 3), (models.load("quadruped"), 9, 17)):
        o = sensor_oracle(m)
        from estimator_backends import mocap_vector
        mc = mocap_vector(m)
        for _ in range(4):
            q = m.qpos0 + 0.2 * rng.normal(size=m.nq)
            v = rng.normal(size=m.nv)
            r = o.step(q[None], v[None], np.zeros((1, m.nu)), mc, [0.0], start, count)
            ref = sensors_fp64(m, q, v, start, count, mc)
            assert np.max(np.abs(r["sensordata"][0] - ref)) < 1e-12


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_touch_on_the_oracle_scenes(cone):
    """A 1 kg ball at rest on a plane: the contact point inside the zone and the ray into the ball hitting the zone
    read m |g| (to the solver tolerance); a zone beside the ray and a zone of another body that contains the contact
    point read 0; a box zone is refused."""
    m = compile_xml(TOUCH_XML.format(cone=cone))
    o = sensor_oracle(m)
    x, w = settle(lambda x, w, t: o.step(x[None, :m.nq], x[None, m.nq:], np.zeros((1, 0)), mocap_of_scene(m), [t], 0, 4,
                                         warmstart=w), m, 500, 0.002)
    r = o.step(x[None, :m.nq], x[None, m.nq:], np.zeros((1, 0)), mocap_of_scene(m), [0.0], 0, 4, warmstart=w)
    y, g = r["sensordata"][0], np.linalg.norm(m.opt_gravity)
    assert r["ncon"][0] == 1
    assert abs(y[0] - g) < 1e-6 * g and abs(y[1] - g) < 1e-6 * g and y[2] == 0 and y[3] == 0, y
    with pytest.raises(ValueError):
        o.step(x[None, :m.nq], x[None, m.nq:], np.zeros((1, 0)), mocap_of_scene(m), [0.0], 0, 5)


def mocap_of_scene(m):
    from estimator_backends import mocap_vector
    return mocap_vector(m)


def test_touch_rest_weight_on_the_oracle():
    """The A1 settled on its feet by a joint PD law: the four foot touch sensors read its weight.  The contact point
    of foot and floor lies below the r = 0.015 site zone, so the ray rule is what makes them read."""
    m = models.load("quadruped")
    o = sensor_oracle(m, 0.005)
    k = m.key_names.index("home")
    home = m.key_qpos[k]
    mc = mocap_of_scene(m)

    def step(x, w, t, start=26, count=4):
        u = np.clip(2.0 * (home[7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:], -1, 1)
        return o.step(x[None, :m.nq], x[None, m.nq:], u[None], mc, [t], start, count, warmstart=w)
    x = np.concatenate([home, np.zeros(m.nv)])
    x, w = settle(step, m, 300, 0.005, x)
    y = step(x, w, 0.0)["sensordata"][0]
    weight = m.body_subtreemass[m.body_names.index("trunk")] * np.linalg.norm(m.opt_gravity)
    assert (y > 0).all() and abs(y.sum() - weight) < 1e-4 * weight, (y, weight)


def test_quadruped_filtering_bar_on_the_oracles():
    """The Quadruped scenario (tests/quadruped_filtering.py) with the sigma points on the fp64 and on the fp32 oracle:
    the two filters' RMS errors agree to 1e-3 relative, so fp32 sigma-point steps cost the filter nothing measurable,
    and the engine-backed filters are held to the fp32-oracle filter's errors + 5 % (tests/test_gpu_estimator.py)."""
    m = models.load("quadruped")
    X, Y, U = plant(m)
    res = {}
    for prec in (64, 32):
        f = Unscented(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, precision=prec))
        res[prec] = run_filter(m, f, X, Y, U, mocap_of_scene(m))
        assert res[prec][2] == 0.0 and res[prec][3] > 0 and f.warnings == 0
    assert abs(res[32][0] - res[64][0]) < 1e-3 * res[64][0] and abs(res[32][1] - res[64][1]) < 1e-3 * res[64][1], res
    assert res[64][0] < 2e-3, res                      # the estimate follows the plant to a few mm / mrad
