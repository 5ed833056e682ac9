"""Record every output of the Unscented and Kalman filters (for bitwise comparison of builds): state, covariance, time
and warnings after every update, and the error of a failed sensor-covariance factorisation.

  python profiles/dump_estimators.py out.npz [--backend oracle|engine] [--updates 40]
  python profiles/dump_estimators.py --cmp a.npz b.npz

Filters: Unscented, Kalman centred and Kalman one-sided.  --backend oracle runs the Python mirrors on the fp64 CPU
oracle (OracleSigmaBackend, no GPU); --backend engine runs CppUnscented / CppKalman, the Python mirrors on
EngineBackend and a CppBatchEstimator of 3 filters with distinct start velocities, sensor noises and sensors (its
failure path: filter 1's sensor noise negative, the statuses and every filter after the update).  Scenes: the
reference's particle1d and box3drot, task_imu, and the Quadruped filtering scenario of tests/quadruped_filtering.py.
The archive is written with fixed zip timestamps, so equal outputs give equal files.
"""
import argparse
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def compare(a, b):
    a, b = np.load(a), np.load(b)
    same = a.files == b.files
    if not same:
        print("keys differ:", sorted(set(a.files) ^ set(b.files)))
    for k in a.files:
        if k not in b.files:
            continue
        x, y = a[k], b[k]
        if x.shape == y.shape and x.tobytes() == y.tobytes():
            continue
        same = False
        print("%-50s differs" % k + ("" if x.dtype.kind in "US" or x.shape != y.shape else
                                      ", max abs %.3g" % np.abs(x - y).max()))
    print("%d arrays, %s" % (len(a.files), "all bitwise equal" if same else "DIFFERENT"))
    return 0 if same else 1


def save(path, arrays):
    with zipfile.ZipFile(path, "w") as z:
        for k, v in arrays.items():
            with z.open(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), "w") as fh:
                np.lib.format.write_array(fh, np.asarray(v))


def scenes(updates):
    from estimator_backends import load_estimator_model, mocap_vector, simulate
    from quadruped_filtering import SENSOR_SD, plant
    from test_kalman_cpu import load_task_imu

    from mujoco_mpc_b200 import models
    for name, m in (("particle1d", load_estimator_model("particle1d")), ("box3drot", load_estimator_model("box3drot"))):
        X, Y, U = simulate(m, m.qpos0, np.full(m.nv, 0.1), updates + 1)
        yield name, m, X, Y, U, mocap_vector(m), None
    m = load_task_imu()
    X, Y, U = simulate(m, [0.25], [0.0], updates + 1)
    yield "task_imu", m, X, Y, U, mocap_vector(m), None
    m = models.load("quadruped")
    X, Y, U = plant(m)
    yield "quadruped", m, X, Y, U, mocap_vector(m), SENSOR_SD ** 2


def record(out, key, f, m, X, Y, U, mocap, sensor_variance, updates):
    f.reset(state=X[0])
    if sensor_variance is not None:
        f.set_noise(sensor=np.full(f.nsensordata, sensor_variance))
    S, P, T, W = [], [], [], []
    for t in range(updates):
        f.update(U[t], Y[t], mocap)
        S.append(f.state); P.append(f.covariance); T.append(f.time); W.append(f.warnings)
    out[key + "/state"], out[key + "/covariance"] = np.array(S), np.array(P)
    out[key + "/time"], out[key + "/warnings"] = np.array(T), np.array(W)
    # the failure path: a negative sensor noise variance, nothing updated
    from mujoco_mpc_b200.estimator import EstimatorError
    f.set_noise(sensor=np.full(f.nsensordata, -1.0))
    try:
        f.update(U[updates], Y[updates], mocap)
        out[key + "/error"] = np.array("no error")
    except EstimatorError as e:
        out[key + "/error"] = np.array(str(e))
    out[key + "/after_error"] = np.concatenate([f.state, f.covariance.ravel(), [f.time, f.warnings]])


def record_batch(out, key, f, m, X, Y, U, mocap, sensor_variance, updates):
    B = f.num_filters
    var = 1e-4 if sensor_variance is None else sensor_variance
    for b in range(B):
        x0 = X[0].copy()
        x0[m.nq:] += 1e-3 * b
        f.reset(b, state=x0)
        f.set_noise(b, sensor=np.full(f.nsensordata, var * (1 + b)))
    mc = np.tile(mocap, (B, 1)) if mocap.size else None
    S, P, T, W = [], [], [], []
    for t in range(updates + 1):
        if t == updates:   # the failure path: filter 1's sensor noise negative
            f.set_noise(1, sensor=np.full(f.nsensordata, -1.0))
        y = np.stack([Y[t] + 1e-4 * b for b in range(B)])
        status = f.update(np.tile(U[t], (B, 1)), y, mc)
        got = [f.get(b) for b in range(B)]
        S.append([g[0] for g in got]); P.append([g[1] for g in got])
        T.append([g[2] for g in got]); W.append([g[3][3] for g in got])
    out[key + "/state"], out[key + "/covariance"] = np.array(S), np.array(P)
    out[key + "/time"], out[key + "/warnings"] = np.array(T), np.array(W)
    out[key + "/status_after_error"] = status


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--cmp", nargs=2)
    ap.add_argument("--backend", choices=("oracle", "engine"), default="oracle")
    ap.add_argument("--updates", type=int, default=40)
    a = ap.parse_args()
    if a.cmp:
        sys.exit(compare(*a.cmp))
    from estimator_backends import OracleSigmaBackend

    from mujoco_mpc_b200.estimator import Kalman, Unscented
    out = {}
    for name, m, X, Y, U, mocap, var in scenes(a.updates):
        kinds = (("unscented", Unscented, {}), ("kalman_centred", Kalman, dict(centered=True)),
                 ("kalman_one_sided", Kalman, dict(centered=False)))
        if a.backend == "oracle":
            for fname, cls, kw in kinds:
                f = cls(m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts), **kw)
                record(out, "python/%s/%s" % (fname, name), f, m, X, Y, U, mocap, var, a.updates)
            continue
        from mujoco_mpc_b200.engine import Engine
        from mujoco_mpc_b200.estimator import CppBatchEstimator, CppKalman, CppUnscented, EngineBackend
        e = Engine(m, 2 * 2 * m.nv + 1, 8, device=0)
        for fname, cls, kw in kinds:
            f = cls(m, lambda s, n, ts: EngineBackend(e, s, n, ts), **kw)
            record(out, "python/%s/%s" % (fname, name), f, m, X, Y, U, mocap, var, a.updates)
            f = (CppUnscented if cls is Unscented else CppKalman)(m, **kw)
            record(out, "cpp/%s/%s" % (fname, name), f, m, X, Y, U, mocap, var, a.updates)
            f.close()
            f = CppBatchEstimator(m, "unscented" if cls is Unscented else "kalman", 3, **kw)
            record_batch(out, "batch/%s/%s" % (fname, name), f, m, X, Y, U, mocap, var, a.updates)
            f.close()
        e.close()
    save(a.out, out)
    print("%d arrays written to %s" % (len(out), a.out))


if __name__ == "__main__":
    main()
