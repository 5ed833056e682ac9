"""The Kalman filter's finite-difference Jacobians on the free-flying IMU body of tests/sensor_scenes.py, per sensor
block, from the fp32 sensor oracle and (with --device) from the engine, against the fp64 oracle's.

Along the fp64-oracle Kalman filter's run on the IMU plant (imu_plant), at every --every-th update the filter's perturbed
states (Kalman.perturbed: 2 * 2 nv + 1 rows at epsilon 1e-3) are stepped by each backend; the measurement Jacobian C
(sensors by tangent state) is split into the framepos, framequat, gyro and accelerometer rows, the transition Jacobian
A (next tangent state by tangent state) into its position and velocity rows, and for each block the largest
|J - J_fp64| is printed, with the largest |J_fp64| of the block for scale.  Then the RMS error of the filter on each
backend, as tests/test_gpu_sensors.py measures it.

usage: python profiles/kalman_imu_jacobians.py [--device] [--every 10] [--steps 60]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from estimator_backends import OracleSigmaBackend  # noqa: E402
from sensor_scenes import ROTATIONS, imu_body, imu_plant  # noqa: E402

from mujoco_mpc_b200.estimator import EngineBackend, Kalman, differentiate_pos  # noqa: E402

BLOCKS = (("framepos", 0, 3), ("framequat", 3, 7), ("gyro", 7, 10), ("accelerometer", 10, 13))


def jacobians(f, backend, ctrl):
    """(C, A) of filter f's current state through backend, as Kalman.update_measurement / update_prediction form them"""
    m = f.m
    X = f.perturbed()
    warm = np.tile(f.qacc_warmstart, (len(X), 1))
    nxt, y, _, _ = backend.step_sensors(X, np.asarray(ctrl, float), np.zeros(0), f.time, warm)
    n, h = f.ndstate, 2 * f.epsilon
    C = np.stack([(y[1 + i] - y[1 + n + i]) / h for i in range(n)], axis=1)
    A = np.stack([np.concatenate([differentiate_pos(m, nxt[1 + n + i, :m.nq], nxt[1 + i, :m.nq]),
                                  nxt[1 + i, m.nq:] - nxt[1 + n + i, m.nq:]]) / h for i in range(n)], axis=1)
    return C, A


def filter_rms(m, f, X, Y, U, T):
    f.reset(state=X[0])
    f.set_noise(sensor=np.full(f.nsensordata, 1e-6))
    e = []
    for t in range(T):
        f.update(U[t], Y[t], np.zeros(0))
        e.append(np.concatenate([f.state[:3] - X[t + 1, :3], f.state[m.nq:] - X[t + 1, m.nq:]]))
    return float(np.sqrt(np.mean(np.square(e[T // 4:]))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", action="store_true")
    ap.add_argument("--every", type=int, default=10)
    ap.add_argument("--steps", type=int, default=60)
    a = ap.parse_args()
    m = imu_body(ROTATIONS[3])
    X, Y, U = imu_plant(m, a.steps)
    backends = {p: (lambda s, n, ts, p=p: OracleSigmaBackend(m, s, n, ts, p)) for p in (64, 32)}
    if a.device:
        from mujoco_mpc_b200.engine import Engine
        e = Engine(m, 64, 8, device=0)
        backends["device"] = lambda s, n, ts: EngineBackend(e, s, n, ts)
    f = Kalman(m, backends[64])
    f.reset(state=X[0])
    f.set_noise(sensor=np.full(f.nsensordata, 1e-6))
    others = {k: b(f.sensor_start, f.nsensor, f.timestep) for k, b in backends.items()}
    nv = m.nv
    for t in range(a.steps):
        if t % a.every == 0:
            C64, A64 = jacobians(f, others[64], U[t])
            row = {"update": t}
            for k in others:
                if k == 64:
                    continue
                C, A = jacobians(f, others[k], U[t])
                for name, r0, r1 in BLOCKS:
                    row["C %s %s" % (name, k)] = float(np.abs(C[r0:r1] - C64[r0:r1]).max())
                row["A pos %s" % k] = float(np.abs(A[:nv] - A64[:nv]).max())
                row["A vel %s" % k] = float(np.abs(A[nv:] - A64[nv:]).max())
            for name, r0, r1 in BLOCKS:
                row["|C %s|" % name] = float(np.abs(C64[r0:r1]).max())
            print(json.dumps(row))
        f.update(U[t], Y[t], np.zeros(0))
    rms = {k: filter_rms(m, Kalman(m, b), X, Y, U, a.steps) for k, b in backends.items()}
    print(json.dumps({"kalman RMS": {str(k): v for k, v in rms.items()}}))


if __name__ == "__main__":
    main()
