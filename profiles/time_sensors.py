"""Time the measurement-sensor stage: mjpc_b200_step_sensors launches and one Unscented filter-bank update.

  * quadruped21: one step_sensors launch of the Quadruped's 21 estimator sensors (5 framepos, 12 jointpos, 4 touch),
    64 rows;
  * quadruped+new / humanoid_track+new / shadow_reorient+new: the same launch of the sensors tests/sensor_scenes.py
    adds to copies of the shipped models (every frame, subtree, ball-joint, actuator and tendon type), 64 rows;
  * unscented_imu B=1 / B=64: one update of a bank of B Unscented filters on the free-flying IMU body of
    tests/sensor_scenes.py (framepos, framequat, gyro, accelerometer).
Each time is the median over the timed calls of the host clock around the call (each call ends in a stream
synchronise), after warm-up calls of the same shape; every timed filter update starts from the same reset state.  The GPU's name and power limit are read in the same run.
With --base-only only quadruped21 is timed (a library without the new sensor types).

usage: python profiles/time_sensors.py [--calls 200] [--warmup 20] [--base-only] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from estimator_backends import mocap_vector  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.engine import Engine  # noqa: E402


def gpu_description():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def _median_ms(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def time_step_sensors(m, start, count, calls, warmup, rows=64):
    e = Engine(m, rows, 8, device=0)
    k = 0
    x = np.concatenate([m.key_qpos[k], np.zeros(m.nv)])
    X = np.repeat(x[None], rows, axis=0)
    u, mc = np.zeros(m.nu), mocap_vector(m)
    ms = _median_ms(lambda: e.step_sensors(X, u, mc, 0.0, start, count), calls, warmup)
    e.close()
    return ms


class _Patch:
    """monkeypatch.setattr for a script"""
    def setattr(self, obj, name, value):
        setattr(obj, name, value)


def time_unscented(B, calls, warmup):
    from sensor_scenes import ROTATIONS, imu_body
    from mujoco_mpc_b200.estimator import CppBatchEstimator
    m = imu_body(ROTATIONS[3])
    f = CppBatchEstimator(m, "unscented", B)
    x0 = np.concatenate([m.qpos0, 0.1 * np.ones(m.nv)])
    for b in range(B):
        f.reset(b, state=x0)
        f.set_noise(b, sensor=np.full(f.nsensordata, 1e-6))
    u, y = np.zeros((B, m.nu)), np.tile(np.concatenate([x0[:3], [1, 0, 0, 0], np.zeros(6)]), (B, 1))

    ts = []
    for i in range(warmup + calls):
        for b in range(B):
            f.reset(b, state=x0)      # every timed update starts from the same filter state
        t0 = time.perf_counter()
        f.update(u, y, None)
        if i >= warmup:
            ts.append(1e3 * (time.perf_counter() - t0))
    f.close()
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--base-only", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"gpu": gpu_description()}
    q = models.load("quadruped")
    res["quadruped21_ms"] = time_step_sensors(q, 9, 21, a.calls, a.warmup)
    if not a.base_only:
        from sensor_scenes import load_augmented
        for name in ("quadruped", "humanoid_track", "shadow_reorient"):
            m, start, count = load_augmented(name, _Patch())
            res[name + "+new_ms"] = time_step_sensors(m, start, count, a.calls, a.warmup)
            res[name + "+new_nsensor"] = count
        for B in (1, 64):
            res["unscented_imu_B%d_ms" % B] = time_unscented(B, a.calls, a.warmup)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "a") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
