"""Kernel time of the magnetometer and rangefinder on the device.

  * step_sensors, 64 rows: one launch of existing sensor types (the Quadruped's 21 estimator sensors; on Humanoid
    Track the 14 sensors tests/sensor_scenes.py adds), and the same launch with the magnetometers and rangefinders of
    tests/test_gpu_range_magnet_sensors.py appended to that range (a magnetometer and a rangefinder on the trunk or
    pelvis, rangefinders on the feet);
  * plant step, B = 256 Quadruped plants: one plant-bank step without sensors, with the 21 existing sensors, and with
    them plus the new ones.
Each time is the median of the launches' CUDA-event kernel times (last_kernel_ms) after warm-up launches of the same
shape.  The GPU's name and power limit are read in the same run.

usage: python profiles/time_range_sensors.py [--calls 200] [--warmup 20] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from estimator_backends import mocap_vector  # noqa: E402
from time_sensors import _Patch, gpu_description  # noqa: E402

from mujoco_mpc_b200.engine import CppPlantBank, Engine  # noqa: E402


def _median(fn, timer, calls, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(calls):
        fn()
        ts.append(timer())
    return float(np.median(ts))


def time_step_sensors(m, start, count, calls, warmup, rows=64):
    e = Engine(m, rows, 8, device=0)
    x = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    X = np.repeat(x[None], rows, axis=0)
    u, mc = np.zeros(m.nu), mocap_vector(m)
    ms = _median(lambda: e.step_sensors(X, u, mc, 0.0, start, count), lambda: e.last_kernel_ms, calls, warmup)
    e.close()
    return ms


def time_plant(m, start, count, calls, warmup, B=256):
    bank = CppPlantBank(m, B, sensor_start=start, nsensor=count)
    home = m.key_qpos[m.key_names.index("home")]
    for b in range(B):
        bank.reset(b, home, np.zeros(m.nv), 0.0)
    u = np.zeros((B, m.nu), np.float32)
    ms = _median(lambda: bank.step(u), bank.last_kernel_ms, calls, warmup)
    bank.close()
    return ms


def main():
    from sensor_scenes import HUMANOID_SENSORS, load_augmented
    from test_gpu_range_magnet_sensors import HUMANOID_EXTRA, _load
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"gpu": gpu_description()}
    # the Quadruped's estimator sensors are [9, nsensor); the new ones are appended right after them
    qr, qstart, qcount = _load("quadruped", _Patch())
    base = qstart - 9
    res["quadruped_step_sensors_%d_ms" % base] = time_step_sensors(qr, 9, base, a.calls, a.warmup)
    res["quadruped_step_sensors_%d+%d_ms" % (base, qcount)] = time_step_sensors(qr, 9, base + qcount, a.calls, a.warmup)
    # Humanoid Track: the existing-type sensors of tests/sensor_scenes.py, then the new ones after them
    hr, hstart, hcount = load_augmented("humanoid_track", _Patch(), extra=HUMANOID_SENSORS + HUMANOID_EXTRA)
    hbase = hcount - HUMANOID_EXTRA.count("<")
    res["humanoid_track_step_sensors_%d_ms" % hbase] = time_step_sensors(hr, hstart, hbase, a.calls, a.warmup)
    res["humanoid_track_step_sensors_%d+%d_ms" % (hbase, hcount - hbase)] = time_step_sensors(hr, hstart, hcount, a.calls,
                                                                                             a.warmup)
    res["quadruped_plant_B256_nosensors_ms"] = time_plant(qr, 0, 0, a.calls, a.warmup)
    res["quadruped_plant_B256_%d_ms" % base] = time_plant(qr, 9, base, a.calls, a.warmup)
    res["quadruped_plant_B256_%d+%d_ms" % (base, qcount)] = time_plant(qr, 9, base + qcount, a.calls, a.warmup)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "a") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
