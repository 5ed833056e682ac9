"""Time one Unscented filter update (mujoco_mpc_b200.estimator) with its sigma-point steps on the engine, for the
Quadruped (21 sensors, 73 sigma points) and the reference's Box3Drot (8 framepos sensors, 13 points).

Per model: the wall time of `update` (host clock around the call; the sigma-point launch ends in a stream synchronise)
and `last_kernel_ms` of that launch (CUDA events), medians over the timed updates; the GPU's name and power limit are
read in the same run.  The same updates with the fp64 CPU oracle as the sigma-point backend are timed too, labelled
as the oracle: this project's CPU reference, not MuJoCo.

usage: python profiles/time_unscented.py [--updates 200] [--out DIR]
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

from estimator_backends import OracleSigmaBackend, load_estimator_model, mocap_vector  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.engine import Engine  # noqa: E402
from mujoco_mpc_b200.estimator import EngineBackend, Unscented  # noqa: E402


def gpu_description():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(m, backend, updates, warmup, **settings):
    f = Unscented(m, backend, **settings)
    x0 = f.state.copy()
    mc = mocap_vector(m)
    u = np.zeros(m.nu)
    # the measurement of the nominal state: a filter that sits on the truth (the time is the work, not the estimate)
    y = None
    wall, kern = [], []
    for i in range(warmup + updates):
        if y is None:
            _, ys, _, _ = f.backend.step_sensors(x0[None], u, mc, 0.0, None)
            y = ys[0]
        t0 = time.perf_counter()
        f.update(u, y, mc)
        t1 = time.perf_counter()
        if i >= warmup:
            wall.append((t1 - t0) * 1e3)
            if hasattr(f.backend, "last_kernel_ms"):
                kern.append(f.backend.last_kernel_ms)
    out = dict(nsigma=f.nsigma, nsensordata=f.nsensordata, updates=updates, update_ms_median=float(np.median(wall)),
               update_ms_p90=float(np.percentile(wall, 90)))
    if kern:
        out["sigma_kernel_ms_median"] = float(np.median(kern))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--oracle-updates", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(gpu=gpu_description(), results={})
    for name, m in (("quadruped", models.load("quadruped")), ("box3drot", load_estimator_model("box3drot"))):
        e = Engine(m, 128, 8, device=0)
        res["results"][name + "/engine"] = run(m, lambda s, n, ts: EngineBackend(e, s, n, ts), a.updates, 10)
        e.close()
        if name == "quadruped":
            continue   # the oracle backend does not evaluate touch
        res["results"][name + "/fp64 CPU oracle"] = run(
            m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, nthreads=1), a.oracle_updates, 2)
    # the Quadruped on the oracle without its touch sensors (framepos + jointpos, 17 of the 21)
    m = models.load("quadruped")
    res["results"]["quadruped (no touch)/fp64 CPU oracle"] = run(
        m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts, nthreads=1), a.oracle_updates, 2, sensor_start=9, nsensor=17)
    e = Engine(m, 128, 8, device=0)
    res["results"]["quadruped (no touch)/engine"] = run(m, lambda s, n, ts: EngineBackend(e, s, n, ts), a.updates, 10,
                                                          sensor_start=9, nsensor=17)
    e.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_unscented.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
