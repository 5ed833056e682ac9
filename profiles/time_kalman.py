"""Time one Kalman filter update (mujoco_mpc_b200.estimator.Kalman: update_measurement + update_prediction, two
launches) with its finite-difference steps on the engine, for the Quadruped (21 sensors; 73 states per launch centred,
37 one-sided) and the reference's task_imu particle (jointpos + accelerometer; 5 / 3 states).

Per case: the wall time of `update` (host clock around the call; each launch ends in a stream synchronise) and
`last_kernel_ms` of its prediction launch (CUDA events), medians over the timed updates; the GPU's name and power limit
are read in the same run.  The same updates with the fp64 CPU oracle as the backend are timed too, labelled as the
oracle: this project's CPU reference, not MuJoCo.

usage: python profiles/time_kalman.py [--updates 200] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from estimator_backends import OracleSigmaBackend, mocap_vector  # noqa: E402
from test_kalman_cpu import load_task_imu  # noqa: E402
from time_unscented import gpu_description  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.engine import Engine  # noqa: E402
from mujoco_mpc_b200.estimator import EngineBackend, Kalman  # noqa: E402


def run(m, backend, updates, warmup, centered):
    f = Kalman(m, backend, centered=centered)
    x0 = f.state.copy()
    mc = mocap_vector(m)
    u = np.zeros(m.nu)
    # the measurement of the reset state: a filter that sits on the truth (the time is the work, not the estimate)
    _, ys, _, _ = f.backend.step_sensors(x0[None], u, mc, 0.0, None)
    wall, kern = [], []
    for i in range(warmup + updates):
        f.reset(state=x0)
        t0 = time.perf_counter()
        f.update(u, ys[0], mc)
        t1 = time.perf_counter()
        if i >= warmup:
            wall.append((t1 - t0) * 1e3)
            if hasattr(f.backend, "last_kernel_ms"):
                kern.append(f.backend.last_kernel_ms)
    out = dict(states_per_launch=f.nstates, nsensordata=f.nsensordata, updates=updates,
               update_ms_median=float(np.median(wall)), update_ms_p90=float(np.percentile(wall, 90)))
    if kern:
        out["kernel_ms_median"] = float(np.median(kern))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--oracle-updates", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = dict(gpu=gpu_description(), results={})
    for name, m in (("quadruped", models.load("quadruped")), ("task_imu", load_task_imu())):
        for centered in (True, False):
            key = "%s/%s" % (name, "centred" if centered else "one-sided")
            e = Engine(m, 2 * 2 * m.nv + 1, 8, device=0)
            res["results"][key + "/engine"] = run(m, lambda s, n, ts: EngineBackend(e, s, n, ts), a.updates, 10,
                                                  centered)
            e.close()
            res["results"][key + "/fp64 CPU oracle"] = run(
                m, lambda s, n, ts: OracleSigmaBackend(m, s, n, ts), a.oracle_updates, 2, centered)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_kalman.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
