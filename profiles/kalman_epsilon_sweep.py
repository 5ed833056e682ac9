"""Choose the Kalman filter's finite differences for fp32 steps (CPU only, no GPU).

The reference's 1e-6 one-sided differences are an fp64 setting: on fp32 steps a 1e-6 perturbation is a few ulps of the
state.  This sweeps centred and one-sided differences over epsilon on the fp32 sensor oracle (the yardstick of the
engine's fp32 kernels) in the two scenarios of the tests, next to the fp64 oracle at the reference's setting:

  task_imu   the reference's Kalman test (tests/test_kalman_cpu.py): max qpos / qvel error norm after each measurement
  quadruped  tests/quadruped_filtering.py: RMS qpos / qvel error over steps 50 .. 199 and the smallest covariance
             eigenvalue

    python profiles/kalman_epsilon_sweep.py [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from estimator_backends import OracleSigmaBackend, mocap_vector  # noqa: E402
from quadruped_filtering import plant, run_filter  # noqa: E402
from test_kalman_cpu import load_task_imu, reference_kalman_test  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.estimator import Kalman  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--eps", default="1e-4,3e-4,1e-3,3e-3")
    a = ap.parse_args()
    imu, quad = load_task_imu(), models.load("quadruped")
    X, Y, U = plant(quad)
    mc = mocap_vector(quad)
    settings = [(64, 1e-6, False)] + [(32, float(e), c) for c in (True, False) for e in a.eps.split(",")]
    rows = []
    for prec, eps, centered in settings:
        ep, ev = reference_kalman_test(imu, lambda s, n, ts: OracleSigmaBackend(imu, s, n, ts, precision=prec),
                                       epsilon=eps, centered=centered)
        f = Kalman(quad, lambda s, n, ts: OracleSigmaBackend(quad, s, n, ts, precision=prec), epsilon=eps,
                   centered=centered)
        rq, rv, asym, mineig = run_filter(quad, f, X, Y, U, mc)
        row = dict(precision=prec, epsilon=eps, centered=centered, task_imu_max_qpos=float(ep.max()),
                   task_imu_max_qvel=float(ev.max()), quadruped_rms_qpos=rq, quadruped_rms_qvel=rv,
                   quadruped_min_eig=mineig, quadruped_warnings=f.warnings)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
