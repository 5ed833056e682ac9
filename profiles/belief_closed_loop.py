"""Does planning over the state estimate's uncertainty lower closed-loop cost?  B Quadruped plants with measurement
noise on the filter's sensors (CppPlantBank.set_sensor_noise), a Kalman bank estimating each plant's state from those
sensors, and a CppBatchSamplingPlanner planning from the filter's state (closed_loop.synchronous_planning_cost), in
three arms:

  mean       the planner plans from the filter's mean state (no state ensemble)
  expected   every candidate scored over K = 4 states drawn from the filter's covariance, worst = K (the mean return)
  worst      the same members, worst = 1 (the worst member)

Reported per arm: each plant's average cost per step, their mean, the plants that diverged and the aggregate
x-realtime.  One seed, not a significance test; whatever comes out is reported.  One JSON line per arm, after a line
with the GPU's name and power limit.
Usage: python profiles/belief_closed_loop.py [--plants 8] [--steps 300] [--N 64] [--H 36] [--noise 0.02] [--seed 3]"""
import argparse
import json
import os
import sys

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, mocap_of  # noqa: E402

from mujoco_mpc_b200.closed_loop import synchronous_planning_cost  # noqa: E402
from mujoco_mpc_b200.engine import PLANT_DIVERGED, CppBatchSamplingPlanner, CppPlantBank  # noqa: E402
from mujoco_mpc_b200.estimator import CppBatchEstimator  # noqa: E402


def run_arm(m, K, worst, args):
    B = args.plants
    pl = CppBatchSamplingPlanner(m, B, args.N, args.H, seeds=[0x5EED + b for b in range(B)])
    if K:
        pl.set_state_ensemble(K, worst=worst, seed=args.seed)
    est = CppBatchEstimator(m, "kalman", B, timestep=m.opt_timestep)
    bank = CppPlantBank(m, B, sensor_start=est.sensor_start, nsensor=est.nsensor)
    rng = np.random.default_rng(args.seed)
    q0, mc = np.asarray(m.key_qpos[0], float), mocap_of(m)
    for b in range(B):
        v = 0.05 * rng.standard_normal(m.nv)
        pl.reset(b)
        bank.reset(b, q0, v, 0.0, mc)
        bank.set_disturbance(b, seed=100 + b)
        bank.set_sensor_noise(b, args.noise)
        est.reset(b, state=np.concatenate([q0, v]), time=0.0)
    out = synchronous_planning_cost(pl, bank, args.steps, 4, estimator=est)
    pl.close(); bank.close(); est.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plants", type=int, default=8)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--N", type=int, default=64)
    ap.add_argument("--H", type=int, default=36)
    ap.add_argument("--noise", type=float, default=0.02)
    ap.add_argument("--seed", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("belief_closed_loop.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    m = get_model("quadruped")
    for arm, K, worst in (("mean", 0, None), ("expected", 4, 4), ("worst", 4, 1)):
        o = run_arm(m, K, worst, args)
        avg = np.asarray(o["average_cost"], float)
        print(json.dumps({"arm": arm, "plants": args.plants, "N": args.N, "H": args.H, "steps": args.steps,
                          "sensor_noise_std": args.noise, "steps_per_planning_iteration": 4,
                          "average_cost": avg.round(5).tolist(), "mean_average_cost": float(avg.mean()),
                          "diverged": int(np.sum(np.asarray(o["final_status"]) == PLANT_DIVERGED)),
                          "x_realtime": float(o["x_realtime"]), "wall_s": float(o["wall_time"]),
                          "planning_s": float(o["planning_time"])}), flush=True)


if __name__ == "__main__":
    main()
