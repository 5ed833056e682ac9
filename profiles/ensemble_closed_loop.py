"""Does planning on a model ensemble make closed-loop MPC robust to a wrong model?  B plants, each on a held-out
Quadruped variant drawn from a seeded range (trunk mass x [0.7, 1.3], foot friction x [0.6, 1.2]), each driven by its
problem of a CppBatchSamplingPlanner (closed_loop.synchronous_planning_cost on a CppPlantBank), in three arms:

  nominal    the planner plans on the nominal model
  expected   the planner scores every candidate on a K = 4 ensemble at the corners of the range, worst = K (the mean)
  worst      the same ensemble, worst = 1 (the worst member)

Reported per arm: each plant's average cost per step, their mean, the plants that diverged and the aggregate
x-realtime (B x simulated seconds / wall time).  Whatever comes out is reported, a gain or none.  One JSON line per arm,
after a line with the GPU's name and power limit and one with the plants' parameters.
Usage: python profiles/ensemble_closed_loop.py [--plants 8] [--steps 300] [--N 60] [--H 36] [--seed 3]"""
import argparse
import json
import os
import sys

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, mocap_of  # noqa: E402
from test_gpu_model_variants import _sub, _variant  # noqa: E402

from mujoco_mpc_b200.closed_loop import synchronous_planning_cost  # noqa: E402
from mujoco_mpc_b200.engine import PLANT_DIVERGED, CppBatchSamplingPlanner, CppPlantBank  # noqa: E402

MASS, FRICTION = 4.713, 0.8


def quadruped(mass_scale, friction_scale):
    def edit(x):
        x = _sub(x, f'<inertial mass="{MASS}"', f'<inertial mass="{MASS * mass_scale:.6g}"')
        return _sub(x, f'friction="{FRICTION} 0.02 0.01"', f'friction="{FRICTION * friction_scale:.6g} 0.02 0.01"')
    return _variant("quadruped", edit)


def run_arm(base, plants, members, worst, N, H, steps, seeds):
    B = len(plants)
    pl = CppBatchSamplingPlanner(base, B, N, H, seeds=seeds)
    bank = CppPlantBank(base, B)
    bank.set_models(plants)
    if members:
        pl.set_ensemble(members, worst=worst)
    q0, mc = base.key_qpos[0], mocap_of(base)
    for b in range(B):
        pl.reset(b); bank.reset(b, q0, np.zeros(base.nv), 0.0, mc)
    out = synchronous_planning_cost(pl, bank, steps, 4)
    pl.close(); bank.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plants", type=int, default=8)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--N", type=int, default=60)
    ap.add_argument("--H", type=int, default=36)
    ap.add_argument("--seed", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ensemble_closed_loop.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    rng = np.random.default_rng(args.seed)
    scales = np.stack([rng.uniform(0.7, 1.3, args.plants), rng.uniform(0.6, 1.2, args.plants)], 1)
    print(json.dumps({"plants": {"trunk_mass_scale": scales[:, 0].round(4).tolist(),
                                 "foot_friction_scale": scales[:, 1].round(4).tolist()}}), flush=True)
    base = get_model("quadruped")
    plants = [quadruped(m, f) for m, f in scales]
    corners = [quadruped(m, f) for m in (0.7, 1.3) for f in (0.6, 1.2)]
    seeds = [0x5EED + b for b in range(args.plants)]
    for arm, members, worst in (("nominal", None, None), ("expected", corners, 4), ("worst", corners, 1)):
        o = run_arm(base, plants, members, worst, args.N, args.H, args.steps, seeds)
        avg = np.asarray(o["average_cost"], float)
        print(json.dumps({"arm": arm, "plants": args.plants, "N": args.N, "H": args.H, "steps": args.steps,
                          "steps_per_planning_iteration": 4, "average_cost": avg.round(5).tolist(),
                          "mean_average_cost": float(avg.mean()),
                          "diverged": int(np.sum(np.asarray(o["final_status"]) == PLANT_DIVERGED)),
                          "x_realtime": float(o["x_realtime"]), "wall_s": float(o["wall_time"]),
                          "planning_s": float(o["planning_time"])}), flush=True)


if __name__ == "__main__":
    main()
