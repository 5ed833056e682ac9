"""Does the Robust planner hold a disturbed plant better than the Sampling planner?  B Quadruped plants on the flat
task (closed_loop.synchronous_planning_cost on a CppPlantBank, a plan every step), each under Ornstein-Uhlenbeck
body-force noise with its own seed (CppPlantBank.set_disturbance), and every plant pushed sideways at the trunk by a
held horizontal force for 0.1 s from t = 1 s (the loop's perturbation).  Arms, with the same plant seeds:

  undisturbed  CppBatchSamplingPlanner, no noise and no push (the reference level)
  sampling     CppBatchSamplingPlanner on the disturbed plants
  robust       CppBatchRobustPlanner on the disturbed plants, planning against the plants' xfrc_std and xfrc_rate

Reported per arm: each plant's average cost per step, their mean, the plants that fell (trunk below 0.15 m at any step)
or diverged, and the aggregate x-realtime (B x simulated seconds / wall time).  One seed and one run per arm: this is
not a significance test.  Then one plant step is timed at B = 1, 32, 132 and 256 on three banks, alternated step by
step: clean (no disturbance), tiny (control and force noise of std 1e-6: every disturbance path runs, the motion is the
clean one) and disturbed (control noise 0.1, force noise 1 and a held trunk wrench: the motion differs, so the solver's
work does too).  CUDA events around the launch and a host clock around the whole call, medians over --timed steps.  One JSON line per arm and per size, after
a line with the GPU's name and power limit.
Usage: python profiles/disturbed_closed_loop.py [--plants 8] [--steps 300] [--N 60] [--H 36] [--xfrc-std 1,3]
                                               [--xfrc-rate 0.1] [--push 60] [--timed 300]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, mocap_of  # noqa: E402

from mujoco_mpc_b200.closed_loop import synchronous_planning_cost  # noqa: E402
from mujoco_mpc_b200.engine import (PLANT_DIVERGED, CppBatchRobustPlanner, CppBatchSamplingPlanner,  # noqa: E402
                                    CppPlantBank)

TRUNK = 3          # the Quadruped's trunk body
FELL = 0.15        # trunk height (m) below which a plant has fallen


def push(m, B, force):
    """perturbation(i, time): force (N) along +y on every trunk held from step 1 s / timestep for 0.1 s."""
    on = np.zeros((B, m.nbody, 6))
    on[:, TRUNK, 1] = force
    i0 = int(round(1.0 / m.opt_timestep))
    i1 = i0 + int(round(0.1 / m.opt_timestep))

    def perturbation(i, t):
        return on if i == i0 else np.zeros_like(on) if i == i1 else None
    return perturbation


def run_arm(m, arm, B, N, H, steps, std, rate, force, plant_seeds, plan_seeds):
    if arm == "robust":
        pl = CppBatchRobustPlanner(m, B, N, H, xfrc_std=std, xfrc_rate=rate, seeds=plan_seeds)
    else:
        pl = CppBatchSamplingPlanner(m, B, N, H, seeds=plan_seeds)
    bank = CppPlantBank(m, B)
    q0, mc = m.key_qpos[0], mocap_of(m)
    for b in range(B):
        pl.reset(b)
        bank.reset(b, q0, np.zeros(m.nv), 0.0, mc)
        if arm != "undisturbed":
            bank.set_disturbance(b, xfrc_std=std, xfrc_rate=rate, seed=plant_seeds[b])
    out = synchronous_planning_cost(pl, bank, steps, 1, perturbation=None if arm == "undisturbed" else push(m, B, force))
    pl.close(); bank.close()
    avg = np.asarray(out["average_cost"], float)
    height = out["states"][:, :, 2].min(0)
    return {"arm": arm, "plants": B, "N": N, "H": H, "steps": steps, "xfrc_std": 0.0 if arm == "undisturbed" else std,
            "xfrc_rate": rate, "push_N": 0.0 if arm == "undisturbed" else force,
            "average_cost": avg.round(5).tolist(), "mean_average_cost": float(avg.mean()),
            "fell": np.flatnonzero(height < FELL).tolist(),
            "diverged": np.flatnonzero(np.asarray(out["final_status"]) == PLANT_DIVERGED).tolist(),
            "min_trunk_height": height.round(4).tolist(), "x_realtime": float(out["x_realtime"]),
            "wall_s": float(out["wall_time"]), "planning_s": float(out["planning_time"])}


def time_steps(m, B, timed, warmup=20):
    q0, mc = m.key_qpos[0], mocap_of(m)
    banks = {"clean": CppPlantBank(m, B), "tiny": CppPlantBank(m, B), "disturbed": CppPlantBank(m, B)}
    w = np.zeros((m.nbody, 6)); w[TRUNK, :3] = [5.0, -3.0, 0.0]
    for b in range(B):
        for name, bank in banks.items():
            bank.reset(b, q0, np.zeros(m.nv), 0.0, mc)
        banks["tiny"].set_disturbance(b, 1e-6, 0.05, 1e-6, 0.1, seed=b)
        banks["disturbed"].set_disturbance(b, 0.1, 0.05, 1.0, 0.1, seed=b)
        banks["disturbed"].set_xfrc(b, w)
    u = np.zeros((B, m.nu), np.float32)
    kernel = {k: [] for k in banks}
    call = {k: [] for k in banks}
    for i in range(warmup + timed):
        for name, bank in banks.items():           # alternated step by step
            t0 = time.perf_counter()
            bank.step(u)
            dt = time.perf_counter() - t0
            if i >= warmup:
                kernel[name].append(bank.last_kernel_ms())
                call[name].append(dt * 1e3)
    running = {k: int(sum(bank.get(b)["status"] == 0 for b in range(B))) for k, bank in banks.items()}
    for bank in banks.values():
        bank.close()
    row = {"B": B, "timed_steps": timed}
    for k in banks:
        row[k] = {"kernel_ms_median": float(np.median(kernel[k])), "kernel_ms_p90": float(np.percentile(kernel[k], 90)),
                  "call_ms_median": float(np.median(call[k])), "running_plants": running[k]}
    for k in ("tiny", "disturbed"):
        row[k + "_kernel_ratio"] = row[k]["kernel_ms_median"] / row["clean"]["kernel_ms_median"]
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plants", type=int, default=8)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--N", type=int, default=60)
    ap.add_argument("--H", type=int, default=36)
    ap.add_argument("--xfrc-std", default="1,3", help="comma-separated plant force-noise levels (N and N m)")
    ap.add_argument("--xfrc-rate", type=float, default=0.1)
    ap.add_argument("--push", type=float, default=60.0, help="sideways trunk push (N) for 0.1 s from t = 1 s")
    ap.add_argument("--timed", type=int, default=300)
    ap.add_argument("--skip-timing", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("disturbed_closed_loop.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    m = get_model("quadruped")
    B = args.plants
    plant_seeds = [1000 + b for b in range(B)]
    plan_seeds = [0x5EED + b for b in range(B)]
    print(json.dumps(run_arm(m, "undisturbed", B, args.N, args.H, args.steps, 0.0, args.xfrc_rate, 0.0, plant_seeds,
                             plan_seeds)), flush=True)
    for std in [float(s) for s in args.xfrc_std.split(",")]:
        for arm in ("sampling", "robust"):
            print(json.dumps(run_arm(m, arm, B, args.N, args.H, args.steps, std, args.xfrc_rate, args.push,
                                     plant_seeds, plan_seeds)), flush=True)
    if not args.skip_timing:
        for nb in (1, 32, 132, 256):
            print(json.dumps({"plant_step_timing": time_steps(m, nb, args.timed)}), flush=True)
    print(json.dumps({"gpu_after": gpu_identity(0)}), flush=True)


if __name__ == "__main__":
    main()
