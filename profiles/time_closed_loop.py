"""Closed-loop MPC on device plants (closed_loop.synchronous_planning_cost on an engine.CppPlantBank): the reference's
testspeed loop for B episodes at once.

  loops      Quadruped, 2 s of simulated time (200 steps of 0.01 s), one planning iteration every 4 steps (testspeed's
             default), a CppBatchSamplingPlanner of N x H and B plants on B distinct model variants (those of
             tests/test_gpu_model_variants.py), B = 1, 4, 8, 16: one batched loop against B sequential loops of one
             (a batch of one and a bank of one on each variant), and at B = 1 the same loop with the fp64 oracle as the
             plant.  Reported: wall time, planning ms per iteration, plant-step kernel ms (CUDA events) and wall ms per
             step, aggregate x-realtime (B x simulated seconds / wall) and each plant's average cost per step.
  step       the kernel time (CUDA events, median over the steps) and host wall time of one plant step of B plants
             on the handle's model, B = 1, 32, 132, 256.

One JSON line per workload, after a line with the GPU's name and power limit.
Usage: python profiles/time_closed_loop.py [--steps 200] [--N 64] [--H 36] [--bs 1,4,8,16]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, mocap_of  # noqa: E402
from test_gpu_model_variants import _quadruped_variant  # noqa: E402

from mujoco_mpc_b200.closed_loop import synchronous_planning_cost  # noqa: E402
from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, CppPlantBank  # noqa: E402


class TimedPlant:
    """A plant bank whose step() records its host wall time and its kernel time."""

    def __init__(self, bank):
        self.bank, self.wall, self.kernel = bank, [], []

    def __getattr__(self, name):
        return getattr(self.bank, name)

    def step(self, ctrl):
        t0 = time.perf_counter()
        o = self.bank.step(ctrl)
        self.wall.append(time.perf_counter() - t0)
        self.kernel.append(self.bank.last_kernel_ms())
        return o


def device_loop(models, N, H, steps, spp, seeds, base):
    B = len(models)
    pl = CppBatchSamplingPlanner(base if B > 1 else models[0], B, N, H, seeds=seeds)
    bank = CppPlantBank(base if B > 1 else models[0], B)
    if B > 1:
        pl.set_models(models); bank.set_models(models)
    q0, mc = base.key_qpos[0], mocap_of(base)
    for b in range(B):
        pl.reset(b); bank.reset(b, q0, np.zeros(base.nv), 0.0, mc)
    plant = TimedPlant(bank)
    out = synchronous_planning_cost(pl, plant, steps, spp)
    pl.close(); bank.close()
    nplan = len(range(0, steps, spp))
    return dict(wall_s=out["wall_time"], planning_ms_per_iteration=1e3 * out["planning_time"] / nplan,
                plant_kernel_ms=float(np.median(plant.kernel)), plant_wall_ms=1e3 * float(np.median(plant.wall)),
                x_realtime=out["x_realtime"], average_cost=[float(c) for c in out["average_cost"]],
                diverged=int((out["final_status"] != 0).sum()))


def oracle_loop(m, N, H, steps, spp, seed):
    """The same loop order with the fp64 oracle as the plant (the planner on the device)."""
    from mujoco_mpc_b200.blob import to_blob
    from oracle import pyoracle
    plant = pyoracle.Oracle(to_blob(m), m, 64)
    pl = CppBatchSamplingPlanner(m, 1, N, H, seeds=[seed])
    pl.reset(0)
    q, v, t, warm, mc = m.key_qpos[0].astype(float), np.zeros(m.nv), 0.0, None, mocap_of(m)
    costs, walls, planning = [], [], 0.0
    start = time.perf_counter()
    for i in range(steps):
        pl.set_state(0, np.concatenate([q, v]), t, mc)
        u = pl.action_from_policy(0, t)
        t0 = time.perf_counter()
        r = plant.forward_debug(q, v, u, mc, time=t, warmstart=warm)
        costs.append(plant.cost_value(r["residual"][: m.task_num_residual]))
        walls.append(time.perf_counter() - t0)
        warm, q, v = r["qacc"], r["next_qpos"], r["next_qvel"]
        t += m.opt_timestep
        if i % spp == 0:
            t0 = time.perf_counter()
            pl.optimize_policy()
            planning += time.perf_counter() - t0
    wall = time.perf_counter() - start
    pl.close()
    return dict(wall_s=wall, planning_ms_per_iteration=1e3 * planning / len(range(0, steps, spp)),
                plant_wall_ms=1e3 * float(np.median(walls)), x_realtime=steps * m.opt_timestep / wall,
                average_cost=[float(np.mean(costs))])


def step_time(m, B, reps):
    bank = CppPlantBank(m, B)
    q0, mc = m.key_qpos[0], mocap_of(m)
    for b in range(B):
        bank.reset(b, q0, np.zeros(m.nv), 0.0, mc)
    u = np.zeros((B, m.nu), np.float32)
    for _ in range(3):
        bank.step(u)
    kern, wall = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        bank.step(u)
        wall.append(time.perf_counter() - t0)
        kern.append(bank.last_kernel_ms())
    bank.close()
    return dict(kernel_ms=float(np.median(kern)), wall_ms=1e3 * float(np.median(wall)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--spp", type=int, default=4)
    ap.add_argument("--N", type=int, default=64)
    ap.add_argument("--H", type=int, default=36)
    ap.add_argument("--bs", default="1,4,8,16")
    ap.add_argument("--step-bs", default="1,32,132,256")
    ap.add_argument("--reps", type=int, default=100)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    base = get_model("quadruped")
    bs = [int(x) for x in a.bs.split(",")]
    V = [_quadruped_variant(k) for k in range(max(bs))]
    seeds = [0x5EED + b for b in range(max(bs))]
    device_loop(V[:1], a.N, a.H, 8, a.spp, seeds[:1], base)          # warm-up
    for B in bs:
        batched = device_loop(V[:B], a.N, a.H, a.steps, a.spp, seeds[:B], base)
        singles = [device_loop(V[b:b + 1], a.N, a.H, a.steps, a.spp, seeds[b:b + 1], base) for b in range(B)]
        seq_wall = sum(s["wall_s"] for s in singles)
        print(json.dumps({"workload": "loop", "B": B, "N": a.N, "H": a.H, "steps": a.steps, "spp": a.spp,
                          "batched": batched,
                          "sequential": {"wall_s": seq_wall, "x_realtime": B * a.steps * base.opt_timestep / seq_wall,
                                         "planning_ms_per_iteration": float(np.mean([s["planning_ms_per_iteration"] for s in singles])),
                                         "plant_kernel_ms": float(np.mean([s["plant_kernel_ms"] for s in singles])),
                                         "plant_wall_ms": float(np.mean([s["plant_wall_ms"] for s in singles])),
                                         "average_cost": [s["average_cost"][0] for s in singles]}}), flush=True)
        if B == 1:
            print(json.dumps({"workload": "loop_fp64_plant", "B": 1,
                              "result": oracle_loop(base, a.N, a.H, a.steps, a.spp, seeds[0])}), flush=True)
    for B in [int(x) for x in a.step_bs.split(",")]:
        print(json.dumps({"workload": "plant_step", "B": B, **step_time(base, B, a.reps)}), flush=True)


if __name__ == "__main__":
    main()
