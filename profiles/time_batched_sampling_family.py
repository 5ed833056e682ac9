"""B independent planning problems of the Cross-Entropy, Robust and Sample Gradient planners: B single C++ planners
(one launch per planner, the Robust planner two) against ONE batch of that kind (one launch per iteration, the Robust
batch two), the two arms alternated in the same run.

  wall_ms    host wall time of one planning iteration of all B problems (median over the alternated repetitions)
  kernel_ms  device time of the rollout and ranking kernels of one such iteration, summed from a torch.profiler CUDA
             trace taken in a separate, unprofiled-timing pass (the planners do not expose their launches' events)

Workloads: Cross-Entropy on the stand-in hand at the reference's shipped Shadow Hand load (60 + 1 candidates x 26 steps,
tasks/shadow_reorient/task.xml), Robust and Sample Gradient on the Quadruped at 60 x 36; B = 1, 4, 8 each.  One JSON line
per workload, after a line with the GPU's name and power limit.  Usage: python profiles/time_batched_sampling_family.py
[--reps 20]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, mocap_of  # noqa: E402
from mujoco_mpc_b200 import engine as E  # noqa: E402


def make(kind, m, B, N, H):
    seeds = [0x5EED + b for b in range(B)]
    if kind == "ce":
        return E.CppBatchCrossEntropyPlanner(m, B, N, H, seeds=seeds), [E.CppCrossEntropyPlanner(m, N, H, seed=s) for s in seeds]
    if kind == "robust":
        return E.CppBatchRobustPlanner(m, B, N, H, seeds=seeds), [E.CppRobustPlanner(m, N, H, seed=s) for s in seeds]
    return (E.CppBatchSampleGradientPlanner(m, B, N, H, num_gradient=6, seeds=seeds),
            [E.CppSampleGradientPlanner(m, N, H, num_gradient=6, seed=s) for s in seeds])


def kernel_ms(f, iters=5):
    """Device time of the project's kernels per call of f, from a torch.profiler CUDA trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            f()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "kernel" in e.key)
    return us / iters / 1e3


def time_kind(kind, label, m, B, N, H, reps):
    batch, singles = make(kind, m, B, N, H)
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    for b in range(B):
        batch.reset(b, np.zeros(m.nu)); batch.set_state(b, state, 0.01 * b, mocap_of(m))
        singles[b].reset(np.zeros(m.nu)); singles[b].set_state(state, 0.01 * b, mocap_of(m))

    def sequential():
        t0 = time.perf_counter()
        for s in singles:
            s.optimize_policy()
        return time.perf_counter() - t0

    def batched():
        t0 = time.perf_counter()
        batch.optimize_policy()
        return time.perf_counter() - t0

    for _ in range(3):
        sequential(); batched()
    seq, bat = [], []
    for _ in range(reps):
        seq.append(sequential()); bat.append(batched())
    res = {"workload": f"{label}, {B} problems x {N} candidates x {H} steps", "planner": kind, "B": B, "N": N, "H": H,
           "reps": reps,
           "sequential": {"wall_ms": float(np.median(seq) * 1e3), "kernel_ms": kernel_ms(sequential)},
           "batched": {"wall_ms": float(np.median(bat) * 1e3), "kernel_ms": kernel_ms(batched)}}
    for k in ("wall_ms", "kernel_ms"):
        res[k.replace("_ms", "_speedup")] = res["sequential"][k] / res["batched"][k]
    batch.close()
    for s in singles:
        s.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_batched_sampling_family.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    hand, quad = get_model("shadow_reorient"), get_model("quadruped")
    for B in (1, 4, 8):
        print(json.dumps(time_kind("ce", "Cross-Entropy, stand-in hand", hand, B, 60, 26, args.reps)), flush=True)
    for kind, label in (("robust", "Robust, Quadruped"), ("sg", "Sample Gradient, Quadruped")):
        for B in (1, 4, 8):
            print(json.dumps(time_kind(kind, label, quad, B, 60, 36, args.reps)), flush=True)


if __name__ == "__main__":
    main()
