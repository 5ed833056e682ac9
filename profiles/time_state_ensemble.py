"""Initial-state ensembles: the cost of scoring every candidate over K initial states drawn from each problem's state
covariance (mjpc_b200_rollout_spline_belief_batched) against the plain launch, the arms alternated on one handle.

  kernel_ms  device-event time of the rollout part of one launch: the rollout of B x K x N trajectories,
             ensemble_score_kernel and the ranking (plain: the rollout of B x N and the ranking)
  sample_us  device time of state_sample_kernel (torch.profiler / CUPTI): the fp64 Cholesky factor of each problem's
             covariance and the K - 1 member states, one CTA per problem

Workloads: Quadruped 60 x 36, K in {1, 2, 4, 8}, B in {1, 8}; and the sampling kernel alone at B = 64 Humanoid Track
problems (2 nv = 54), K = 8.  One JSON line per workload, after a line with the GPU's name and power limit.
Usage: python profiles/time_state_ensemble.py [--reps 20] [--rounds 3]"""
import argparse
import json
import os
import sys

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model  # noqa: E402
from time_batched import quadruped_problems, track_problems  # noqa: E402
from time_model_variants import _alternate  # noqa: E402

from mujoco_mpc_b200.engine import Engine  # noqa: E402

N, H = 60, 36


def covariances(m, B, scale=1e-3, seed=0):
    rng = np.random.default_rng(seed)
    n = 2 * m.nv
    A = rng.standard_normal((B, n, n))
    return scale * (A @ A.transpose(0, 2, 1) / n + 0.2 * np.eye(n))


def sample_kernel_us(fn, reps):
    """mean device time [us] of state_sample_kernel over reps calls of fn, from a torch.profiler trace"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    for a in prof.key_averages():
        if a.key == "state_sample_kernel":
            total = getattr(a, "device_time_total", None)
            if total is None:
                total = a.cuda_time_total
            return {"mean": float(total) / max(a.count, 1), "count": int(a.count)}
    return None


def time_launch(m, make, B, K, n, rounds, reps, name):
    e = Engine(m, B * max(K, 1) * n, H)
    states, mocaps, knots, kt = make(m, B, n, H)
    times = 0.1 * np.arange(B)
    kts = np.stack([kt + t for t in times])
    P = covariances(m, B)

    def plain():
        e.rollout_spline_batched(states, times, mocaps, knots, kts, 2, H)
        return e.last_kernel_ms

    def belief():
        e.rollout_spline_belief_batched(states, P, times, mocaps, knots, kts, 2, H, K, K, 5, 0)
        return e.last_kernel_ms

    res = _alternate({"plain": plain, "belief": belief}, rounds, reps)
    out = {"workload": f"{name} {B} problems x {n} candidates x {H} steps, K = {K} members", "B": B, "K": K, "N": n,
           "H": H, "trajectories": B * K * n, "rounds": rounds, "reps": reps, "kernel_ms": res,
           "belief_over_plain": res["belief"]["median"] / res["plain"]["median"],
           "sample_us": sample_kernel_us(belief, reps)}
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_state_ensemble.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad = get_model("quadruped")
    for B in (1, 8):
        for K in (1, 2, 4, 8):
            print(json.dumps(time_launch(quad, quadruped_problems, B, K, N, args.rounds, args.reps, "Quadruped")),
                  flush=True)
    track = get_model("humanoid_track")
    # the sampling kernel at B = 64 Humanoid-sized problems (one candidate each: the rollout is not the point here)
    print(json.dumps(time_launch(track, track_problems, 64, 8, 1, 1, args.reps, "Humanoid Track")), flush=True)


if __name__ == "__main__":
    main()
