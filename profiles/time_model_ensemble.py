"""Model ensembles: the cost of scoring every candidate on K member models (mjpc_b200_set_model_ensemble) against the
same launch without an ensemble, the arms alternated on one handle in the same run.

  kernel_ms  device-event time of one mjpc_b200_rollout_spline_batched launch: the rollout of B x K x N trajectories,
             ensemble_score_kernel and the ranking (without an ensemble: the rollout of B x N and the ranking)
  wall_ms    host wall time of one planning iteration of a CppSamplingPlanner (B = 1) or a CppBatchSamplingPlanner
             (B = 4) of 60 candidates, with and without set_ensemble

Members are the Quadruped variants tests/test_gpu_model_variants.py plans on (trunk mass, foot friction, actuator gain,
joint damping and armature differ), K of them (K = 8 repeats the four).  Workload: Quadruped 60 x 36, K in {1, 2, 4, 8},
B in {1, 4}.  B x K x 60 passes 2 x 132 CTAs (two co-resident candidates per SM) from B K = 5 on.  One JSON line per
workload, after a line with the GPU's name and power limit.  Usage: python profiles/time_model_ensemble.py [--reps 20]
[--rounds 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, quadruped_inputs  # noqa: E402
from test_gpu_model_variants import _variants  # noqa: E402
from time_batched import quadruped_problems  # noqa: E402
from time_model_variants import _alternate  # noqa: E402

from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, CppSamplingPlanner, Engine  # noqa: E402

N, H = 60, 36


def members(K):
    V = _variants("quadruped", 4)
    return [V[k % 4] for k in range(K)]


def time_rollouts(m, B, K, rounds, reps):
    e = Engine(m, B * N, H)
    states, mocaps, knots, kt = quadruped_problems(m, B, N, H)
    times = 0.1 * np.arange(B)
    kts = np.stack([kt + t for t in times])
    V = members(K)
    current = [None]

    def launch(models):
        def run():
            if current[0] is not models:
                e.set_model_ensemble(models, worst=len(models) if models else None)
                current[0] = models
            e.rollout_spline_batched(states, times, mocaps, knots, kts, 2, H)
            return e.last_kernel_ms
        return run

    res = _alternate({"plain": launch(None), "ensemble": launch(V)}, rounds, reps)
    out = {"workload": f"Quadruped {B} problems x {N} candidates x {H} steps, K = {K} members", "B": B, "K": K, "N": N,
           "H": H, "trajectories": B * K * N, "rounds": rounds, "reps": reps, "kernel_ms": res,
           "ensemble_over_plain": res["ensemble"]["median"] / res["plain"]["median"]}
    e.close()
    return out


def time_planner(m, B, K, rounds, reps):
    state, mocap, _, _ = quadruped_inputs(m, N=8, H=H)
    single = B == 1
    pl = CppSamplingPlanner(m, N, H) if single else CppBatchSamplingPlanner(m, B, N, H)
    if single:
        pl.reset(); pl.set_state(state, 0.0, mocap)
    else:
        for b in range(B):
            pl.reset(b); pl.set_state(b, state, 0.0, mocap)
    V = members(K)
    current = [None]

    def iterate(models):
        def run():
            if current[0] is not models:
                pl.set_ensemble(models, worst=len(models) if models else None)
                current[0] = models
            t0 = time.perf_counter()
            pl.optimize_policy()
            return (time.perf_counter() - t0) * 1e3
        return run

    res = _alternate({"plain": iterate(None), "ensemble": iterate(V)}, rounds, reps)
    name = "CppSamplingPlanner" if single else f"CppBatchSamplingPlanner ({B} problems)"
    pl.close()
    return {"workload": f"Quadruped {name} planning iteration, {N} candidates x {H} steps, K = {K} members", "B": B,
            "K": K, "rounds": rounds, "reps": reps, "wall_ms": res,
            "ensemble_over_plain": res["ensemble"]["median"] / res["plain"]["median"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_model_ensemble.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad = get_model("quadruped")
    for B in (1, 4):
        for K in (1, 2, 4, 8):
            print(json.dumps(time_rollouts(quad, B, K, args.rounds, args.reps)), flush=True)
    for B in (1, 4):
        for K in (1, 2, 4, 8):
            print(json.dumps(time_planner(quad, B, K, args.rounds, args.reps)), flush=True)


if __name__ == "__main__":
    main()
