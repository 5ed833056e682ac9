"""Per-problem model variants: one batched launch of B problems with B distinct model variants
(mjpc_b200_set_model_variants) against the same launch with every problem on the one model, the two alternated on one
handle in the same run.

  rollouts   device-event kernel time of one mjpc_b200_rollout_spline_batched launch
  arms       one_model: no variants; same_model_variants: B variants that are all the handle's own model (the same
             physics, so the difference is the cost of the per-problem model blocks alone); variants: B distinct
             variants (other physics: their solver iterations and contacts differ, so their time does too)
  planner    host wall time of one planning iteration of a CppBatchSamplingPlanner and a CppBatchILQGPlanner, with and
             without set_models

The variants are the ones tests/test_gpu_model_variants.py plans on (trunk / torso mass, friction, actuator gain,
joint damping and armature differ per problem).  Workloads: Quadruped 60 x 36 at B = 4 and 8, Humanoid Track 32 x 101
at B = 8, and the two planners on the Quadruped at B = 4.  One JSON line per workload, after a line with the GPU's
name and power limit.  Usage: python profiles/time_model_variants.py [--reps 20] [--rounds 3]"""
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
from time_batched import quadruped_problems, track_problems  # noqa: E402

from mujoco_mpc_b200.engine import CppBatchILQGPlanner, CppBatchSamplingPlanner, Engine  # noqa: E402


def _alternate(arms, rounds, reps):
    """rounds x (each arm reps times, in turn); per arm the median and minimum over all its samples and each round's
    median"""
    for f in arms.values():
        f(); f()                                   # warm-up
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            out[k].append([f() for _ in range(reps)])
    return {k: {"median": float(np.median(v)), "min": float(np.min(v)), "round_medians": [float(np.median(r)) for r in v]}
            for k, v in out.items()}


def time_rollouts(name, m, make, B, N, H, rounds, reps):
    V = _variants("quadruped" if name == "Quadruped" else "humanoid_track", B)
    e = Engine(m, B * N, H)
    states, mocaps, knots, kt = make(m, B, N, H)
    times = 0.1 * np.arange(B)
    kts = np.stack([kt + t for t in times])

    current = [None]

    def launch(models):
        def run():
            if current[0] is not models:
                e.set_model_variants(models)
                current[0] = models
            e.rollout_spline_batched(states, times, mocaps, knots, kts, 2, H)
            return e.last_kernel_ms
        return run

    same = [m] * B
    res = _alternate({"one_model": launch(None), "same_model_variants": launch(same), "variants": launch(V)}, rounds, reps)
    out = {"workload": f"{name} {B} problems x {N} candidates x {H} steps", "B": B, "N": N, "H": H, "rounds": rounds,
           "reps": reps, "static_kernel": int(e.last_kernel_shape), "kernel_ms": res,
           "same_model_variants_over_one_model": res["same_model_variants"]["median"] / res["one_model"]["median"]}
    e.close()
    return out


def time_planner(kind, m, B, H, rounds, reps):
    V = _variants("quadruped", B)
    state, mocap, _, _ = quadruped_inputs(m, N=8, H=H)
    pl = CppBatchSamplingPlanner(m, B, 60, H) if kind == "sampling" else CppBatchILQGPlanner(m, B, H)
    for b in range(B):
        pl.reset(b); pl.set_state(b, state, 0.0, mocap)
    current = [None]

    def iterate(models):
        def run():
            if current[0] is not models:
                pl.set_models(models)
                current[0] = models
            t0 = time.perf_counter()
            pl.optimize_policy()
            return (time.perf_counter() - t0) * 1e3
        return run

    same = [m] * B
    res = _alternate({"one_model": iterate(None), "same_model_variants": iterate(same), "variants": iterate(V)}, rounds, reps)
    name = "CppBatchSamplingPlanner (60 candidates)" if kind == "sampling" else "CppBatchILQGPlanner (10 rollouts)"
    pl.close()
    return {"workload": f"Quadruped {name} planning iteration, {B} problems x {H} steps", "B": B, "H": H,
            "rounds": rounds, "reps": reps, "wall_ms": res,
            "same_model_variants_over_one_model": res["same_model_variants"]["median"] / res["one_model"]["median"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_model_variants.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad, track = get_model("quadruped"), get_model("humanoid_track")
    for B in (4, 8):
        print(json.dumps(time_rollouts("Quadruped", quad, quadruped_problems, B, 60, 36, args.rounds, args.reps)), flush=True)
    print(json.dumps(dict(time_rollouts("Humanoid Track", track, track_problems, 8, 32, 101, args.rounds, args.reps),
                          keyframes=getattr(track, "key_source", "?"))), flush=True)
    for kind in ("sampling", "ilqg"):
        print(json.dumps(time_planner(kind, quad, 4, 36, args.rounds, args.reps)), flush=True)


if __name__ == "__main__":
    main()
