"""B independent planning problems: B sequential single-problem launches (mjpc_b200_rollout_spline) against ONE batched
launch (mjpc_b200_rollout_spline_batched), the two alternated in the same run.

  rollouts   device-event kernel time (sum over the B launches / the one launch) and host wall time of one planning
             iteration's rollouts of all B problems, host buffers in and out
  planner    host wall time of one full planning iteration of B problems: B CppSamplingPlanners against one
             CppBatchSamplingPlanner (the planners do not expose their kernel time)

Workloads: the reference's shipped Quadruped load (60 candidates x 36 steps, B = 1, 2, 4), Humanoid Track on the
reference keyframes (32 x 101, B = 1, 4, 8) and the Quadruped planner at B = 4.  One JSON line per workload, after a
line with the GPU's name and power limit.  Usage: python profiles/time_batched.py [--reps 20]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, quadruped_inputs  # noqa: E402
from mujoco_mpc_b200.engine import CppBatchSamplingPlanner, CppSamplingPlanner, Engine  # noqa: E402


def quadruped_problems(m, B, N, H):
    state, mocap, _, kt = quadruped_inputs(m, N=N, H=H)
    knots = np.stack([quadruped_inputs(m, N=N, H=H, seed=b)[2] for b in range(B)])
    return np.tile(state, (B, 1)), np.tile(mocap, (B, 1)), knots, kt


def track_problems(m, B, N, H):
    P = int(m.numeric.get("sampling_spline_points", [16])[0])
    rng = np.random.default_rng(0)
    state = np.concatenate([m.key_qpos[0], m.key_qvel[0]])
    mocap = np.concatenate([m.key_mpos[0].reshape(-1, 3), np.tile([1.0, 0, 0, 0], (m.nmocap, 1))], 1).reshape(-1)
    knots = np.clip(0.15 * rng.standard_normal((B, N, P, m.nu)), -1, 1); knots[:, 0] = 0
    kt = np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    return np.tile(state, (B, 1)), np.tile(mocap, (B, 1)), knots, kt


def time_rollouts(name, m, make, B, N, H, reps):
    e = Engine(m, B * N, H)
    states, mocaps, knots, kt = make(m, B, N, H)
    times = 0.1 * np.arange(B)
    kts = np.stack([kt + t for t in times])

    def sequential():
        t0, ms = time.perf_counter(), 0.0
        for b in range(B):
            e.rollout_spline(states[b], times[b], mocaps[b], knots[b], kts[b], 2, H)
            ms += e.last_kernel_ms
        return ms, time.perf_counter() - t0

    def batched():
        t0 = time.perf_counter()
        e.rollout_spline_batched(states, times, mocaps, knots, kts, 2, H)
        return e.last_kernel_ms, time.perf_counter() - t0

    arms = {"sequential": sequential, "batched": batched}
    for f in arms.values():
        f(); f()                                   # warm-up
    out = {k: [] for k in arms}
    for _ in range(reps):                          # alternated
        for k, f in arms.items():
            out[k].append(f())
    res = {"workload": f"{name} {B} x {N} candidates x {H} steps", "B": B, "N": N, "H": H, "reps": reps,
           "static_kernel": int(e.last_kernel_shape)}
    for k, v in out.items():
        a = np.asarray(v)
        res[k] = {"kernel_ms": float(np.median(a[:, 0])), "kernel_ms_min": float(a[:, 0].min()),
                  "wall_ms": float(np.median(a[:, 1]) * 1e3)}
    res["kernel_speedup"] = res["sequential"]["kernel_ms"] / res["batched"]["kernel_ms"]
    res["wall_speedup"] = res["sequential"]["wall_ms"] / res["batched"]["wall_ms"]
    e.close()
    return res


def time_planner(m, B, N, H, reps):
    seeds = [0x5EED + b for b in range(B)]
    state, mocap, _, _ = quadruped_inputs(m, N=N, H=H)
    batch = CppBatchSamplingPlanner(m, B, N, H, seeds=seeds)
    singles = [CppSamplingPlanner(m, N, H, seed=s) for s in seeds]
    for b in range(B):
        batch.reset(b); batch.set_state(b, state, 0.0, mocap)
        singles[b].reset(); singles[b].set_state(state, 0.0, mocap)

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
    res = {"workload": f"Quadruped planning iteration, {B} problems x {N} candidates x {H} steps", "B": B, "N": N, "H": H,
           "reps": reps, "sequential": {"wall_ms": float(np.median(seq) * 1e3)}, "batched": {"wall_ms": float(np.median(bat) * 1e3)}}
    res["wall_speedup"] = res["sequential"]["wall_ms"] / res["batched"]["wall_ms"]
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
        raise SystemExit("time_batched.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad, track = get_model("quadruped"), get_model("humanoid_track")
    for B in (1, 2, 4):
        print(json.dumps(time_rollouts("Quadruped", quad, quadruped_problems, B, 60, 36, args.reps)), flush=True)
    for B in (1, 4, 8):
        print(json.dumps(dict(time_rollouts("Humanoid Track", track, track_problems, B, 32, 101, args.reps),
                              keyframes=getattr(track, "key_source", "?"))), flush=True)
    print(json.dumps(time_planner(quad, 4, 60, 36, args.reps)), flush=True)


if __name__ == "__main__":
    main()
