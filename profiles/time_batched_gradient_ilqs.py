"""B independent Gradient and iLQS planning problems on the Quadruped (H = 64, 10 line-search / action rollouts, iLQS
with 60 sampling candidates; B = 1, 4, 8), the two arms alternated in the same run:

  planner   wall time of one planning iteration of all B problems: B single CppGradientPlanners (their own launches and
            the host GradientSweep each) against ONE CppBatchGradientPlanner, and B single CppILQSPlanners against ONE
            CppBatchILQSPlanner (median over the repetitions; iLQS alternates exploration 0.1 and 0, so that both
            its sampling and its iLQG halves run)
  sweep     the gradient of B nominal trajectories: mjpc_b200_gradient_batched (kernel_ms = its last_kernel_ms, from
            the first derivative kernel to the end of the sweep; wall_ms around the call) against
            model_derivatives_batched + cost_derivatives_batched + the host GradientSweep per problem (kernel_ms = the
            two calls' last_kernel_ms summed; wall_ms around all three)

One JSON line per workload, after a line with the GPU's name and power limit.
Usage: python profiles/time_batched_gradient_ilqs.py [--reps 20]"""
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

H, K = 64, 10


def time_planner(kind, m, B, reps):
    seeds = [0x5EED + b for b in range(B)]
    if kind == "gradient":
        kw = dict(num_trajectory=K, num_spline_points=5, representation=1, fd_tolerance=3e-4, fd_mode=1)
        batch = E.CppBatchGradientPlanner(m, B, H, **kw)
        singles = [E.CppGradientPlanner(m, H, **kw) for _ in range(B)]
    else:
        kw = dict(num_trajectory=60, num_rollouts=K, fd_tolerance=3e-4, fd_mode=1)
        batch = E.CppBatchILQSPlanner(m, B, H, seeds=seeds, **kw)
        singles = [E.CppILQSPlanner(m, H, seed=s, **kw) for s in seeds]
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    for b in range(B):
        batch.reset(b, np.zeros(m.nu)); batch.set_state(b, state, 0.01 * b, mocap_of(m))
        singles[b].reset(np.zeros(m.nu)); singles[b].set_state(state, 0.01 * b, mocap_of(m))
    calls = [0]

    def explore():                      # iLQS: sampling wins at 0.1 and cannot at 0, so the iLQG half runs too
        calls[0] += 1
        if kind == "ilqs":
            sigma = 0.1 if calls[0] % 4 < 2 else 0.0
            batch.set_exploration(sigma)
            for s in singles:
                s.set_exploration(sigma)

    def sequential():
        t0 = time.perf_counter()
        for s in singles:
            s.optimize_policy()
        return time.perf_counter() - t0

    def batched():
        explore()
        t0 = time.perf_counter()
        batch.optimize_policy()
        return time.perf_counter() - t0

    for _ in range(3):
        sequential(); batched()
    seq, bat = [], []
    for _ in range(reps):
        seq.append(sequential()); bat.append(batched())
    batch.close()
    for s in singles:
        s.close()
    what = (f"Gradient planner, Quadruped, {B} problems x {K} line-search candidates x {H} steps" if kind == "gradient" else
            f"iLQS planner, Quadruped, {B} problems x (60 sampling + {K} action rollouts) x {H} steps")
    res = {"workload": what, "planner": kind, "B": B,
           "reps": reps, "sequential": {"wall_ms": float(np.median(seq) * 1e3)},
           "batched": {"wall_ms": float(np.median(bat) * 1e3)}}
    res["wall_speedup"] = res["sequential"]["wall_ms"] / res["batched"]["wall_ms"]
    return res


def time_sweep(m, B, reps):
    """The nominal of one zero-action spline rollout per problem, each from its own start time."""
    e = E.Engine(m, max(B, 1), H)
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    times = 0.01 * np.arange(B)
    kt = np.arange(3) * (H - 1) * m.opt_timestep / 2
    e.rollout_spline_batched(np.tile(state, (B, 1)), times, np.tile(mocap_of(m), (B, 1)), np.zeros((B, 1, 3, m.nu)),
                             np.stack([kt + t for t in times]), 2, H)
    tr = e.fetch_all()
    x, u, t, res = tr["states"], tr["actions"], tr["times"], tr["residual"]
    mc = np.tile(mocap_of(m), (B, 1))

    def fused():
        t0 = time.perf_counter()
        e.gradient_batched(x, u, t, mc, res, 3e-4, mode=1)
        return time.perf_counter() - t0, e.last_kernel_ms

    def host():
        t0 = time.perf_counter()
        A, Bm, Cm, D = e.model_derivatives_batched(x, u, t, mc, 3e-4, mode=1)
        ms = e.last_kernel_ms
        cx, cu, _, _, _ = e.cost_derivatives_batched(res, Cm, D)
        ms += e.last_kernel_ms
        for b in range(B):
            E.host_gradient_sweep(A[b], Bm[b], cx[b], cu[b])
        return time.perf_counter() - t0, ms

    for _ in range(3):
        fused(); host()
    f, h = [], []
    for _ in range(reps):
        f.append(fused()); h.append(host())
    e.close()
    med = lambda v, i: float(np.median([r[i] for r in v]))  # noqa: E731
    out = {"workload": f"gradient of {B} Quadruped nominals x {H} steps", "B": B, "reps": reps,
           "separate_plus_host_sweep": {"wall_ms": med(h, 0) * 1e3, "kernel_ms": med(h, 1)},
           "gradient_batched": {"wall_ms": med(f, 0) * 1e3, "kernel_ms": med(f, 1)}}
    out["wall_speedup"] = out["separate_plus_host_sweep"]["wall_ms"] / out["gradient_batched"]["wall_ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_batched_gradient_ilqs.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad = get_model("quadruped")
    for kind in ("gradient", "ilqs"):
        for B in (1, 4, 8):
            print(json.dumps(time_planner(kind, quad, B, args.reps)), flush=True)
    for B in (1, 4, 8):
        print(json.dumps(time_sweep(quad, B, args.reps)), flush=True)


if __name__ == "__main__":
    main()
