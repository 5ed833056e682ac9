"""B independent iLQG problems: B sequential single-problem calls against ONE batched call per sweep, the two alternated
in the same run.

  sweeps     device-event kernel time of each iLQG sweep (sum over the B calls / the one batched call) for BASELINE
             config 4 (Quadruped, H = 64, K = 10, centred FD 3e-4): model derivatives, cost derivatives, backward pass,
             action (line-search) rollouts; B = 1, 4, 8
  planner    host wall time of one full iLQG planning iteration of B problems: B CppILQGPlanners against one
             CppBatchILQGPlanner, B = 4, 8 (the planners do not expose their kernel time)

One JSON line per workload, after a line with the GPU's name and power limit.
Usage: python profiles/time_batched_ilqg.py [--reps 20]"""
import argparse
import json
import os
import sys
import time

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from bench import gpu_identity  # noqa: E402
from conftest import get_model, quadruped_inputs  # noqa: E402
from mujoco_mpc_b200.engine import CppBatchILQGPlanner, CppILQGPlanner, Engine  # noqa: E402

H, K, TOL = 64, 10, 3e-4


def nominal(m, e, B):
    """B nominal trajectories from different start times: the rollouts of B seeded splines."""
    state, mocap, _, kt = quadruped_inputs(m, N=1, H=H)
    knots = np.stack([quadruped_inputs(m, N=1, H=H, seed=b)[2] for b in range(B)])
    times = 0.1 * np.arange(B)
    e.rollout_spline_batched(np.tile(state, (B, 1)), times, np.tile(mocap, (B, 1)), knots, np.stack([kt + t for t in times]), 2, H)
    tr = e.fetch_all()
    return dict(states=np.tile(state, (B, 1)), times=times, mocaps=np.tile(mocap, (B, 1)), x=tr["states"], u=tr["actions"],
                t=tr["times"], residual=tr["residual"])


def time_sweeps(m, B, reps):
    e = Engine(m, B * K, H)
    e.set_differentiable(True)
    pr = nominal(m, e, B)
    A, Bm, Cm, D = e.model_derivatives_batched(pr["x"], pr["u"], pr["t"], pr["mocaps"], TOL, mode=1)
    cx, cu, cxx, cuu, cxu = e.cost_derivatives_batched(pr["residual"], Cm, D)
    mu = np.ones(B, np.float32)
    bp = e.backward_pass_batched(A, Bm, cx, cu, cxx, cxu, cuu, pr["u"], mu=mu)
    steps = np.tile(np.concatenate([np.logspace(0, -3, K - 1), [0.0]]), (B, 1))
    sweeps = {
        "model_derivatives": (
            lambda b: e.model_derivatives(pr["x"][b], pr["u"][b], pr["t"][b], pr["mocaps"][b], TOL, mode=1),
            lambda: e.model_derivatives_batched(pr["x"], pr["u"], pr["t"], pr["mocaps"], TOL, mode=1)),
        "cost_derivatives": (
            lambda b: e.cost_derivatives(pr["residual"][b], Cm[b], D[b]),
            lambda: e.cost_derivatives_batched(pr["residual"], Cm, D)),
        "backward_pass": (
            lambda b: e.backward_pass(A[b], Bm[b], cx[b], cu[b], cxx[b], cxu[b], cuu[b], pr["u"][b], mu=1.0),
            lambda: e.backward_pass_batched(A, Bm, cx, cu, cxx, cxu, cuu, pr["u"], mu=mu)),
        "action_rollouts": (
            lambda b: e.rollout_feedback(pr["states"][b], pr["times"][b], pr["mocaps"][b], pr["u"][b], pr["x"][b], pr["t"][b],
                                         bp["K"][b], bp["du"][b], steps[b], 3),
            lambda: e.rollout_feedback_batched(pr["states"], pr["times"], pr["mocaps"], pr["u"], pr["x"], pr["t"], bp["K"],
                                               bp["du"], steps, 3)),
    }
    res = {"workload": f"Quadruped iLQG sweeps, {B} problems, H = {H}, K = {K}, centred FD {TOL}", "B": B, "reps": reps,
           "backward_status": bp["status"].tolist()}
    for name, (single, batched) in sweeps.items():
        def seq():
            ms = 0.0
            for b in range(B):
                single(b)
                ms += e.last_kernel_ms
            return ms

        def bat():
            batched()
            return e.last_kernel_ms
        for _ in range(2):
            seq(); bat()
        s, t = [], []
        for _ in range(reps):                       # alternated
            s.append(seq()); t.append(bat())
        res[name] = {"sequential_kernel_ms": float(np.median(s)), "batched_kernel_ms": float(np.median(t)),
                     "speedup": float(np.median(s) / np.median(t))}
    e.close()
    return res


def time_planner(m, B, reps):
    state, mocap, _, _ = quadruped_inputs(m, N=K, H=H)
    batch = CppBatchILQGPlanner(m, B, H, num_rollouts=K, representation=1)
    singles = [CppILQGPlanner(m, H, num_rollouts=K, representation=1) for _ in range(B)]
    for b in range(B):
        t0 = 0.1 * b
        batch.reset(b); batch.set_state(b, state, t0, mocap)
        singles[b].reset(); singles[b].set_state(state, t0, mocap)

    def sequential():
        t0 = time.perf_counter()
        for s in singles:
            s.optimize_policy()
        return time.perf_counter() - t0

    def batched():
        t0 = time.perf_counter()
        batch.optimize_policy()
        return time.perf_counter() - t0

    for _ in range(2):
        sequential(); batched()
    seq, bat = [], []
    for _ in range(reps):                           # alternated
        seq.append(sequential()); bat.append(batched())
    res = {"workload": f"Quadruped iLQG planning iteration, {B} problems, H = {H}, K = {K}", "B": B, "reps": reps,
           "sequential": {"wall_ms": float(np.median(seq) * 1e3)}, "batched": {"wall_ms": float(np.median(bat) * 1e3)}}
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
        raise SystemExit("time_batched_ilqg.py: no CUDA device")
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    quad = get_model("quadruped")
    for B in (1, 4, 8):
        print(json.dumps(time_sweeps(quad, B, args.reps)), flush=True)
    for B in (4, 8):
        print(json.dumps(time_planner(quad, B, args.reps)), flush=True)


if __name__ == "__main__":
    main()
