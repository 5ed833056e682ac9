"""Record every output of the C++ host planners (for bitwise comparison of builds): each planning iteration's return
code, every get_result array, and action_from_policy samples (current and previous policy; with and without a state
for the planners whose policy reads it).

  python profiles/dump_planners.py out.npz [--iters 10]
  python profiles/dump_planners.py --cmp a.npz b.npz

Covered, on Particle and Quadruped: every single planner kind (Sampling, Cross-Entropy, Sample Gradient, Robust,
Gradient, iLQG, iLQS), the Agent with each of its seven planner ids, and every batch kind at B = 3 (the batched iLQG
planner included).  One iteration of each single planner and Agent is its NominalTrajectory (planning disabled).  iLQS,
single and batched, follows an exploration schedule that drives sampling to 0, so that its iLQG half and the
iLQG-to-spline conversion both run.  The problems differ in start state, start time, mocap and task snapshot.
Run it once per build on the same GPU; the archive is written with fixed zip timestamps, so equal outputs give equal
files.  The library is the one mujoco_mpc_b200.build.SO names (MJPC_B200_SO selects another build).
"""
import argparse
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B = 3
SEEDS = [0x5EED, 7, 123456]
SIGMA = [0.1, 0.1, 0.0, 0.0, 0.0, 0.0, 0.0, 0.1, 0.1, 0.1]   # iLQS exploration: 0 leaves the iteration to iLQG
DTS = (0.0, 0.013, 0.05, 0.2)
HORIZON = {"particle": 26, "quadruped": 24}
NOMINAL_ITER = 3                                             # the iteration that runs NominalTrajectory instead


def compare(a, b):
    a, b = np.load(a), np.load(b)
    same = a.files == b.files
    if not same:
        print("keys differ:", sorted(set(a.files) ^ set(b.files)))
    for k in a.files:
        if k not in b.files:
            continue
        x, y = a[k], b[k]
        if x.shape == y.shape and x.tobytes() == y.tobytes():
            continue
        same = False
        print("%-60s differs" % k + ("" if x.dtype.kind in "US" or x.shape != y.shape else
                                      ", max abs %.3g" % np.abs(x - y).max()))
    print("%d arrays, %s" % (len(a.files), "all bitwise equal" if same else "DIFFERENT"))
    return 0 if same else 1


def save(path, arrays):
    with zipfile.ZipFile(path, "w") as z:
        for k, v in arrays.items():
            with z.open(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), "w") as fh:
                np.lib.format.write_array(fh, np.asarray(v))


def put(out, key, result):
    for k, v in result.items():
        out["%s/%s" % (key, k)] = np.asarray(v)


def actions(out, key, act, t0, state, feedback):
    """act(time, state, use_previous) at t0 + DTS, current and previous; with the state too when the policy reads it."""
    rows = []
    for dt in DTS:
        for prev in (False, True):
            rows.append(act(t0 + dt, None, prev))
            if feedback:
                rows.append(act(t0 + dt, state, prev))
    out[key + "/actions"] = np.array(rows)


def singles(m, H):
    from mujoco_mpc_b200 import engine as E
    N, s = 16, SEEDS[0]
    yield "sampling", E.CppSamplingPlanner(m, N, H, seed=s), False
    yield "cross_entropy", E.CppCrossEntropyPlanner(m, N, H, seed=s), False
    yield "sample_gradient", E.CppSampleGradientPlanner(m, N, H, num_gradient=4, gradient_filter=0.6, seed=s), False
    yield "robust", E.CppRobustPlanner(m, N, H, ncandidates=3, nrepetitions=4, xfrc_std=1.0, xfrc_rate=0.1, seed=s), False
    yield "gradient", E.CppGradientPlanner(m, H, num_trajectory=8, fd_tolerance=1e-3, fd_mode=0), False
    yield "ilqg", E.CppILQGPlanner(m, H, num_rollouts=10, fd_tolerance=1e-3, fd_mode=0), True
    yield "ilqs", E.CppILQSPlanner(m, H, num_trajectory=8, num_rollouts=6, fd_tolerance=1e-3, fd_mode=0, seed=s), True


def batches(m, H):
    from mujoco_mpc_b200 import engine as E
    N = 16
    yield "sampling", E.CppBatchSamplingPlanner(m, B, N, H, seeds=SEEDS)
    yield "cross_entropy", E.CppBatchCrossEntropyPlanner(m, B, N, H, seeds=SEEDS)
    yield "sample_gradient", E.CppBatchSampleGradientPlanner(m, B, N, H, num_gradient=4, gradient_filter=0.6, seeds=SEEDS)
    yield "robust", E.CppBatchRobustPlanner(m, B, N, H, ncandidates=3, nrepetitions=4, xfrc_std=1.0, xfrc_rate=0.1,
                                            seeds=SEEDS)
    yield "gradient", E.CppBatchGradientPlanner(m, B, H, num_trajectory=8, fd_tolerance=1e-3, fd_mode=0)
    yield "ilqs", E.CppBatchILQSPlanner(m, B, H, num_trajectory=8, num_rollouts=6, fd_tolerance=1e-3, fd_mode=0,
                                        seeds=SEEDS)
    yield "ilqg", E.CppBatchILQGPlanner(m, B, H, num_rollouts=10, fd_tolerance=1e-3, fd_mode=0)


def state_at(pr, b, it):
    return pr["states"][b], pr["times"][b] + 0.01 * it, pr["mocaps"][b]


def run_single(out, key, pl, feedback, pr, iters):
    b = 1
    pl.reset()
    pl.set_task(pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    for it in range(iters):
        if key.endswith("/ilqs"):
            pl.set_exploration(SIGMA[it % len(SIGMA)])
        pl.set_state(*state_at(pr, b, it))
        k = "%s/%02d" % (key, it)
        if it == NOMINAL_ITER:
            code = pl.nominal_trajectory()
        else:
            code = pl.optimize_policy()
        out[k + "/code"] = np.asarray(code if isinstance(code, int) else 0)
        put(out, k, pl.result())
        actions(out, k, lambda t, s, p: pl.action_from_policy(t, s, p) if feedback else pl.action_from_policy(t, p),
                state_at(pr, b, it)[1], pr["states"][b], feedback)
    pl.close()


def run_batch(out, key, bp, pr, iters):
    kind = key.rsplit("/", 1)[1]
    for b in range(B):
        bp.reset(b)
        bp.set_task(b, pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    for it in range(iters):
        if kind == "ilqs":
            bp.set_exploration(SIGMA[it % len(SIGMA)])
        for b in range(B):
            bp.set_state(b, *state_at(pr, b, it))
        k = "%s/%02d" % (key, it)
        if kind == "ilqg" and it == NOMINAL_ITER:
            out[k + "/code"] = np.asarray(bp.nominal_trajectory())
        else:
            res = bp.optimize_policy()
            if kind in ("gradient", "ilqs", "ilqg"):
                out[k + "/code"] = np.asarray(res)
        for b in range(B):
            kb = "%s/%d" % (k, b)
            put(out, kb, bp.result(b))
            t0 = state_at(pr, b, it)[1]
            if kind == "ilqg":
                actions(out, kb, lambda t, s, p: bp.action_from_policy(b, t, s), t0, pr["states"][b], True)
            elif kind == "ilqs":
                actions(out, kb, lambda t, s, p: bp.action_from_policy(b, t, s, p), t0, pr["states"][b], True)
            else:
                actions(out, kb, lambda t, s, p: bp.action_from_policy(b, t, p), t0, pr["states"][b], False)
    bp.close()


def run_agent(out, key, m, planner, pr, iters):
    from mujoco_mpc_b200.engine import CppAgent
    a = CppAgent(m, planner=planner, num_trajectory=16, ilqg_num_rollouts=6, fd_tolerance=1e-3, seed=SEEDS[2])
    b = 2
    a.reset()
    a.set_task(pr["weights"][b], pr["parameters"][b], pr["task_states"][b])
    for it in range(iters):
        a.set_state(*state_at(pr, b, it))
        a.set_plan_enabled(it != NOMINAL_ITER)
        k = "%s/%02d" % (key, it)
        out[k + "/code"] = np.asarray(a.plan_iteration())
        actions(out, k, lambda t, s, p: a.action_from_policy(t, s, p), state_at(pr, b, it)[1], pr["states"][b], True)
    a.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--cmp", nargs=2)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if a.cmp:
        sys.exit(compare(*a.cmp))
    from conftest import get_model
    from test_gpu_batched_ilqg import _problems

    from mujoco_mpc_b200.engine import CppAgent
    out = {}
    for name in ("particle", "quadruped"):
        m, H = get_model(name), HORIZON[name]
        pr = _problems(m, H, B=B)
        for kind, pl, feedback in singles(m, H):
            run_single(out, "single/%s/%s" % (name, kind), pl, feedback, pr, a.iters)
        for kind, bp in batches(m, H):
            run_batch(out, "batch/%s/%s" % (name, kind), bp, pr, a.iters)
        for planner in CppAgent.PLANNERS:
            run_agent(out, "agent/%s/%s" % (name, planner), m, planner, pr, a.iters)
    save(a.out, out)
    print("%d arrays written to %s" % (len(out), a.out))


if __name__ == "__main__":
    main()
