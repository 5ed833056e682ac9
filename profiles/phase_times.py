"""Per-phase cycle split of the rollout kernel (needs the -DMJPC_PHASE_TIMING build: MJPC_B200_SO=profiles/var_phase.so).
--map M must name the timer mapping the library was built with (-DMJPC_PHASE_MAP=M, csrc/dev_data.cuh): 0 pipeline
phases (default), 1 the Newton solve, 2 the first fork of the task-warp CTA."""
import argparse, os, sys
import numpy as np
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model, quadruped_inputs
from mujoco_mpc_b200.engine import Engine
ap = argparse.ArgumentParser()
ap.add_argument("--map", type=int, default=0, choices=[0, 1, 2])
args = ap.parse_args()
m = get_model("quadruped")
e = Engine(m, 256, 64)
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
state, mocap, knots, kt = d["state"], d["mocap"], d["knots"], d["kt"]   # the profiled inputs (prof_rollout.py)
for _ in range(2):
    e.rollout_spline(state, 0.0, mocap, knots, kt, 2, 64)
st = e.fetch_stats().astype(float)
tot = st[:, 0]
NAMES = {
    0: ["kinematics+com+crb", "collision", "make_constraint", "vel+smooth+reference", "solve (rest)", "solve: Hessian assembly",
        "solve: Cholesky factor+solve", "policy+residual+cost+euler+output"],
    1: ["J^T f + gradient + termination", "M/J products", "line search", "step + constraint update", "warm-start evaluations",
        "Hessian (assembly, or post + join wait)", "Cholesky factor + solve", "-"],
    2: ["kinematics+com", "collision", "make_constraint", "wait at join 1", "reference + solve", "-", "-", "rest of the step"],
}[args.map]
print("kernel %.2f ms; per-candidate cycles median %.3g" % (e.last_kernel_ms, np.median(tot)))
for k, n in enumerate(NAMES):
    if n != "-":
        print("  %-40s %5.1f%% of cycles  (%.0f cycles/step)" % (n, 100 * st[:, 4 + k].sum() / tot.sum(), st[:, 4 + k].mean() / 64))
if args.map == 0:
    print("  newton iterations/step %.2f  -> cycles per Newton iteration: all of solve %.0f, Hessian %.0f, Cholesky %.0f" % (
        st[:, 1].mean() / 64, st[:, 8:11].sum() / st[:, 1].sum(), st[:, 9].sum() / st[:, 1].sum(), st[:, 10].sum() / st[:, 1].sum()))
elif args.map == 1:
    rest = tot - st[:, 4:11].sum(1)
    print("  %-40s %5.1f%% of cycles  (%.0f cycles/step)" % ("outside the solve", 100 * rest.sum() / tot.sum(), rest.mean() / 64))
    print("  newton iterations/step %.2f, line-search evaluations/step %.2f (%.2f per iteration)" % (
        st[:, 1].mean() / 64, st[:, 11].mean() / 64, st[:, 11].sum() / st[:, 1].sum()))
else:
    print("  %-40s %5s   (%.0f cycles/step; the main warp's collision + constraint rows: %.0f)" % (
        "task warp: CRB+velocities+smooth forces", "", st[:, 9].mean() / 64, st[:, 5:7].sum(1).mean() / 64))
