"""Kernel-time probe: Quadruped 256x64 rollout (zero nominal + steady nominal), prints device ms and stats."""
import os, sys
import numpy as np
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model, mocap_of, quadruped_inputs
from mujoco_mpc_b200.engine import Engine
from mujoco_mpc_b200.planner import SamplingPlanner, candidate_knots
m = get_model("quadruped")
e = Engine(m, 256, 64)
state, mocap, knots, kt = quadruped_inputs(m, N=256, H=64)
for i in range(3):
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, 64)
st = e.fetch_stats()
print("%s static=%d zero-nominal: kernel %.2f ms  newton/step %.2f  checksum %.6f" % (os.environ.get("MJPC_B200_SO", "default")[-24:], e.last_kernel_static, e.last_kernel_ms, st[:, 1].mean() / 64, float(ret.sum())))
pl = SamplingPlanner(m, e, num_trajectory=256, horizon=64)
pl.reset(); pl.set_state(state, 0.0, mocap)
for _ in range(30):
    pl.optimize_policy()
pl.make_candidates()
k2 = candidate_knots(pl.values, pl.sigma, pl.ctrlrange, 99, 256)
for i in range(3):
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, k2, pl.times, 2, 64)
st = e.fetch_stats()
cyc = st[:, 0] / 1e6
print("   steady-nominal: kernel %.2f ms  newton/step %.2f  per-cand M cycles min/med/max %.1f/%.1f/%.1f  best return %.4f" % (
    e.last_kernel_ms, st[:, 1].mean() / 64, cyc.min(), np.median(cyc), cyc.max(), float(ret.min())))
