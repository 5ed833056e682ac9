"""The profiled command: Quadruped 256x64 rollout through the C ABI on steady-state planner inputs
(profiles/inputs_quadruped_256x64.npz, written by tests/test_gpu_teacher_forced.py::_steady_state_inputs)."""
import sys, numpy as np
import os; R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model
from mujoco_mpc_b200.engine import Engine
m = get_model("quadruped")
e = Engine(m, 256, 64)
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
state, mocap, knots, kt = d["state"], d["mocap"], d["knots"], d["kt"]
ms = []
for i in range(int(sys.argv[1]) if len(sys.argv) > 1 else 2):
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, 64)
    ms.append(e.last_kernel_ms)
print("kernel ms", ms[-1], "min", min(ms), "static", e.last_kernel_static)
if len(sys.argv) > 2:
    np.save(sys.argv[2], ret)   # returns of this build (compared across experiment builds)
st = e.fetch_stats()
cyc = st[:, 0] / 1e6
print("per-candidate M cycles: min %.2f median %.2f max %.2f ; newton iters/step mean %.2f max-cand %.2f ; ncon/step %.2f nefc/step %.2f" % (
    cyc.min(), np.median(cyc), cyc.max(), st[:, 1].mean() / 64, st[:, 1].max() / 64, st[:, 2].mean() / 64, st[:, 3].mean() / 64))
