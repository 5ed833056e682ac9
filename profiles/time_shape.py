"""Kernel ms of one static shape at N candidates (12 launches, first two dropped): python profiles/time_shape.py wide|plain [N]"""
import os, sys, numpy as np
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model
from mujoco_mpc_b200.engine import Engine
os.environ["MJPC_B200_SHAPE"] = sys.argv[1]   # wide | plain
N = int(sys.argv[2]) if len(sys.argv) > 2 else 256
m = get_model("quadruped")
e = Engine(m, N, 64)
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
kn = np.concatenate([d["knots"]] * ((N + 255) // 256))[:N]
ms = []
for rep in range(12):
    e.rollout_spline(d["state"], 0.0, d["mocap"], kn, d["kt"], 2, 64)
    if rep >= 2: ms.append(e.last_kernel_ms)
st = e.fetch_stats(); c = st[:, 0] / 1e6
print("%s N=%d %s: kernel ms min %.3f median %.3f | per-candidate M cycles min %.2f median %.2f max %.2f" % (os.environ.get("MJPC_B200_SO", "default")[-12:], N, sys.argv[1], min(ms), np.median(ms), c.min(), np.median(c), c.max()))
