"""Interleaved A/B of the co-resident pair synchronisation (MJPC_B200_PAIR_SYNC=0/1) at N candidates; also checks that
the returns are bitwise the same."""
import os, sys, numpy as np
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model
from mujoco_mpc_b200.engine import Engine
m = get_model("quadruped")
N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
e = Engine(m, N, 64)
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
kn = np.concatenate([d["knots"]] * ((N + 255) // 256))[:N]
modes = ("0", "1")   # off, meet at every time step
ms = {k: [] for k in modes}; ret = {}
for rep in range(12):
    for on in modes:
        os.environ["MJPC_B200_PAIR_SYNC"] = on
        r, _, _ = e.rollout_spline(d["state"], 0.0, d["mocap"], kn, d["kt"], 2, 64)
        ret[on] = r
        if rep >= 2: ms[on].append(e.last_kernel_ms)
    if rep == 11:
        st = e.fetch_stats(); c = st[:, 0] / 1e6
        print("   (last mode) per-candidate M cycles min %.2f median %.2f max %.2f" % (c.min(), np.median(c), c.max()))
for k, v in ms.items():
    print("N=%d pair sync %s: kernel ms min %.3f median %.3f max %.3f" % (N, k, min(v), np.median(v), max(v)))
print("returns bitwise equal:", all(np.array_equal(ret[modes[0]], ret[k]) for k in modes))
