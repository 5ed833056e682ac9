"""Where the 256 one-warp CTAs of the Quadruped 256x64 launch run: SM, hardware warp slot (slot % 4 = scheduler), and how a
candidate's duration depends on sharing its SM / its scheduler with another candidate."""
import sys, numpy as np
import os; R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model
from mujoco_mpc_b200.engine import Engine
m = get_model("quadruped")
N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
e = Engine(m, N, 64)
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
kn = np.concatenate([d["knots"]] * ((N + 255) // 256))[:N]
for i in range(3):
    e.rollout_spline(d["state"], 0.0, d["mocap"], kn, d["kt"], 2, 64)
st = e.fetch_stats()
ms = st[:, 0] / 1e6; sm = st[:, 4]; slot = st[:, 5]; it = st[:, 1] / 64   # ms: M SM cycles
print("kernel %.2f ms; SMs used %d; slots seen %s" % (e.last_kernel_ms, len(set(sm)), sorted(set(slot))))
alone = np.array([np.sum(sm == s) == 1 for s in sm])
same_sched = np.zeros(N, bool)
for s in set(sm):
    idx = np.nonzero(sm == s)[0]
    if len(idx) > 1:
        sch = slot[idx] % 4
        for a in idx:
            same_sched[a] = np.sum(sch == slot[a] % 4) > 1
per_iter = ms / it
for name, mask in (("alone on its SM", alone), ("shares SM, own scheduler", ~alone & ~same_sched), ("shares SM and scheduler", same_sched)):
    if mask.any():
        print("%-28s n=%3d  M cycles median %.2f max %.2f | M cycles per (Newton iteration/step) median %.3f" % (name, mask.sum(), np.median(ms[mask]), ms[mask].max(), np.median(per_iter[mask])))
