"""Is the slowdown of two candidates on one SM instruction-fetch interference?  With S SMs, N = 2 S (two per SM on
every SM): (a) 2 S different candidates, (b) candidates i and i+S identical (they land on the same SM and execute the
same instruction stream in step) - if (b) runs at the speed of a candidate that is alone on its SM (N = S), the shared
resource is the instruction cache / fetch path.  Per-candidate times are in SM cycles."""
import sys, numpy as np
import torch
import os; R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model
from mujoco_mpc_b200.engine import Engine
m = get_model("quadruped")
d = np.load(os.path.join(R, "profiles", "inputs_quadruped_256x64.npz"))
k = d["knots"]
S = torch.cuda.get_device_properties(0).multi_processor_count
def run(kn, label):
    N = len(kn)
    e = Engine(m, N, 64)
    for i in range(3):
        e.rollout_spline(d["state"], 0.0, d["mocap"], kn, d["kt"], 2, 64)
    st = e.fetch_stats(); mc = st[:, 0] / 1e6; sm = st[:, 4]
    pair_same = np.mean([np.sum(sm == sm[i]) for i in range(N)])
    print("%-44s N=%3d kernel %.2f ms  per-candidate M cycles median %.2f max %.2f  (candidates per SM %.2f)" % (label, N, e.last_kernel_ms, np.median(mc), mc.max(), pair_same))
    same_sm = [sm[i] == sm[i + S] for i in range(N - S)] if N > S else []
    if same_sm: print("    candidate i and i+%d on the same SM: %d of %d" % (S, sum(same_sm), len(same_sm)))
    e.close()
run(k[:S], "alone (S different)")
run(np.concatenate([k[:S], k[256 - S:256]]), "two per SM, different")
run(np.concatenate([k[:S], k[:S]]), "two per SM, identical pairs (i, i+S)")
