"""Kernel time of the Quadruped 64-step rollout as a function of the number of candidates (1 CTA each):
up to one candidate per SM every CTA has an SM to itself, above that SMs are shared by two CTAs.
Per-candidate times are in SM cycles (clock-independent)."""
import os, sys
import numpy as np
import torch
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import get_model, quadruped_inputs
from mujoco_mpc_b200.engine import Engine
m = get_model("quadruped")
e = Engine(m, 1024, 64)
S = torch.cuda.get_device_properties(0).multi_processor_count
for N in sorted({32, S // 2, S, 200, 256, 2 * S, 3 * S, 4 * S, 1024}):
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=64)
    ms = []
    for i in range(4):
        ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, 64)
        ms.append(e.last_kernel_ms)
    st = e.fetch_stats()[:N]
    cyc = st[:, 0] / 1e6
    print("N=%4d kernel %.2f ms (%.3e env-steps/s) per-candidate M cycles min/med/max %.1f/%.1f/%.1f newton/step %.2f" % (
        N, np.mean(ms[1:]), N * 64 / (np.mean(ms[1:]) * 1e-3), cyc.min(), np.median(cyc), cyc.max(), st[:, 1].mean() / 64))
