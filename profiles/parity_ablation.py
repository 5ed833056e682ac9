#!/usr/bin/env python
"""Parity of the library selected by MJPC_B200_SO (default: the in-tree build) on BASELINE config 2 inputs:
teacher-forced per-step error, 256x64 return parity, Newton iterations, kernel time.  One JSON line.
Used for the -use_fast_math ablation:
  MJPC_B200_NO_FAST_MATH=1 MJPC_B200_SO=$PWD/mujoco_mpc_b200/csrc/libmjpc_b200_ieee.so python -m mujoco_mpc_b200.build
  MJPC_B200_SO=... python profiles/parity_ablation.py <label>
"""
import json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import get_model
from test_gpu_teacher_forced import _steady_state_inputs, _pct
from mujoco_mpc_b200.blob import to_blob
from mujoco_mpc_b200.engine import Engine
from oracle import pyoracle

label = sys.argv[1] if len(sys.argv) > 1 else "default"
m = get_model("quadruped")
N, H = 256, 64
state, mocap, knots, kt = _steady_state_inputs(m, N, H)
o64, o32 = pyoracle.Oracle(to_blob(m), m, 64), pyoracle.Oracle(to_blob(m), m, 32)
r = o64.rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=16, full=True)
nq = m.nq
S = r["states"][:, : H - 1].reshape(-1, nq + m.nv); U = r["actions"][:, : H - 1].reshape(-1, m.nu); T = r["times"][:, : H - 1].reshape(-1)
ref = o64.step_batch(S[:, :nq], S[:, nq:], U, mocap, T, nthreads=16)
f32 = o32.step_batch(S[:, :nq], S[:, nq:], U, mocap, T, nthreads=16)
e = Engine(m, N, H)
dev = e.step_batch(S[:, :nq], S[:, nq:], U, mocap, T)
ev = np.abs(dev["next_qvel"] - ref["next_qvel"]).max(1); ev32 = np.abs(f32["next_qvel"] - ref["next_qvel"]).max(1)
ms = []
for i in range(6):
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    ms.append(e.last_kernel_ms)
st = e.fetch_stats()
r32 = o32.rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=16, full=False)["returns"]
rel = np.abs(ret - r["returns"]) / np.abs(r["returns"]); floor = np.abs(r32 - r["returns"]) / np.abs(r["returns"])
out = {"label": label, "so": os.environ.get("MJPC_B200_SO", "in-tree"), "static": bool(e.last_kernel_static),
       "teacher_forced_steps": int(len(ev)), "dev_qvel_err_p50_p99_max": _pct(ev), "fp32_oracle_qvel_err_p50_p99_max": _pct(ev32),
       "count_mismatch_steps": int(((dev["ncon"] != ref["ncon"]) | (dev["nefc"] != ref["nefc"])).sum()),
       "newton_iters_step_batch": {"device": float(dev["niter"].mean()), "fp32_oracle": float(f32["niter"].mean()), "fp64_oracle": float(ref["niter"].mean())},
       "newton_iters_per_step_rollout": float(st[:, 1].sum() / (N * H)),
       "returns_rel_err_max": float(rel.max()), "returns_rel_err_median": float(np.median(rel)),
       "candidates_above_1e-4": int((rel > 1e-4).sum()), "fp32_oracle_candidates_above_1e-4": int((floor > 1e-4).sum()),
       "fp32_oracle_rel_max": float(floor.max()), "argmin_agrees": bool(int(order[0]) == int(np.argmin(r["returns"]))),
       "kernel_ms_256x64": float(np.mean(ms[2:]))}
print(json.dumps(out), flush=True)
e.close()
