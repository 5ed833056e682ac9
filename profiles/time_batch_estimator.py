"""Time the batched Kalman and Unscented filters (mujoco_mpc_b200.estimator.CppBatchEstimator) against the single C++
filters, on the Quadruped scenario of tests/quadruped_filtering.py (21 sensors, 73 step rows per filter), for
B in {1, 8, 32, 64} filters.

Per kind and B, in one process:
  * batched: the wall time of one `update` of all B filters (host clock around the call, which ends in a stream
    synchronise), median over the timed updates of a free-running run along the plant;
  * single: the wall time of B `update`s of B single C++ filters (CppUnscented / CppKalman) over the same updates,
    and of the first filter's alone (`update` returns the state: one update plus one state read);
  * kernels: in a separate profiled pass (torch.profiler, CUDA activities), the mean kernel time of each launch of one
    batched update by kernel name, and the launches of each name per update.
The GPU's name and power limit are read in the same run.

usage: python profiles/time_batch_estimator.py [--updates 100] [--warmup 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from estimator_backends import mocap_vector  # noqa: E402
from quadruped_filtering import SENSOR_SD, plant  # noqa: E402

from mujoco_mpc_b200 import models  # noqa: E402
from mujoco_mpc_b200.estimator import CppBatchEstimator, CppKalman, CppUnscented  # noqa: E402

SINGLE = {"unscented": CppUnscented, "kalman": CppKalman}


def gpu_description():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def _batched(m, kind, B, X):
    f = CppBatchEstimator(m, kind, B)
    for b in range(B):
        f.reset(b, state=X[0])
        f.set_noise(b, sensor=np.full(f.nsensordata, SENSOR_SD ** 2))
    return f


def time_kind(m, kind, B, X, Y, U, updates, warmup):
    mc = mocap_vector(m)
    f = _batched(m, kind, B, X)
    singles = [SINGLE[kind](m) for _ in range(B)]
    for s in singles:
        s.reset(state=X[0])
        s.set_noise(sensor=np.full(s.nsensordata, SENSOR_SD ** 2))
    batch_ms, single_ms, one_ms = [], [], []
    for t in range(warmup + updates):
        u, y, mcs = (np.tile(a, (B, 1)) for a in (U[t], Y[t], mc))
        t0 = time.perf_counter()
        status = f.update(u, y, mcs)
        t1 = time.perf_counter()
        singles[0].update(U[t], Y[t], mc)
        t1a = time.perf_counter()
        for s in singles[1:]:
            s.update(U[t], Y[t], mc)
        t2 = time.perf_counter()
        assert (status == 0).all()
        if t >= warmup:
            batch_ms.append((t1 - t0) * 1e3)
            single_ms.append((t2 - t1) * 1e3)
            one_ms.append((t1a - t1) * 1e3)
    f.close()
    for s in singles:
        s.close()
    return dict(batched_update_ms_median=float(np.median(batch_ms)),
                batched_update_ms_p90=float(np.percentile(batch_ms, 90)),
                single_updates_ms_median=float(np.median(single_ms)),
                single_updates_ms_p90=float(np.percentile(single_ms, 90)),
                one_single_update_and_state_ms_median=float(np.median(one_ms)))


def kernel_times(m, kind, B, X, Y, U, updates):
    """Mean device time per launch of each kernel of a batched update, and launches per update, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    mc = mocap_vector(m)
    f = _batched(m, kind, B, X)
    for t in range(3):   # warm up outside the trace
        f.update(np.tile(U[t], (B, 1)), np.tile(Y[t], (B, 1)), np.tile(mc, (B, 1)))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(3, 3 + updates):
            f.update(np.tile(U[t], (B, 1)), np.tile(Y[t], (B, 1)), np.tile(mc, (B, 1)))
    f.close()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "DeviceType.CUDA" in str(ev.device_type) and "emcpy" not in ev.key \
                and "emset" not in ev.key:
            total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[ev.key] = dict(launches_per_update=ev.count / updates, ms_per_launch=total_us / ev.count / 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sizes", default="1,8,32,64")
    ap.add_argument("--out")
    a = ap.parse_args()
    m = models.load("quadruped")
    X, Y, U = plant(m)
    assert a.warmup + a.updates <= len(U) - 4
    res = dict(gpu=gpu_description(), results={})
    for kind in ("unscented", "kalman"):
        for B in (int(s) for s in a.sizes.split(",")):
            r = time_kind(m, kind, B, X, Y, U, a.updates, a.warmup)
            r["kernels"] = kernel_times(m, kind, B, X, Y, U, 20)
            res["results"]["%s/B=%d" % (kind, B)] = r
            print(kind, B, json.dumps(r), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_batch_estimator.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
