"""TEST INFRASTRUCTURE - measurement sensors on the CPU oracle (sensor_oracle/sensors.cc), ctypes binding.

Only tests/ and profiles/ import this; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libsensor_oracle.so")
_LIB = None
_dp = C.POINTER(C.c_double)


def build(force=False):
    srcs = [os.path.join(_HERE, "sensors.cc")] + [os.path.join(_HERE, "..", "oracle", f)
                                                  for f in ("physics.h", "model.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O3", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-o", _SO, srcs[0]])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        _LIB.sensor_oracle_create.restype = C.c_void_p
        _LIB.sensor_oracle_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
        _LIB.sensor_oracle_destroy.argtypes = [C.c_void_p]
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


class SensorOracle:
    """One-step oracle with the measurement sensors of each pre-step state (fp64 or fp32)."""

    def __init__(self, blob: bytes, model, precision=64):
        self.m, self._blob = model, blob
        self.h = C.c_void_p(lib().sensor_oracle_create(blob, len(blob), precision))
        if not self.h:
            raise RuntimeError("sensor_oracle_create failed (blob without sensor entries?)")

    def __del__(self):
        if getattr(self, "h", None):
            lib().sensor_oracle_destroy(self.h)
            self.h = None

    def step(self, qpos, qvel, ctrl, mocap, times, start, count, warmstart=None, xfrc=None):
        """B single steps; xfrc: None or xfrc_applied [B][nbody][6] for the step."""
        m = self.m
        q, v, u, mc, t, ws = _d(qpos), _d(qvel), _d(ctrl), _d(mocap), _d(times), _d(warmstart)
        xf = None if xfrc is None else np.ascontiguousarray(np.asarray(xfrc, np.float64).reshape(-1, 6 * m.nbody))
        B = q.shape[0]
        dim = int(np.sum(m.sensor_dim[start:start + count])) if count > 0 else 0
        o = dict(next_qpos=np.zeros((B, m.nq)), next_qvel=np.zeros((B, m.nv)), qacc=np.zeros((B, m.nv)),
                 sensordata=np.zeros((B, dim)))
        counts = np.zeros((B, 4), np.int32)
        rc = lib().sensor_oracle_step(self.h, B, _p(q), _p(v), _p(u), _p(ws), _p(mc), _p(t), int(start), int(count),
                                      _p(o["next_qpos"]), _p(o["next_qvel"]), _p(o["qacc"]), _p(o["sensordata"]),
                                      counts.ctypes.data_as(C.POINTER(C.c_int)), _p(xf))
        if rc != 0:
            raise ValueError("sensor_oracle_step: sensor range [%d, %d) not evaluated" % (start, start + count))
        o.update(ncon=counts[:, 0], nefc=counts[:, 1], niter=counts[:, 2], warning=counts[:, 3])
        return o
