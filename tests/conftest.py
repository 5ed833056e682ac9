import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def mocap_of(m):
    if m.nmocap == 0:
        return np.zeros(0)
    return np.concatenate([np.concatenate([m.mocap_pos0[i], m.mocap_quat0[i]]) for i in range(m.nmocap)])


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


_MODELS = {}


def get_model(name, agent_timestep=True):
    from mujoco_mpc_b200 import models
    key = (name, agent_timestep)
    if key not in _MODELS:
        _MODELS[key] = models.load(name, agent_timestep=agent_timestep)
    return _MODELS[key]


@pytest.fixture(scope="session")
def quadruped():
    return get_model("quadruped")


def quadruped_inputs(m, N=16, H=64, seed=0, sigma=0.04, iteration=0):
    """Seeded synthetic planner inputs (SURVEY.md 8d): home keyframe, zero nominal, Philox noise."""
    from mujoco_mpc_b200.planner import candidate_knots
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    P = 3
    T = (H - 1) * m.opt_timestep
    kt = np.arange(P) * T / (P - 1)
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    knots = candidate_knots(np.zeros((P, m.nu)), sigma, cr, iteration, N, seed=0x5EED + seed)
    return state, mocap_of(m), knots, kt


class OracleBackend:
    """The CPU oracle behind the same five calls Engine exposes (tests + CPU baseline only)."""

    def __init__(self, m, threads=2, precision=64):
        from mujoco_mpc_b200.blob import to_blob
        from oracle import pyoracle
        self.m, self.po, self.threads = m, pyoracle, threads
        self.o = pyoracle.Oracle(to_blob(m), m, precision)
        self.last = None

    def rollout_spline(self, state, time, mocap, knots, kt, interp, H):
        r = self.o.rollout_spline(state, time, mocap, knots, kt, interp, H, nthreads=self.threads, full=True)
        self.last = r
        return r["returns"], r["failure"], np.argsort(r["returns"], kind="stable")

    def set_xfrc_noise(self, std, rate=1.0, seed=0):
        self.o.set_xfrc_noise(std, rate, seed)

    def set_differentiable(self, on=True):
        self.o.set_differentiable(on)

    def rollout_feedback(self, state, time, mocap, u_nom, x_nom, t_nom, gains, du, step_sizes, mode):
        r = self.o.rollout_feedback(state, time, mocap, u_nom, x_nom, t_nom, gains, du, step_sizes, mode, nthreads=self.threads)
        self.last = r
        return r["returns"], r["failure"], np.argsort(r["returns"], kind="stable")

    def fetch_trajectory(self, i):
        return {k: self.last[k][i] for k in ("states", "actions", "times", "residual", "costs", "trace")}

    def model_derivatives(self, x, u, t, mocap, tol, skip=0, mode=0):
        return self.o.model_derivatives(np.asarray(x, float), np.asarray(u, float), np.asarray(t, float), mocap, tol=tol,
                                        skip=skip, mode=mode, nthreads=self.threads)

    def cost_derivatives(self, residual, C, D):
        return self.o.cost_derivatives(np.asarray(residual, float), np.asarray(C, float), np.asarray(D, float))

    def backward_pass(self, A, B, cx, cu, cxx, cxu, cuu, actions, mu=0.0, reg_type=0, limits=1):
        cr = np.asarray(self.m.actuator_ctrlrange, float).reshape(-1, 2)
        return self.po.backward_pass(A, B, cx, cu, cxx, cxu, cuu, actions, cr, mu=mu, reg_type=reg_type, limits=limits)
