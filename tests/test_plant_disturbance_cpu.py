"""CPU: the plants' disturbances without a device - the new entry points refuse NULL handles, the noise stream's numpy
restatement (tests/plant_noise.py) gives a known sequence, and the closed loop holds a perturbation's wrench on every
plant before the right steps and hands the estimator the ctrl the plant applied."""
import ctypes
import types

import numpy as np
import pytest

import plant_noise as PN
from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
from mujoco_mpc_b200.planner import philox4x32

NQ, NV, NU, NBODY = 2, 2, 1, 2
DT = 0.01


def test_entry_points_refuse_null_handle_and_bank_needs_a_device():
    import torch
    from mujoco_mpc_b200.engine import CppPlantBank, EngineError, load_library
    lib = load_library()
    d = ctypes.c_double
    assert lib.mjpc_b200_plant_set_disturbance(None, 0, d(0.1), d(1.0), d(0.0), d(1.0), ctypes.c_uint32(0)) == -1
    assert lib.mjpc_b200_plant_set_xfrc(None, 0, None) == -1
    assert lib.mjpc_b200_plant_get_disturbance(None, 0, None, None) == -1
    buf = (ctypes.c_float * 4)()
    assert lib.mjpc_b200_plant_last_ctrl(None, buf) == -1
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from conftest import get_model
    with pytest.raises(EngineError) as e:
        CppPlantBank(get_model("particle"), 2)
    assert "(-4)" in str(e.value)


def test_philox_known_answers():
    """The generator under the restatement is Philox4x32-10 (Random123's known-answer vectors)."""
    z = philox4x32(np.zeros((1, 4), np.uint32), (0, 0))[0]
    assert [int(x) for x in z] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    z = philox4x32(np.array([[0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344]], np.uint32), (0xA4093822, 0x299F31D0))[0]
    assert [int(x) for x in z] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_plant_noise_known_sequence():
    """Key (seed, 2), counter (step, 0, element, tag): pinned values for seed 7 and seed 0."""
    np.testing.assert_allclose(PN.plant_normal(7, 0, 4, PN.TAG_CTRL),
                               [-0.0262050847, -0.1101330004, 0.4166716406, -0.1590399321], atol=1e-9)
    np.testing.assert_allclose(PN.plant_normal(7, 3, 2, PN.TAG_XFRC), [1.1348436579, -0.6132927881], atol=1e-9)
    np.testing.assert_allclose(PN.plant_normal(0, 0, 2, PN.TAG_CTRL), [0.8785946218, 1.1438509817], atol=1e-9)
    # the key word 2 keeps the plant away from the rollouts' stream (key word 1) with the same seed and counter
    ctr = np.array([[0, 0, e, PN.TAG_XFRC] for e in range(8)], np.uint32)
    assert not np.array_equal(philox4x32(ctr, (7, 2)), philox4x32(ctr, (7, 1)))
    # the tags and the steps are distinct streams
    assert not np.allclose(PN.plant_normal(7, 0, 4, PN.TAG_CTRL), PN.plant_normal(7, 0, 4, PN.TAG_XFRC))
    assert not np.allclose(PN.plant_normal(7, 0, 4, PN.TAG_CTRL), PN.plant_normal(7, 1, 4, PN.TAG_CTRL))


def test_ou_restatement_is_the_app_recursion():
    """n_k = r n_{k-1} + s z_k from 0, r = exp(-dt / rate), s = std sqrt(1 - r^2): stationary variance std^2."""
    std, rate, dt = 0.3, 0.05, 0.002
    x = PN.ou_states(11, 3, 5, std, rate, dt, PN.TAG_CTRL)
    r = np.exp(-dt / rate); s = std * np.sqrt(1 - r * r)
    np.testing.assert_allclose(x[0], s * PN.plant_normal(11, 0, 5, PN.TAG_CTRL), rtol=1e-15)
    np.testing.assert_allclose(x[2], r * x[1] + s * PN.plant_normal(11, 2, 5, PN.TAG_CTRL), rtol=1e-15)
    long = PN.ou_states(3, 4000, 4, std, rate, dt, PN.TAG_XFRC)[1000:]   # past ~40 time constants
    assert abs(long.std() / std - 1) < 0.15


class Log(list):
    def add(self, *entry):
        self.append(entry)


class DisturbedStubPlant:
    """A bank of B plants that applies the commanded ctrl + 0.25 (b + 1) and reports it as the applied ctrl; its
    sensors are the step index.  set_xfrc calls are logged."""

    def __init__(self, log, B):
        self.log, self.num_plants, self.k = log, B, 0
        self.m = types.SimpleNamespace(nq=NQ, nv=NV, nu=NU, nmocap=0, nbody=NBODY, opt_timestep=DT)
        self.mocap = np.zeros((B, 0), np.float32)
        self.x, self.t = np.zeros((B, NQ + NV), np.float32), np.zeros(B)

    def get(self, b):
        return dict(state=self.x[b].copy(), time=self.t[b], status=0)

    def set_xfrc(self, b, xfrc=None):
        self.log.add("set_xfrc", self.k, b, None if xfrc is None else np.array(xfrc).copy())

    def step(self, ctrl):
        B = self.num_plants
        applied = np.asarray(ctrl, np.float32) + 0.25 * (np.arange(B, dtype=np.float32)[:, None] + 1)
        self.log.add("step", self.k, np.array(ctrl, np.float32).copy(), applied.copy())
        self.k += 1
        self.t += DT
        return dict(state=self.x.copy(), time=self.t.copy(), cost=np.zeros(B, np.float32), status=np.zeros(B, np.int32),
                    sensordata=np.full((B, 3), self.k, np.float32), ctrl=applied)


class StubPlanner:
    def set_state(self, b, state, time, mocap):
        pass

    def action_from_policy(self, b, time):
        return np.array([10.0 * b + time])

    def optimize_policy(self):
        pass


class StubEstimator:
    def __init__(self, log):
        self.log = log

    def state(self, b):
        return np.zeros(NQ + NV)

    def update(self, ctrl, sensor, mocap):
        self.log.add("estimator.update", np.array(ctrl).copy())


def test_perturbation_is_held_before_the_right_steps():
    log, B, steps = Log(), 3, 6
    seen = []

    def push(i, time):
        seen.append((i, time.copy()))
        if i == 2:
            return np.ones((B, NBODY, 6)) * np.arange(B)[:, None, None]
        if i == 4:
            return np.zeros((B, NBODY, 6))
        return None

    synchronous_planning_cost(StubPlanner(), DisturbedStubPlant(log, B), steps, 1, perturbation=push)
    # asked before every step with the plants' pre-step times
    assert [s[0] for s in seen] == list(range(steps))
    assert all(np.allclose(s[1], DT * s[0]) and s[1].shape == (B,) for s in seen)
    sets = [e for e in log if e[0] == "set_xfrc"]
    assert [(e[1], e[2]) for e in sets] == [(2, b) for b in range(B)] + [(4, b) for b in range(B)]
    for e in sets[:B]:
        assert e[3].shape == (NBODY, 6) and np.all(e[3] == e[2])
    assert all(np.all(e[3] == 0) for e in sets[B:])
    # each step's set_xfrc calls come right before that step
    order = [(e[0], e[1]) for e in log]
    assert order.index(("set_xfrc", 2)) == order.index(("step", 2)) - B


def test_estimator_receives_the_applied_ctrl():
    log, B = Log(), 2
    synchronous_planning_cost(StubPlanner(), DisturbedStubPlant(log, B), 4, 1, estimator=StubEstimator(log))
    st = [e for e in log if e[0] == "step"]
    up = [e for e in log if e[0] == "estimator.update"]
    assert len(st) == len(up) == 4
    for s, u in zip(st, up):
        assert np.array_equal(u[1], s[3]) and not np.array_equal(u[1], s[2])
