"""CPU: the batched closed loop (mujoco_mpc_b200.closed_loop) drives its planner, plant and estimator in the order of
the reference's testspeed loop (mjpc/testspeed.cc:96-113), checked against stub objects that record their calls; and
without a device the plant entry points fail loudly or refuse NULL handles."""
import ctypes
import types

import numpy as np
import pytest

from mujoco_mpc_b200.closed_loop import synchronous_planning_cost

NQ, NV, NU, NM = 2, 2, 1, 1
DT = 0.01


class Log(list):
    def add(self, *entry):
        self.append(entry)


class StubPlant:
    """A bank of B plants whose state after a step is the ctrl + the step index; the cost of plant b's step is
    b + 0.5 + the step index.  Plant `diverge_at[b]`'s step at that index diverges instead."""

    def __init__(self, log, B, diverge_at=None):
        self.log, self.num_plants = log, B
        self.m = types.SimpleNamespace(nq=NQ, nv=NV, nu=NU, nmocap=NM, opt_timestep=DT)
        self.mocap = np.zeros((B, 7 * NM), np.float32)
        self.x = np.tile(np.arange(NQ + NV, dtype=np.float32), (B, 1))
        self.t = np.arange(B) * 0.5
        self.status = np.zeros(B, np.int32)
        self.sum, self.steps, self.k = np.zeros(B), np.zeros(B, int), 0
        self.diverge_at = diverge_at or {}

    def get(self, b):
        return dict(state=self.x[b].copy(), time=self.t[b], status=int(self.status[b]), cost_sum=self.sum[b],
                    steps=self.steps[b])

    def set(self, b, qpos=None, qvel=None, mocap=None):
        self.log.add("plant.set", b, qpos is not None, mocap is not None)
        if qpos is not None:
            self.x[b, :NQ] = qpos
        if qvel is not None:
            self.x[b, NQ:] = qvel
        if mocap is not None:
            self.mocap[b] = mocap

    def set_task(self, b, task_state=None, **kw):
        self.log.add("plant.set_task", b, tuple(task_state))

    def step(self, ctrl):
        self.log.add("step", self.k, np.array(ctrl, np.float32).copy())
        cost = np.zeros(self.num_plants, np.float32)
        for b in range(self.num_plants):
            if self.status[b]:
                continue
            if self.diverge_at.get(b) == self.k:
                self.status[b] = 1
                continue
            cost[b] = b + 0.5 + self.k
            self.x[b] = ctrl[b, 0] + self.k
            self.t[b] += DT
            self.sum[b] += cost[b]
            self.steps[b] += 1
        self.k += 1
        return dict(state=self.x.copy(), time=self.t.copy(), cost=cost, status=self.status.copy(),
                    sensordata=np.full((self.num_plants, 3), self.k, np.float32))


class StubPlanner:
    def __init__(self, log, reads_state=False):
        self.log = log
        if reads_state:
            self.action_reads_state = True

    def set_state(self, b, state, time, mocap):
        self.log.add("set_state", b, np.array(state).copy(), time)

    def set_task(self, b, task_state=None, **kw):
        self.log.add("planner.set_task", b, tuple(task_state))

    def action_from_policy(self, b, time, *state):
        self.log.add("action", b, time, len(state))
        return np.array([10.0 * b + time])

    def optimize_policy(self):
        self.log.add("plan")


class StubEstimator:
    def __init__(self, log, B):
        self.log, self.B = log, B

    def state(self, b):
        return np.full(NQ + NV, 100.0 + b)

    def update(self, ctrl, sensor, mocap):
        self.log.add("estimator.update", np.array(ctrl).copy(), np.array(sensor).copy())


class StubTransition:
    def __init__(self, log, b):
        self.log, self.b = log, b

    def transition(self, time, qpos, qvel):
        self.log.add("transition", self.b, time)
        # plant 1 is put back to a fixed pose at every step; plant 0 keeps its state
        q = np.full(NQ, 7.0) if self.b == 1 else qpos
        return q, qvel, np.full(7 * NM, self.b, float)

    def task_state(self):
        return (float(self.b), 0.25)


def kinds(log):
    return [e[0] for e in log]


@pytest.mark.parametrize("spp", [1, 3])
def test_order_and_planning_steps(spp):
    log, B, steps = Log(), 2, 7
    synchronous_planning_cost(StubPlanner(log), StubPlant(log, B), steps, spp)
    expect = []
    for i in range(steps):
        expect += ["set_state", "action"] * B + ["step"] + (["plan"] if i % spp == 0 else [])
    assert kinds(log) == expect
    # set_state hands over the pre-step state and time: step 0 the plant's initial ones, then the last step's output
    st = [e for e in log if e[0] == "set_state"]
    assert np.array_equal(st[0][2], np.arange(4.0)) and st[0][3] == 0.0 and st[1][3] == 0.5
    steps_ = [e for e in log if e[0] == "step"]
    assert np.array_equal(st[2][2], np.full(4, steps_[0][2][0, 0] + 0))
    assert st[2][3] == DT and st[3][3] == 0.5 + DT
    # the action is taken at the plant's time, without the state for the sampling kinds
    acts = [e for e in log if e[0] == "action"]
    assert all(a[3] == 0 for a in acts) and acts[1][2] == 0.5
    assert np.allclose(steps_[0][2][:, 0], [0.0, 10.5])


def test_feedback_kinds_receive_the_state():
    log = Log()
    synchronous_planning_cost(StubPlanner(log, reads_state=True), StubPlant(log, 2), 3, 2)
    assert all(e[3] == 1 for e in log if e[0] == "action")


def test_costs_and_averages():
    log, B, steps = Log(), 3, 6
    plant = StubPlant(log, B, diverge_at={2: 4})
    out = synchronous_planning_cost(StubPlanner(log), plant, steps, 4)
    for b in range(B):
        n = plant.steps[b]
        assert np.array_equal(out["costs"][:n, b], np.float32(b + 0.5 + np.arange(n)))
        assert out["average_cost"][b] == plant.sum[b] / n
    assert plant.steps.tolist() == [6, 6, 4]
    assert out["final_status"].tolist() == [0, 0, 1] and out["status"][4].tolist() == [0, 0, 1]
    assert out["costs"][4, 2] == 0 and out["x_realtime"] > 0 and out["planning_time"] <= out["wall_time"]


def test_estimator_state_replaces_the_plant_state():
    log, B = Log(), 2
    synchronous_planning_cost(StubPlanner(log), StubPlant(log, B), 3, 1, estimator=StubEstimator(log, B))
    assert kinds(log)[:6] == ["set_state", "action", "set_state", "action", "step", "estimator.update"]
    for e in log:
        if e[0] == "set_state":
            assert np.array_equal(e[2], np.full(4, 100.0 + e[1]))
    up = [e for e in log if e[0] == "estimator.update"]
    st = [e for e in log if e[0] == "step"]
    assert all(np.array_equal(u[1], s[2]) for u, s in zip(up, st))          # that step's ctrl
    assert np.array_equal(up[1][2], np.full((B, 3), 2.0))                    # that step's sensors


def test_transitions_run_first():
    log, B = Log(), 2
    tr = [StubTransition(log, b) for b in range(B)]
    synchronous_planning_cost(StubPlanner(log), StubPlant(log, B), 2, 1, transitions=tr)
    per_plant = ["transition", "plant.set", "plant.set_task", "planner.set_task", "set_state", "action"]
    assert kinds(log) == (per_plant * B + ["step", "plan"]) * 2
    sets = [e for e in log if e[0] == "plant.set"]
    assert sets[0][1:] == (0, False, True) and sets[1][1:] == (1, True, True)   # a changed state is written through
    st = [e for e in log if e[0] == "set_state"]
    assert np.array_equal(st[1][2][:NQ], [7.0, 7.0])                            # ... and handed to the planner


def test_plant_entry_points_without_device():
    """No CUDA device: creating the bank fails with MJPC_B200_ERR_CUDA; every plant call refuses a NULL handle."""
    import torch
    from mujoco_mpc_b200.engine import CppPlantBank, EngineError, load_library
    lib = load_library()
    for name, args in (("init", (1, 0, 0)), ("reset", (0, None, None, ctypes.c_double(0.0), None)),
                       ("set", (0, None, None, None)), ("set_task", (0, None, None, None)),
                       ("step", (None,) * 6), ("get", (0,) + (None,) * 7)):
        assert getattr(lib, f"mjpc_b200_plant_{name}")(None, *args) == -1, name
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from conftest import get_model
    with pytest.raises(EngineError) as e:
        CppPlantBank(get_model("particle"), 2)
    assert "(-4)" in str(e.value)
