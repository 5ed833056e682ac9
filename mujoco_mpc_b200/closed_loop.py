"""Closed-loop MPC episodes of many plants at once: the reference's testspeed loop (mjpc/testspeed.cc:96-113) restated
for B episodes, one per problem of a batch planner, on a bank of device plants (engine.CppPlantBank).

Per physics step i, for every episode b, in the reference's order:
  1. the task's Transition, if given (it may move the mocap, replace the state and change the task state);
  2. planner.set_state(b, pre-step state, time, mocap): the plant's state, or with an estimator the filter's;
  3. ctrl_b = planner.action_from_policy(b, time) (the iLQG kinds also read the state);
  4. one plant step of every episode; its cost is CostValue of the pre-step residual (testspeed.cc:104);
  5. planner.optimize_policy() when i % steps_per_planning_iteration == 0, from the states set in 2.
With an estimator (a CppBatchEstimator of B filters on the plants' sensor range), every plant step is followed by one
filter update from the ctrl the plant applied (the commanded ctrl plus any control noise: the app's estimator reads the
noisy d->ctrl, app.cc:174), the plant's pre-step sensors (with the plant's measurement noise, set_sensor_noise) and its
mocap (app.cc:155-197); a planner with a state ensemble (set_state_ensemble) also gets the filter's covariance in 2.  A perturbation (a function of
the step index and the plants' times) may hold a wrench on every plant before a step, as the app applies the user's
force perturbation before each physics step (app.cc:323-326, 349-352)."""
from __future__ import annotations

import time as _time

import numpy as np

from .engine import PLANT_RUNNING


def synchronous_planning_cost(planner, plant, steps, steps_per_planning_iteration=4, transitions=None, estimator=None,
                              perturbation=None):
    """Run `steps` physics steps of plant.num_plants episodes with `planner` (a batch planner of as many problems),
    from the plants as reset() left them.  transitions: None or one Transition per plant (transition(time, qpos,
    qvel) -> (qpos, qvel, mocap) and task_state(), as transition.HumanoidTrackTransition).  perturbation: None or
    perturbation(i, time [B]) -> None or xfrc [B][nbody][6]; an array is held on plant b (plant.set_xfrc) from step i on.

    Returns dict(average_cost [B] (cost sum / steps of each plant), costs [steps][B], states [steps][B][nq+nv] and
    status [steps][B] after each step, final_status [B], wall_time and planning_time [s], x_realtime (B x simulated
    seconds / wall time))."""
    m = plant.m
    B, nq = plant.num_plants, m.nq
    spp = int(steps_per_planning_iteration)
    reads_state = getattr(planner, "action_reads_state", False)
    first = [plant.get(b) for b in range(B)]
    x = np.array([f["state"] for f in first], np.float32)
    t = np.array([f["time"] for f in first])
    status = np.array([f["status"] for f in first], np.int32)
    costs = np.zeros((steps, B), np.float32)
    states = np.zeros((steps, B, nq + m.nv), np.float32)
    statuses = np.zeros((steps, B), np.int32)
    total, count = np.zeros(B), np.zeros(B, np.int64)
    ctrl = np.zeros((B, m.nu), np.float32)
    planning = 0.0
    start = _time.perf_counter()
    for i in range(steps):
        xfrc = None if perturbation is None else perturbation(i, t.copy())
        if xfrc is not None:
            xfrc = np.asarray(xfrc, np.float32).reshape(B, m.nbody, 6)
            for b in range(B):
                plant.set_xfrc(b, xfrc[b])
        for b in range(B):
            if transitions is not None:
                q, v, mocap = transitions[b].transition(t[b], x[b, :nq].astype(float), x[b, nq:].astype(float))
                q, v = np.asarray(q, np.float32), np.asarray(v, np.float32)
                if np.array_equal(q, x[b, :nq]) and np.array_equal(v, x[b, nq:]):
                    plant.set(b, mocap=mocap)
                else:
                    plant.set(b, qpos=q, qvel=v, mocap=mocap)
                    x[b] = np.concatenate([q, v])
                ts = transitions[b].task_state()
                plant.set_task(b, task_state=ts)
                planner.set_task(b, task_state=ts)
            state = x[b] if estimator is None else estimator.state(b)
            state = np.asarray(state, float)
            planner.set_state(b, state, t[b], np.asarray(plant.mocap[b], float))
            if estimator is not None and getattr(planner, "state_members", 0):
                planner.set_state_covariance(b, estimator.covariance(b))
            if status[b] == PLANT_RUNNING:
                ctrl[b] = planner.action_from_policy(b, t[b], state) if reads_state else \
                    planner.action_from_policy(b, t[b])
        o = plant.step(ctrl)
        stepped = o["status"] == PLANT_RUNNING
        costs[i] = o["cost"]
        total[stepped] += o["cost"][stepped].astype(float)
        count[stepped] += 1
        x, t, status = o["state"].copy(), o["time"].copy(), o["status"].copy()
        states[i], statuses[i] = x, status
        if estimator is not None:
            applied = o.get("ctrl", ctrl)   # (a plant that reports no applied ctrl applied the commanded one)
            estimator.update(applied, o["sensordata"].astype(float), plant.mocap if m.nmocap else None)
        if i % spp == 0:
            t0 = _time.perf_counter()
            planner.optimize_policy()
            planning += _time.perf_counter() - t0
    wall = _time.perf_counter() - start
    return dict(average_cost=total / np.maximum(count, 1), costs=costs, states=states, status=statuses,
                final_status=status, wall_time=wall, planning_time=planning,
                x_realtime=B * steps * m.opt_timestep / wall)
