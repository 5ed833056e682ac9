"""GPU: Agent::PlanIteration dispatches to its planner through the Planner interface (csrc/host/planner.h) - an Agent of
each kind plans exactly as the directly driven C++ planner with the same settings - and SetState with a NULL mocap keeps
the mocap given before."""
import numpy as np
import pytest

from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

H, TIMESTEP = 32, 0.01          # Agent: steps = 0.31 / 0.01 + 1; the quadruped's own timestep is 0.01
TIMES = (0.0, 0.013, 0.05, 0.2)


def _quadruped():
    m = get_model("quadruped")
    assert m.opt_timestep == TIMESTEP and m.nmocap > 0
    return m, np.concatenate([m.key_qpos[0], np.zeros(m.nv)])


def _pair(kind, m):
    """(CppAgent, directly driven planner with the settings the Agent passes to it, whether actions take the state)."""
    from mujoco_mpc_b200 import engine as E
    agent = lambda **kw: E.CppAgent(m, kind, horizon=0.31, timestep=TIMESTEP, seed=7, **kw)
    if kind == "gradient":
        return (agent(num_trajectory=8, num_spline_points=5, representation=1, fd_tolerance=3e-4),
                E.CppGradientPlanner(m, H, num_trajectory=8, num_spline_points=5, representation=1, fd_tolerance=3e-4),
                False)
    if kind == "ilqg":
        return (agent(ilqg_num_rollouts=6, ilqg_representation=1, fd_tolerance=3e-4),
                E.CppILQGPlanner(m, H, num_rollouts=6, representation=1, fd_tolerance=3e-4), True)
    if kind == "robust":       # 20 trajectories, 5 repetitions: both count 4 robust candidates
        return agent(num_trajectory=20), E.CppRobustPlanner(m, 20, H, seed=7), False
    return agent(num_trajectory=20), E.CppCrossEntropyPlanner(m, 20, H, seed=7), False


def _actions(planner, state, use_state):
    return [planner.action_from_policy(t, state) if use_state else planner.action_from_policy(t) for t in TIMES]


@pytest.mark.parametrize("kind", ["gradient", "ilqg", "robust", "cross_entropy"])
def test_agent_plans_as_the_direct_planner(kind):
    m, state = _quadruped()
    ag, direct, use_state = _pair(kind, m)
    assert ag.steps == H
    for p in (ag, direct):
        p.reset(); p.set_state(state, 0.0, mocap_of(m))
    for _ in range(3):
        ag.plan_iteration(); direct.optimize_policy()
    a_agent, a_direct = _actions(ag, state, use_state), _actions(direct, state, use_state)
    for t, x, y in zip(TIMES, a_agent, a_direct):
        np.testing.assert_allclose(x, y, atol=1e-12, err_msg=f"{kind} t={t}")
    ag.set_plan_enabled(False)
    assert ag.plan_iteration() >= 0
    for x, y in zip(_actions(ag, state, use_state), a_agent):
        np.testing.assert_array_equal(x, y)
    ag.close(); direct.close()


def test_agent_ilqs_actions_are_finite_and_in_range():
    from mujoco_mpc_b200.engine import CppAgent
    m, state = _quadruped()
    ag = CppAgent(m, "ilqs", horizon=0.31, timestep=TIMESTEP, num_trajectory=16, ilqg_num_rollouts=6)
    ag.reset(); ag.set_state(state, 0.0, mocap_of(m))
    for _ in range(3):
        assert ag.plan_iteration() >= 0
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    for t in TIMES:
        a = ag.action_from_policy(t, state)
        assert np.isfinite(a).all() and (a >= cr[:, 0] - 1e-12).all() and (a <= cr[:, 1] + 1e-12).all()
    ag.close()


@pytest.mark.parametrize("kind", ["sampling", "cross_entropy", "sample_gradient", "gradient", "ilqg"])
def test_null_mocap_keeps_the_previous_mocap(kind):
    from mujoco_mpc_b200 import engine as E
    m, state = _quadruped()
    make = {"sampling": lambda: E.CppSamplingPlanner(m, 16, H),
            "cross_entropy": lambda: E.CppCrossEntropyPlanner(m, 16, H),
            "sample_gradient": lambda: E.CppSampleGradientPlanner(m, 16, H, num_gradient=4),
            "gradient": lambda: E.CppGradientPlanner(m, H, num_trajectory=6),
            "ilqg": lambda: E.CppILQGPlanner(m, H, num_rollouts=6)}[kind]
    every, once = make(), make()
    mocap = mocap_of(m).reshape(-1, 7)
    mocap[:, :3] += 0.05                 # not the model's own mocap positions, so a lost value shows
    mocap = mocap.reshape(-1)
    for p in (every, once):
        p.reset()
    for it in range(3):
        every.set_state(state, 0.01 * it, mocap)
        once.set_state(state, 0.01 * it, mocap if it == 0 else None)
        every.optimize_policy(); once.optimize_policy()
        for key, value in every.result().items():
            np.testing.assert_array_equal(once.result()[key], value, err_msg=f"{kind} iteration {it} {key}")
    every.close(); once.close()
