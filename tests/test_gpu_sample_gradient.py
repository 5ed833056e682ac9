"""GPU: the Sample Gradient planner (mjpc/planners/sample_gradient/planner.cc) - the C++ host class through its C
wrappers against the Python mirror driving the same rollout ABI, the reference's behavioural criterion on the particle,
and the Agent glue for agent_planner = 6."""
import numpy as np
import pytest

from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu


def test_cpp_sample_gradient_planner_matches_python_mirror():
    """Same injected noise, same launches: same winner and winner type, installed knots, gradient candidates and
    gradient over several iterations (the first computes and caches the fitness weights, the later ones reuse them)."""
    from mujoco_mpc_b200.engine import CppSampleGradientPlanner, Engine
    from mujoco_mpc_b200.planner import SampleGradientPlanner
    m = get_model("quadruped")
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    mocap = mocap_of(m)
    N, G, H, f = 48, 8, 32, 0.6
    cpp = CppSampleGradientPlanner(m, N, H, num_gradient=G, gradient_filter=f)
    e = Engine(m, N, H)
    py = SampleGradientPlanner(m, e, num_trajectory=N, horizon=H, num_gradient=G, gradient_filter=f)
    cpp.reset(np.zeros(m.nu)); py.reset(np.zeros(m.nu))
    types = []
    for it in range(5):
        t = 0.01 * it
        cpp.set_state(state, t, mocap); py.set_state(state, t, mocap)
        rc = cpp.optimize_policy()
        ret, fail = py.optimize_policy()
        assert not fail.any()
        np.testing.assert_allclose(rc["returns"], ret, rtol=1e-5)
        assert (rc["winner"], rc["winner_type"]) == (py.winner, py.winner_type), it
        np.testing.assert_allclose(rc["knot_times"], py.times, atol=1e-12)
        np.testing.assert_allclose(rc["knots"], py.values, atol=1e-6)
        np.testing.assert_allclose(rc["gradient"], py.gradient, atol=1e-6)
        assert rc["gradient_knots"].shape == (G, py.P, m.nu)
        np.testing.assert_allclose(rc["gradient_knots"], py.gradient_knots, atol=1e-6)
        assert list(rc["order"]) == list(py.order), it
        assert abs(rc["improvement"] - py.improvement) < 1e-5
        types.append(rc["winner_type"])
    print("winner types", types)
    for t in (0.0, 0.02, 0.1):
        np.testing.assert_allclose(cpp.action_from_policy(t), py.action_from_policy(t), atol=1e-6)
    # previous_policy is never updated after Reset (the reference's behaviour): the zero plan
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    np.testing.assert_array_equal(cpp.action_from_policy(0.02, use_previous=True), np.clip(np.zeros(m.nu), cr[:, 0], cr[:, 1]))
    cpp.close(); e.close()


def test_cpp_sample_gradient_particle_reaches_goal():
    """The bar of test_sampling_particle_reaches_goal, on the C++ planner: the installed policy, rolled out from the
    start state, ends at the mocap goal."""
    from mujoco_mpc_b200.engine import CppSampleGradientPlanner, Engine
    m = get_model("particle")
    H = 11
    pl = CppSampleGradientPlanner(m, 16, H, num_gradient=4, gradient_filter=0.5)
    pl.reset(); pl.set_state(np.zeros(4), 0.0, mocap_of(m))
    for _ in range(150):
        r = pl.optimize_policy()
        assert r["improvement"] >= 0
    e = Engine(m, 1, H)
    e.rollout_spline(np.zeros(4), 0.0, mocap_of(m), r["knots"][None], r["knot_times"], int(m.numeric.get("sampling_representation", [2])[0]), H)
    tr = e.fetch_trajectory(0)
    assert np.abs(tr["states"][-1, :2] - mocap_of(m)[:2]).max() < 0.1
    assert (np.abs(tr["actions"]) <= 1 + 1e-6).all()
    pl.close(); e.close()


def test_agent_sample_gradient_glue():
    """Agent::PlanIteration with agent_planner = 6 equals the directly driven C++ planner; with planning disabled the
    iteration rolls out the nominal and leaves the policy as it was."""
    from mujoco_mpc_b200.engine import CppAgent, CppSampleGradientPlanner
    m = get_model("quadruped")
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    ag = CppAgent(m, "sample_gradient", horizon=0.31, timestep=0.01, num_trajectory=16, num_gradient=4, gradient_filter=0.5)
    assert ag.steps == 32
    ag.reset(); ag.set_state(state, 0.0, mocap_of(m))
    ag.plan_iteration(); ag.plan_iteration()
    direct = CppSampleGradientPlanner(m, 16, 32, num_gradient=4, gradient_filter=0.5)
    direct.reset(); direct.set_state(state, 0.0, mocap_of(m))
    direct.optimize_policy(); direct.optimize_policy()
    for t in (0.0, 0.02, 0.2):
        np.testing.assert_allclose(ag.action_from_policy(t), direct.action_from_policy(t), atol=1e-12)
    ag.set_plan_enabled(False)
    before = [ag.action_from_policy(t) for t in (0.0, 0.02, 0.2)]
    assert ag.plan_iteration() == 0
    for t, a in zip((0.0, 0.02, 0.2), before):
        np.testing.assert_array_equal(ag.action_from_policy(t), a)
    ag.close(); direct.close()
    # right after Reset the plan is empty: the nominal rollout is the clamped zero action
    ag2 = CppAgent(m, "sample_gradient", horizon=0.31, timestep=0.01, num_trajectory=8, num_gradient=2)
    ag2.reset(); ag2.set_state(state, 0.0, mocap_of(m)); ag2.set_plan_enabled(False)
    assert ag2.plan_iteration() == 0
    cr = np.asarray(m.actuator_ctrlrange, float).reshape(-1, 2)
    np.testing.assert_array_equal(ag2.action_from_policy(0.05), np.clip(np.zeros(m.nu), cr[:, 0], cr[:, 1]))
    ag2.close()
