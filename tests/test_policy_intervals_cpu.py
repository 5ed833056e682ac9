"""The policy step table of a rollout launch (mjpc_b200_host_policy_intervals) against the fp64 oracle, without a GPU.

For each step the table holds the rollout time, accumulated in double from the start time as mj_step accumulates it,
and the upper_bound of that time among the policy's absolute node times.  The kernels read nothing else to place a
spline knot or a feedback node, so this is where the interval the device uses is decided."""
import numpy as np
import pytest


def planner_knot_times(time0, dt, H, P, interp):
    """SamplingPlanner::UpdateNominalPolicy's knot times: the shift accumulated in double from the plan's time."""
    horizon = (H - 1) * dt
    shift = max(horizon / P, 1e-5) if interp == 0 else max(horizon / max(P - 1, 1), 1e-5)   # (P = 1: one knot)
    t, out = time0, []
    for _ in range(P):
        out.append(t)
        t += shift
    return np.array(out)


def agent_times(n, dt=0.01):
    t, out = 0.0, []
    for _ in range(n):
        out.append(t)
        t += dt
    return out


def cases():
    rng = np.random.default_rng(3)
    out = []
    for interp in (0, 1, 2):
        for time0 in agent_times(300)[::7] + [1000.25, 86400.0]:
            out.append((planner_knot_times(time0, 0.01, 26, 5, interp), time0, 0.01, 26))      # the Shadow task
            out.append((planner_knot_times(time0, 0.01, 64, 3, interp), time0, 0.01, 64))      # the Quadruped
    for P in (1, 2, 3, 64):
        out.append((planner_knot_times(0.37, 0.01, 64, P, 0), 0.37, 0.01, 64))
    kt = 0.37 + np.cumsum(rng.uniform(0.003, 0.07, 12))                       # non-uniform, first knot after time0
    out.append((kt, 0.37, 0.01, 64))
    out.append((kt[:4] - 0.1, 0.37, 0.01, 64))                                 # last knot before the end
    out.append((np.arange(64) * 0.005, 0.0, 0.005, 64))                        # nominal times as arange(H) dt
    out.append((np.array(agent_times(64, 0.005)) + 3.0, 3.0, 0.005, 64))       # the rollout's own times
    out.append((np.array([0.5]), 0.0, 0.1, 1))
    return out


def cubic(nodes, values, u, s):
    """the cubic Hermite sample the kernel forms from (upper, frac): finite-difference slopes at the two knots"""
    def slope(k):
        if k == 0:
            return (values[1] - values[0]) / (nodes[1] - nodes[0])
        if k == len(nodes) - 1:
            return (values[k] - values[k - 1]) / (nodes[k] - nodes[k - 1])
        return 0.5 * (values[k + 1] - values[k]) / (nodes[k + 1] - nodes[k]) + \
            0.5 * (values[k] - values[k - 1]) / (nodes[k] - nodes[k - 1])
    lo, dt = u - 1, nodes[u] - nodes[u - 1]
    return ((2 * s ** 3 - 3 * s ** 2 + 1) * values[lo] + (s ** 3 - 2 * s ** 2 + s) * dt * slope(lo) +
            (-2 * s ** 3 + 3 * s ** 2) * values[u] + (s ** 3 - s ** 2) * dt * slope(u))


def test_table_times_are_the_reference_clock():
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import host_policy_intervals
    build.build()
    for nodes, time0, dt, H in cases():
        times, _, _ = host_policy_intervals(nodes, time0, dt, H)
        ref, t = [], time0
        for _ in range(H):
            ref.append(t)
            t += dt
        assert np.array_equal(times, np.array(ref))


def test_table_intervals_match_the_oracle(oracle_lib):
    """upper gives FindInterval's bounds over every node and over all but the last (the nominal actions and gains), and
    the zero-order, linear and cubic samples of the fp64 spline at the table's time."""
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import host_policy_intervals
    build.build()
    rng = np.random.default_rng(0)
    checked = 0
    for nodes, time0, dt, H in cases():
        P = len(nodes)
        times, upper, frac = host_policy_intervals(nodes, time0, dt, H)
        values = rng.normal(size=(P, 3))
        for t in range(H):
            T = times[t]
            u = int(upper[t])
            assert u == int(np.searchsorted(nodes, T, side="right"))
            for length in (P, P - 1):
                if length < 1:
                    continue
                b = (0, 0) if u == 0 else (min(u - 1, length - 1), min(u, length - 1))
                assert b == tuple(oracle_lib.find_interval(nodes[:length], T)), (t, T, length)
            if 0 < u < P:
                ref = (T - nodes[u - 1]) / (nodes[u] - nodes[u - 1])
                assert frac[t] == np.float32(ref)
            else:
                assert frac[t] == 0
            for interp in (0, 1, 2):
                ref = oracle_lib.spline_sample(nodes, values, interp, T)
                if u == 0 or u == P or interp == 0:
                    mine = values[0] if u == 0 else values[P - 1] if u == P else values[u - 1]
                    assert np.array_equal(mine, ref)
                elif interp == 1:
                    np.testing.assert_allclose(values[u - 1] * (1 - frac[t]) + values[u] * frac[t], ref, atol=1e-6)
                else:
                    np.testing.assert_allclose(cubic(nodes, values, u, float(frac[t])), ref, atol=1e-6)
            checked += 1
    assert checked > 5000


@pytest.mark.parametrize("time0", [0.0, 1000.25, 86400.0])
def test_knot_coincident_steps_follow_double_time(time0):
    """Zero-order Shadow spacing: knots land on steps 5, 10, 15 and 20, and the step's knot is the one double time has
    reached (fp32 time relative to the start can sit one ulp below the knot)."""
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import host_policy_intervals
    build.build()
    nodes = planner_knot_times(time0, 0.01, 26, 5, 0)
    times, upper, _ = host_policy_intervals(nodes, time0, 0.01, 26)
    assert list(upper) == [int(np.searchsorted(nodes, T, side="right")) for T in times]
    assert list(upper[:5]) == [1] * 5
