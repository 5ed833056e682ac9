"""CPU: the host twin of an initial-state ensemble's members (mjpc_b200_host_state_member), which the device's
state_sample_kernel must equal to float rounding: member 0 is the mean, a zero covariance gives the mean for every
member, a quaternion member is estimator.integrate_pos of L z and stays unit-norm, and the empirical covariance of many
members is the covariance given.  Also the NULL-handle refusals of the new entry points."""

import numpy as np
import pytest

from conftest import get_model

BAD_ARGUMENT = -1


def _model():
    return get_model("quadruped")


def _mean(m):
    rng = np.random.default_rng(3)
    v = 0.1 * rng.standard_normal(m.nv)
    return np.concatenate([np.asarray(m.key_qpos[0], float), v]).astype(np.float32).astype(float)


def _member(m, x, P, k, seed=7, iteration=0, problem=0):
    from mujoco_mpc_b200.engine import host_state_member
    return host_state_member(m, x, P, seed, iteration, problem, k)


def _correlated(n, seed=1, scale=1e-2):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    return scale * (A @ A.T / n + 0.1 * np.eye(n))


def test_member_zero_is_the_mean():
    m = _model()
    x = _mean(m)
    out = _member(m, x, _correlated(2 * m.nv), 0)
    assert out.tobytes() == x.tobytes()


def test_zero_covariance_gives_the_mean_for_every_member():
    m = _model()
    x = _mean(m)
    P = np.zeros((2 * m.nv, 2 * m.nv))
    for k in range(8):
        assert _member(m, x, P, k).tobytes() == x.tobytes(), k


def _z(seed, iteration, problem, k, n):
    """The draw restated in numpy: Philox4x32-10, key (seed + problem, 3), counter (iteration, k, element, 'BELF'),
    Box-Muller in fp64 on the first two words."""
    from mujoco_mpc_b200.planner import philox4x32
    ctr = np.array([[iteration, k, e, 0x42454C46] for e in range(n)], np.uint32).reshape(n, 4)
    r = philox4x32(ctr, ((seed + problem) & 0xFFFFFFFF, 3))
    u1 = (r[:, 0].astype(np.float64) + 0.5) / 4294967296.0
    u2 = (r[:, 1].astype(np.float64) + 0.5) / 4294967296.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def test_a_quaternion_member_is_integrate_pos_of_l_z():
    from mujoco_mpc_b200 import estimator
    m = _model()
    assert 0 in list(m.jnt_type)   # the Quadruped's trunk is a free joint
    x = _mean(m)
    n = 2 * m.nv
    P = _correlated(n, seed=4, scale=1e-1)
    out = _member(m, x, P, 3, seed=11, iteration=5, problem=2)
    dx = np.linalg.cholesky(0.5 * (P + P.T)) @ _z(11, 5, 2, 3, n)
    np.testing.assert_allclose(out[:m.nq], estimator.integrate_pos(m, x[:m.nq], dx[:m.nv], 1.0), rtol=0, atol=1e-12)
    np.testing.assert_allclose(out[m.nq:], x[m.nq:] + dx[m.nv:], rtol=0, atol=1e-12)
    for j in range(m.njnt):
        if m.jnt_type[j] == 0:
            a = m.jnt_qposadr[j] + 3
            assert abs(np.linalg.norm(out[a:a + 4]) - 1.0) < 1e-14
            assert not np.array_equal(out[a:a + 4], x[a:a + 4])


def _empirical(m, x, P, count, problem=0):
    from mujoco_mpc_b200 import estimator
    n = 2 * m.nv
    D = np.zeros((count, n))
    for i in range(count):
        # members 1..31 of successive iterations: every draw independent
        it, k = divmod(i, 31)
        out = _member(m, x, P, k + 1, seed=5, iteration=it, problem=problem)
        D[i, :m.nv] = estimator.differentiate_pos(m, x[:m.nq], out[:m.nq])
        D[i, m.nv:] = out[m.nq:] - x[m.nq:]
    return D


@pytest.mark.parametrize("kind", ["diagonal", "correlated"])
def test_the_members_have_the_covariance_given(kind):
    m = _model()
    x = _mean(m)
    n = 2 * m.nv
    rng = np.random.default_rng(2)
    P = np.diag(10.0 ** rng.uniform(-4, -2, n)) if kind == "diagonal" else _correlated(n, seed=6)
    count = 4096
    D = _empirical(m, x, P, count)
    S = D.T @ D / count   # the mean of the draws is zero
    sd = np.sqrt(np.diag(P))
    # the standard error of a sample covariance entry is about sqrt((P_ii P_jj + P_ij^2) / count)
    se = np.sqrt((np.outer(np.diag(P), np.diag(P)) + P ** 2) / count)
    assert np.all(np.abs(S - P) < 5 * se), np.max(np.abs(S - P) / se)
    assert np.all(np.abs(D.mean(0)) < 5 * sd / np.sqrt(count))


def test_problems_draw_independently_and_seed_plus_problem_is_the_key():
    m = _model()
    x = _mean(m)
    P = _correlated(2 * m.nv)
    a = _member(m, x, P, 1, seed=10, problem=0)
    b = _member(m, x, P, 1, seed=10, problem=1)
    c = _member(m, x, P, 1, seed=11, problem=0)
    assert not np.array_equal(a, b)
    assert b.tobytes() == c.tobytes()


def test_a_covariance_that_is_not_psd_is_refused():
    from mujoco_mpc_b200.engine import EngineError
    m = _model()
    x = _mean(m)
    n = 2 * m.nv
    P = np.eye(n) * 1e-3
    P[5, 5] = -1e-3
    with pytest.raises(EngineError):
        _member(m, x, P, 1)
    P = np.eye(n) * 1e-3
    P[3, 3] = 0.0
    P[3, 4] = P[4, 3] = 1e-4   # a zero pivot with a coupling below it
    with pytest.raises(EngineError):
        _member(m, x, P, 1)
    P = np.eye(n) * 1e-3
    P[2, 2] = np.nan
    with pytest.raises(EngineError):
        _member(m, x, P, 1)
    P = np.eye(n) * 1e-3
    d = m.nv + 3
    P[d, d] = 0.0   # a direction without uncertainty alone is allowed: that velocity keeps the mean's bits
    out = _member(m, x, P, 1)
    assert out[m.nq + 3] == x[m.nq + 3] and out[m.nq + 4] != x[m.nq + 4]


def test_null_handles_are_refused():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    z = None
    assert lib.mjpc_b200_rollout_spline_belief_batched(None, 1, 2, 1, 0, 0, z, z, z, z, z, z, z, z, z, 0, 1, 1, 1, z, z,
                                                       z) == BAD_ARGUMENT
    assert lib.mjpc_b200_plant_set_sensor_noise(None, 0, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_planner_set_state_ensemble(None, 2, 1, 0) == BAD_ARGUMENT
    assert lib.mjpc_b200_planner_set_state_covariance(None, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_state_ensemble(None, 2, 1, 0) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_state_covariance(None, 0, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_host_state_member(None, z, z, 0, 0, 0, 0, z) == BAD_ARGUMENT


def test_the_loop_passes_the_covariance_only_with_a_state_ensemble():
    from mujoco_mpc_b200.closed_loop import synchronous_planning_cost
    from mujoco_mpc_b200.engine import PLANT_RUNNING

    class Plant:
        num_plants = 1

        def __init__(self, m):
            self.m = m
            self.mocap = np.zeros((1, 7 * m.nmocap), np.float32)

        def get(self, b):
            return dict(state=np.zeros(self.m.nq + self.m.nv, np.float32), time=0.0, status=PLANT_RUNNING)

        def step(self, ctrl):
            m = self.m
            return dict(state=np.zeros((1, m.nq + m.nv), np.float32), time=np.zeros(1), cost=np.zeros(1, np.float32),
                        sensordata=np.zeros((1, 2), np.float32), status=np.zeros(1, np.int32))

    class Estimator:
        def state(self, b):
            return np.zeros(m.nq + m.nv)

        def covariance(self, b):
            return np.eye(2 * m.nv)

        def update(self, *a):
            pass

    class Planner:
        def __init__(self, members):
            self.calls = []
            if members:
                self.state_members = members

        def set_state(self, b, *a):
            self.calls.append("set_state")

        def set_state_covariance(self, b, P):
            self.calls.append("set_state_covariance")

        def action_from_policy(self, b, t):
            return np.zeros(m.nu)

        def optimize_policy(self):
            self.calls.append("optimize_policy")

    m = _model()
    for members, expect in ((0, ["set_state", "optimize_policy"]),
                            (4, ["set_state", "set_state_covariance", "optimize_policy"])):
        p = Planner(members)
        synchronous_planning_cost(p, Plant(m), 1, estimator=Estimator())
        assert p.calls == expect
