"""GPU: a handle whose buffers grew computes what a fresh handle computes.

The engine sizes some buffers at create and grows them on demand, never shrinking them: the feedback policies, the iLQG
sweep buffers, the per-trajectory buffers of a model ensemble, the state-ensemble tables, the step scratch and the plant
bank.  Each test drives one handle from small to large to small and requires every output to be BITWISE equal to that of
a fresh handle for the same call.

The state estimators' filter bank is not covered: replacing a handle's bank (mjpc_b200_bank::Init on a handle that has
one) cannot be reached through the public API, since every estimator creates its own handle and initialises its bank
once."""
import numpy as np
import pytest

from conftest import get_model, mocap_of
from test_gpu_batched import _problems as _spline_problems
from test_gpu_batched_ilqg import _feedback_inputs, _lq, _problems, _task
from test_gpu_model_variants import _assert_equal, _spline, _variants
from test_gpu_state_ensemble import _belief, _covs

pytestmark = pytest.mark.gpu


def _sub(pr, B):
    return {k: v[:B] for k, v in pr.items()}


def _fresh(m, N, H, call):
    from mujoco_mpc_b200.engine import Engine
    e = Engine(m, N, H)
    try:
        return call(e)
    finally:
        e.close()


def test_feedback_rollouts_after_growth():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    H, K = 16, 6
    pr = _problems(m, H)
    gains, du, steps = _feedback_inputs(m, pr, K, True)

    def run(e, B):
        p = _sub(pr, B)
        ret, fail, order = e.rollout_feedback_batched(p["states"], p["times"], p["mocaps"], p["u"], p["x"], p["t"],
                                                      gains[:B], du[:B], steps[:B], 1, **_task(p))
        return dict(e.fetch_all(), returns=ret, failure=fail, order=order)

    e = Engine(m, 3 * K, H)
    for B in (1, 3, 2):
        _assert_equal(run(e, B), _fresh(m, 3 * K, H, lambda f: run(f, B)), f"feedback rollouts, B = {B}")
    e.close()


def test_ilqg_sweeps_after_growth():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    H = 16
    pr = _problems(m, H)
    mu = np.array([1e-3, 0.5, 1.0, 4.0], np.float32)

    def run(e, B):
        lq = _lq(e, _sub(pr, B))
        bp = e.backward_pass_batched(**lq, mu=mu[:B])
        return dict(lq, **{f"bp_{k}": v for k, v in bp.items()})

    e = Engine(m, 8, H)
    for B in (1, 4):
        _assert_equal(run(e, B), _fresh(m, 8, H, lambda f: run(f, B)), f"iLQG sweeps, B = {B}")
    e.close()


def test_model_ensemble_and_state_ensemble_after_growth():
    from mujoco_mpc_b200.engine import Engine
    base, V = get_model("quadruped"), _variants("quadruped")
    B, N, H = 2, 4, 12
    pr = _spline_problems(base, N, H, B=B)

    def launch(e, K):
        if K:
            e.set_model_ensemble(V[:K], worst=K)
        out = _spline(e, pr, H)
        if K:
            out["member_returns"], out["member_failure"] = e.fetch_ensemble()
        return out

    e = Engine(base, B * N, H)
    for K in (2, 4, 0):
        if not K:
            e.set_model_ensemble(None)
        _assert_equal(launch(e, K), _fresh(base, B * N, H, lambda f: launch(f, K)), f"model ensemble, K = {K}")
    covs = _covs(base, B)

    def belief(e):
        out = _belief(e, pr, covs, H, 3, 2)
        out["member_returns"], out["member_failure"] = e.fetch_ensemble()
        return out

    _assert_equal(belief(e), _fresh(base, B * N, H, belief), "state ensemble")
    e.close()


def test_step_sensors_after_growth():
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    k = m.key_names.index("home")
    rng = np.random.default_rng(2)
    X = np.tile(np.concatenate([m.key_qpos[k], np.zeros(m.nv)]), (6, 1))
    X[:, m.nq:] += 0.1 * rng.standard_normal((6, m.nv))
    u = 0.2 * rng.standard_normal(m.nu)
    mc = mocap_of(m)

    def run(e, B):
        return e.step_sensors(X[:B], u, mc, 0.05, 26, 4)

    e = Engine(m, 8, 1)
    for B in (1, 3, 6, 2):
        _assert_equal(run(e, B), _fresh(m, 8, 1, lambda f: run(f, B)), f"step_sensors, B = {B}")
    e.close()


def test_plant_bank_after_reinit():
    from mujoco_mpc_b200.engine import CppPlantBank
    m = get_model("quadruped")
    k = m.key_names.index("home")
    q, v = np.asarray(m.key_qpos[k], np.float32), np.zeros(m.nv, np.float32)
    rng = np.random.default_rng(4)
    U = 0.3 * rng.standard_normal((5, 3, m.nu))

    def episode(bank):
        for b in range(bank.num_plants):
            bank.reset(b, q, v + 0.05 * b, 0.1 * b)
        outs = [bank.step(U[i, :bank.num_plants]) for i in range(len(U))]
        return {f"{i} {key}": val for i, o in enumerate(outs) for key, val in o.items()}

    def fresh(n):
        f = CppPlantBank(m, n, sensor_start=26, nsensor=4)
        try:
            return episode(f)
        finally:
            f.close()

    bank = CppPlantBank(m, 3, sensor_start=26, nsensor=4)
    _assert_equal(episode(bank), fresh(3), "plants, B = 3")
    for n in (2, 3):
        assert bank.lib.mjpc_b200_plant_init(bank.h, n, 26, 4) == 0, bank.lib.mjpc_b200_last_error().decode()
        bank.num_plants = n
        _assert_equal(episode(bank), fresh(n), f"plants re-initialised, B = {n}")
    bank.close()
