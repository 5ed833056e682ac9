"""GPU: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances (fp32 device arithmetic):
  * single forward-dynamics evaluation vs the fp64 oracle: 2e-3 relative on qacc (a contact solve amplifies
    rounding by the condition number of the Newton Hessian), 1e-4 on next state, 1e-4 absolute on residuals;
  * per-candidate returns over the full horizon: 1e-4 relative vs the fp32 oracle is the north-star target; it is
    asserted at 5e-4 because contact make/break within 64 steps is not bit-reproducible between two fp32
    orderings (SURVEY.md section 0 finding 5); the measured maximum is printed and recorded by bench.py.
"""
import numpy as np
import pytest

from conftest import get_model, mocap_of, quadruped_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import Engine
    build.build()
    cache = {}

    def get(name, N=256, H=128, **kw):
        key = (name, N, H, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = Engine(get_model(name, **kw), N, H)
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.fixture(scope="module")
def oracles(oracle_lib):
    from mujoco_mpc_b200.blob import to_blob
    cache = {}

    def get(name, precision=64, **kw):
        key = (name, precision, tuple(sorted(kw.items())))
        if key not in cache:
            m = get_model(name, **kw)
            cache[key] = oracle_lib.Oracle(to_blob(m), m, precision)
        return cache[key]
    return get


def test_particle_rollout_identity(engines, oracles):
    """rollout_test.cc:67-153 through the device path (step-indexed feedback policy = the PD controller)."""
    m = get_model("particle_copy", agent_timestep=False)
    e = engines("particle_copy", 8, 128, agent_timestep=False)
    H = 100
    K = np.zeros((H, 2, 4)); K[:, 0, 0] = K[:, 1, 1] = -10.0; K[:, 0, 2] = K[:, 1, 3] = -2.5
    xn = np.zeros((H, 4)); xn[:, :2] = 0.1
    ret, fail, order = e.rollout_feedback(np.zeros(4), 0.0, mocap_of(m), np.zeros((H, 2)), xn, np.arange(H) * 0.01, K,
                                          np.zeros((H, 2)), [1.0], 3)
    tr = e.fetch_trajectory(0)
    assert fail[0] == 0
    assert np.abs(tr["states"][-1, :2] - 0.1).sum() < 0.1 and np.abs(tr["states"][-1, 2:]).sum() < 0.1
    assert np.abs(tr["states"] - tr["residual"]).sum() < 1e-5
    o = oracles("particle_copy", 64, agent_timestep=False)
    r = o.rollout_feedback(np.zeros(4), 0.0, mocap_of(m), np.zeros((H, 2)), xn, np.arange(H) * 0.01, K, np.zeros((H, 2)), [1.0], 3)
    np.testing.assert_allclose(tr["states"], r["states"][0], atol=2e-6)
    np.testing.assert_allclose(ret[0], r["returns"][0], rtol=1e-5)


@pytest.mark.parametrize("name", ["particle", "cartpole"])
def test_no_contact_rollouts(engines, oracles, name):
    from mujoco_mpc_b200.planner import candidate_knots
    m = get_model(name)
    e, o = engines(name, 64, 64), oracles(name, 64)
    N, H, P = 8, 32, int(m.numeric["sampling_spline_points"][0])
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    state = np.concatenate([m.key_qpos[0] if name == "cartpole" else np.zeros(m.nq), np.zeros(m.nv)])
    kt = np.arange(P) * (H - 1) * m.opt_timestep / (P - 1)
    knots = candidate_knots(np.zeros((P, m.nu)), 0.5, cr, 0, N)
    ret, fail, order = e.rollout_spline(state, 0.0, mocap_of(m), knots, kt, 2, H)
    r = o.rollout_spline(state, 0.0, mocap_of(m), knots, kt, 2, H)
    assert not fail.any() and not r["failure"].any()
    np.testing.assert_allclose(ret, r["returns"], rtol=1e-4)
    tr = e.fetch_all()
    np.testing.assert_allclose(tr["states"], r["states"], atol=2e-4)
    # each step's knot interval and fraction are chosen in double at the reference's rollout time
    # (largest cubic-spline error measured 3e-7 on an H100; a step in the wrong interval moves an action far more)
    np.testing.assert_allclose(tr["actions"], r["actions"], rtol=0, atol=1e-6 * (1 + np.abs(knots).max()))
    np.testing.assert_allclose(tr["residual"], r["residual"], atol=2e-4)
    assert np.array_equal(tr["times"], r["times"])
    assert list(order) == list(np.argsort(r["returns"], kind="stable"))


def test_quadruped_single_step(engines, oracles, quadruped):
    m = quadruped
    e, o = engines("quadruped"), oracles("quadruped", 64)
    rng = np.random.default_rng(0)
    mocap = mocap_of(m)
    for trial in range(6):
        q = m.key_qpos[0].copy()
        q[2] = [0.245, 0.25, 0.26, 0.3, 0.245, 0.24][trial]
        q[7:] += rng.normal(size=12) * 0.05
        v = rng.normal(size=m.nv) * (0.0 if trial == 0 else 0.3)
        u = rng.uniform(-1, 1, m.nu)
        g = e.step_debug(q, v, u, mocap)
        r = o.forward_debug(q, v, u, mocap)
        assert g["ncon"] == r["ncon"] and g["nefc"] == r["nefc"]
        assert np.abs(g["qM"] - r["qM"]).max() < 1e-5
        scale = np.abs(r["qacc"]).max() + 1.0
        assert np.abs(g["qacc"] - r["qacc"]).max() < 2e-3 * scale, (trial, np.abs(g["qacc"] - r["qacc"]).max())
        assert np.abs(g["next_qpos"] - r["next_qpos"]).max() < 1e-4
        assert np.abs(g["next_qvel"] - r["next_qvel"]).max() < 2e-3 * 0.01 * scale + 1e-5
        assert np.abs(g["residual"] - r["residual"][: m.task_num_residual]).max() < 1e-4


def test_quadruped_rollout_returns(engines, oracles, quadruped):
    m = quadruped
    e = engines("quadruped")
    N, H = 32, 64
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    r32 = oracles("quadruped", 32).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=False)
    r64 = oracles("quadruped", 64).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=True)
    assert not fail.any()
    rel32 = np.abs(ret - r32["returns"]) / np.abs(r32["returns"])
    rel64 = np.abs(ret - r64["returns"]) / np.abs(r64["returns"])
    print("max rel return error vs fp32 oracle %.2e, vs fp64 oracle %.2e" % (rel32.max(), rel64.max()))
    # the fp64 oracle is the reference arithmetic (the reference is all-double).  A candidate whose contacts
    # make/break within the horizon bifurcates between the two oracle precisions themselves (4.6e-3 apart on one
    # of these 32); the device must agree with at least one of them, with the fp64 one in the median, and at most
    # 2 of 32 candidates may sit on the fp32 branch.
    assert np.minimum(rel32, rel64).max() < 5e-4 and np.median(rel64) < 5e-5
    assert (rel64 > 5e-4).sum() <= 2
    assert int(order[0]) == int(np.argmin(r64["returns"])) or abs(r64["returns"][order[0]] - r64["returns"].min()) < 5e-4 * r64["returns"].min()
    # short-horizon trajectories (before contact chatter can decorrelate) agree tightly
    tr = e.fetch_all()
    nq = m.nq
    np.testing.assert_allclose(tr["states"][:, :4], r64["states"][:, :4], atol=2e-5)            # free flight: tight
    np.testing.assert_allclose(tr["states"][:, :8, :nq], r64["states"][:, :8, :nq], atol=5e-4)   # first impacts: positions
    np.testing.assert_allclose(tr["states"][:, :8, nq:], r64["states"][:, :8, nq:], atol=2e-2)   # ... velocities (stiff)
    np.testing.assert_allclose(tr["actions"], r64["actions"], atol=2e-5)


def test_full_size_properties(engines, quadruped):
    """BASELINE config 2 sizes (256 x 64): size-independent properties instead of an oracle run."""
    m = quadruped
    e = engines("quadruped")
    N, H = 256, 64
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    knots[17] = knots[0]                                   # duplicate candidate -> identical result
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    tr = e.fetch_all()
    assert not fail.any() and np.isfinite(ret).all()
    assert ret[17] == ret[0] and np.array_equal(tr["states"][17], tr["states"][0])     # determinism across warps
    assert sorted(order.tolist()) == list(range(N)) and (np.diff(ret[order]) >= 0).all()  # sortedness
    np.testing.assert_allclose(ret, tr["costs"].mean(axis=1), rtol=1e-5)               # return = mean cost
    assert np.allclose(tr["actions"][:, -1], tr["actions"][:, -2])                     # last action repeats
    assert (np.abs(tr["actions"]) <= 1.0 + 1e-6).all()                                  # ctrlrange clamp
    np.testing.assert_allclose(np.linalg.norm(tr["states"][:, :, 3:7], axis=-1), 1.0, atol=1e-5)  # unit quaternions
    np.testing.assert_allclose(tr["times"], np.broadcast_to(np.arange(H) * 0.01, (N, H)), atol=1e-5)
    # same call again: bit-identical (no hidden state in the handle)
    ret2, _, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    assert np.array_equal(ret, ret2)
    # time-shift invariance of the task-state rebasing: rollout at t0 = 1000 s with shifted knot times
    ret3, _, _ = e.rollout_spline(state, 1000.0, mocap, knots, kt + 1000.0, 2, H)
    # the gait phase depends on absolute time; with phase_start_time = 0 it differs, so only finiteness is required
    assert np.isfinite(ret3).all()


def test_edge_cases(engines, quadruped):
    from mujoco_mpc_b200.engine import EngineError
    m = quadruped
    e = engines("quadruped")
    state, mocap, knots, kt = quadruped_inputs(m, N=4, H=8)
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots[:1], kt, 2, 1)      # H = 1, N = 1
    assert ret.shape == (1,) and np.isfinite(ret).all()
    for interp in (0, 1, 2):
        ret, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, interp, 8)
        assert np.isfinite(ret).all()
    bad = state.copy(); bad[0] = np.nan
    ret, fail, _ = e.rollout_spline(bad, 0.0, mocap, knots, kt, 2, 8)                 # divergence -> failure, 1e6
    assert fail.all() and (ret == 1.0e6).all()
    with pytest.raises(EngineError):
        e.rollout_spline(state, 0.0, mocap, np.zeros((100000, 3, 12)), kt, 2, 8)      # above capacity
    with pytest.raises(EngineError):
        e.rollout_spline(state, 0.0, mocap, knots, kt, 7, 8)                           # bad interpolation id


def test_cpp_host_planner_matches_python_mirror(engines, quadruped):
    """The C++ SamplingPlanner (csrc/host) and the Python mirror drive the same C ABI with the same injected noise:
    identical winners / installed knots over several planning iterations."""
    from mujoco_mpc_b200.engine import CppSamplingPlanner
    from mujoco_mpc_b200.planner import SamplingPlanner
    m = quadruped
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    mocap = mocap_of(m)
    N, H = 64, 32
    cpp = CppSamplingPlanner(m, N, H)
    py = SamplingPlanner(m, engines("quadruped"), num_trajectory=N, horizon=H)
    cpp.reset(np.zeros(m.nu)); py.reset(np.zeros(m.nu))
    cpp.set_state(state, 0.0, mocap); py.set_state(state, 0.0, mocap)
    for it in range(4):
        rc = cpp.optimize_policy()
        ret, fail = py.optimize_policy()
        np.testing.assert_allclose(rc["knot_times"], py.times, atol=1e-12)
        assert rc["winner"] == py.winner, it
        np.testing.assert_allclose(rc["knots"], py.values, atol=1e-6)
        np.testing.assert_allclose(rc["returns"], ret, rtol=1e-5)
    a = cpp.action_from_policy(0.1)
    np.testing.assert_allclose(a, py.action_from_policy(0.1), atol=1e-6)
    cpp.close()


def test_cpp_cross_entropy_planner_matches_python_mirror(engines, quadruped):
    """Cross-Entropy planner (mjpc/planners/cross_entropy/planner.cc): the C++ host class and the Python mirror
    drive the same rollout ABI with the same injected noise - same elite order, installed mean knots and
    variance over several iterations; the nominal (candidate N) is the returned best trajectory."""
    from mujoco_mpc_b200.engine import CppCrossEntropyPlanner
    from mujoco_mpc_b200.planner import CrossEntropyPlanner
    m = quadruped
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    mocap = mocap_of(m)
    N, H, ne = 48, 32, 6
    cpp = CppCrossEntropyPlanner(m, N, H, n_elite=ne)
    py = CrossEntropyPlanner(m, engines("quadruped"), num_trajectory=N, horizon=H, n_elite=ne)
    cpp.reset(np.zeros(m.nu)); py.reset(np.zeros(m.nu))
    cpp.set_state(state, 0.0, mocap); py.set_state(state, 0.0, mocap)
    for it in range(4):
        rc = cpp.optimize_policy()
        ret, fail = py.optimize_policy()
        assert len(rc["returns"]) == N + 1
        np.testing.assert_allclose(rc["returns"], ret, rtol=1e-5)
        assert list(rc["order"][:ne]) == list(py.order[:ne]), it
        np.testing.assert_allclose(rc["knot_times"], py.times, atol=1e-12)
        np.testing.assert_allclose(rc["knots"], py.values, atol=1e-6)
        np.testing.assert_allclose(rc["variance"], py.variance, rtol=1e-4, atol=1e-10)
        assert abs(rc["improvement"] - py.improvement) < 1e-5
    np.testing.assert_allclose(cpp.action_from_policy(0.1), py.action_from_policy(0.1), atol=1e-6)
    cpp.close()


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_static_and_generic_kernels_agree(name, monkeypatch):
    """The statically specialised rollout kernels (csrc/spec_*.h) and the generic one run the same device
    functions: same returns on the same inputs, and the shipped task models must select their static instance."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model(name)
    if name == "quadruped":
        state, mocap, knots, kt = quadruped_inputs(m, N=32, H=64)
        H = 64
    else:
        rng = np.random.default_rng(1)
        H, P = 48, 16
        state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
        mocap = _track_mocap(m)
        knots = np.clip(0.05 * rng.standard_normal((32, P, m.nu)), -1, 1)
        kt = np.arange(P) * (H - 1) * 0.005 / (P - 1)
    e = Engine(m, 32, H)
    r1, f1, o1 = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    assert e.last_kernel_static, "csrc/spec_%s.h is stale: run python -m mujoco_mpc_b200.build" % name
    monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    r2, f2, o2 = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    assert not e.last_kernel_static
    np.testing.assert_allclose(r1, r2, rtol=2e-4)
    assert (f1 == f2).all()
    e.close()


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_helper_warp_kernel_equals_one_warp_kernel_bitwise(name, monkeypatch):
    """The shipped static rollout instance spreads one candidate over several warps (wide Hessian assembly; fork / join
    of the phases that do not depend on the constraint pipeline - DESIGN.md section 5).  That only moves work between
    warps, so every recorded array must be BITWISE equal to the one-warp-per-candidate instance of the same source
    (MJPC_B200_SHAPE=plain) - for spline rollouts, NoisyRollout, and the iLQG feedback policy (whose action depends on
    the next state and stays on the main warp)."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model(name)
    N = 24
    if name == "quadruped":
        H = 40
        state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    else:
        rng = np.random.default_rng(3)
        H, P = 32, 8
        state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
        mocap = _track_mocap(m)
        knots = np.clip(0.05 * rng.standard_normal((N, P, m.nu)), -1, 1)
        kt = np.arange(P) * (H - 1) * 0.005 / (P - 1)
    e = Engine(m, N, H)

    def both(run):
        out = {}
        for shape, code in (("wide", 1), ("plain", 2)):
            monkeypatch.setenv("MJPC_B200_SHAPE", shape)
            ret, fail, _ = run()
            assert e.last_kernel_shape == code
            out[shape] = dict(e.fetch_all(), returns=ret, failure=fail)
        for k in out["wide"]:
            assert np.array_equal(out["wide"][k], out["plain"][k]), k
        return out["wide"]

    clean = both(lambda: e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H))
    assert not clean["failure"].any()
    e.set_xfrc_noise(1.0, 0.1, 5)
    try:
        noisy = both(lambda: e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H))
    finally:
        e.set_xfrc_noise(0.0)
    assert np.abs(noisy["returns"] - clean["returns"]).max() > 1e-5
    # feedback policy around candidate 0's trajectory (discrete and time-interpolated modes)
    n = 2 * m.nv
    gains = 0.01 * np.random.default_rng(4).standard_normal((H, m.nu, n)).astype(np.float32)
    du = np.zeros((H, m.nu), np.float32)
    steps = np.linspace(0.0, 1.0, 6)
    for mode in (0, 3):
        both(lambda: e.rollout_feedback(state, 0.0, mocap, clean["actions"][0], clean["states"][0], clean["times"][0],
                                        gains, du, steps, mode))
    e.close()


def test_pair_synchronisation_is_timing_only(monkeypatch):
    """When candidates outnumber the SMs, the two candidates resident on an SM keep in step through a flag record in HBM
    (csrc/dev_data.cuh, pair_sync_*): it orders nothing but time, so every recorded array must be bitwise the same with
    it off (MJPC_B200_PAIR_SYNC=0) and on (1, the default: a meeting at every time step)."""
    import torch
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    N, H = nsm + 40, 12
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    e = Engine(m, N, H)
    out = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("MJPC_B200_PAIR_SYNC", mode)
        ret, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
        out[mode] = dict(e.fetch_all(), returns=ret, failure=fail)
    assert not out["0"]["failure"].any()
    for k in out["0"]:
        assert np.array_equal(out["0"][k], out["1"][k]), k
    e.close()


def test_set_task_and_time_rebasing(engines, oracles, quadruped):
    """mjpc_b200_set_task (the per-iteration residual snapshot, agent.cc:316-319) and the host-side time rebasing."""
    from mujoco_mpc_b200 import task as T
    m = quadruped
    e, o = engines("quadruped"), oracles("quadruped", 64)
    N, H = 8, 24
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    base, _, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    # (1) new weights / parameters change the returns exactly as in the oracle
    w = np.asarray(m.task_weight, float).copy(); w[0] = 3.0; w[5] = 0.5
    prm = np.asarray(m.task_parameters, float).copy(); prm[m.task_parameter_names.index("residual_Amplitude")] = 0.1
    e.set_task(weight=w, parameters=prm); o.set_task(weight=w, parameters=prm)
    ret, _, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    ref = o.rollout_spline(state, 0.0, mocap, knots, kt, 2, H, full=False)["returns"]
    assert np.abs(ret - base).max() > 1e-3
    np.testing.assert_allclose(ret, ref, rtol=5e-4)
    # (2) a rollout that starts at t0 = 1000 s with the task clock shifted by the same amount is the same rollout
    ts = np.asarray(m.task_state, float).copy()
    ts[T.QS_MODE_START_TIME] += 1000.0; ts[T.QS_PHASE_START_TIME] += 1000.0
    e.set_task(weight=w, parameters=prm, task_state=ts)
    ret2, _, _ = e.rollout_spline(state, 1000.0, mocap, knots, kt + 1000.0, 2, H)
    np.testing.assert_allclose(ret2, ret, rtol=1e-5)
    tr = e.fetch_trajectory(0)
    np.testing.assert_allclose(tr["times"], 1000.0 + np.arange(H) * 0.01, atol=1e-5)
    # (3) other modes of the quadruped residual (Biped / Walk / Scramble / Flip) agree with the oracle
    for mode in (1, 2, 3, 4):
        ts2 = np.asarray(m.task_state, float).copy()
        ts2[T.QS_MODE] = mode; ts2[T.QS_HEADING] = 1.0; ts2[T.QS_SPEED] = 0.5; ts2[T.QS_ORIENTATION] = 1.0
        e.set_task(task_state=ts2); o.set_task(task_state=ts2)
        r1, f1, _ = e.rollout_spline(state, 0.0, mocap, knots[:4], kt, 2, 12)
        r2 = o.rollout_spline(state, 0.0, mocap, knots[:4], kt, 2, 12, full=False)
        assert not f1.any() and not r2["failure"].any()
        np.testing.assert_allclose(r1, r2["returns"], rtol=1e-3, err_msg="mode %d" % mode)
    e.set_task(weight=np.asarray(m.task_weight, float), parameters=np.asarray(m.task_parameters, float),
               task_state=np.asarray(m.task_state, float))
    o.set_task(weight=np.asarray(m.task_weight, float), parameters=np.asarray(m.task_parameters, float),
               task_state=np.asarray(m.task_state, float))


def test_handles_are_independent(quadruped):
    """Two handles (different models) alive at once; create/destroy does not leak or disturb the other."""
    from mujoco_mpc_b200.engine import Engine
    m = quadruped
    state, mocap, knots, kt = quadruped_inputs(m, N=4, H=8)
    e1 = Engine(m, 8, 16)
    r1, _, _ = e1.rollout_spline(state, 0.0, mocap, knots, kt, 2, 8)
    for _ in range(5):
        e2 = Engine(get_model("cartpole"), 8, 16)
        mc = get_model("cartpole")
        e2.rollout_spline(np.array([1.0, 0, 0, 0]), 0.0, np.zeros(0), np.zeros((4, 10, 1)), np.arange(10) * 0.03, 2, 8)
        e2.close()
    r2, _, _ = e1.rollout_spline(state, 0.0, mocap, knots, kt, 2, 8)
    assert np.array_equal(r1, r2)
    e1.close()


def _humanoid_poses(m):
    """(qpos, qvel, ctrl) cases: standing contact, random airborne, tendon lower limit, deep crouch with contacts."""
    rng = np.random.default_rng(3)
    jn = m.jnt_names
    hip, knee = m.jnt_qposadr[jn.index("hip_y_right")], m.jnt_qposadr[jn.index("knee_right")]
    cases = []
    q = m.qpos0.copy(); cases.append((q, np.zeros(m.nv), np.zeros(m.nu)))
    q = m.qpos0.copy(); q[7:] += 0.3 * rng.standard_normal(m.nq - 7); q[2] = 2.0
    cases.append((q, 0.5 * rng.standard_normal(m.nv), rng.uniform(-1, 1, m.nu)))
    q = m.qpos0.copy(); q[2] = 3.0; q[hip] = -1.0; q[knee] = 0.0
    cases.append((q, 0.2 * rng.standard_normal(m.nv), np.zeros(m.nu)))
    q = m.qpos0.copy(); q[2] -= 0.02; q[7:] += 0.05 * rng.standard_normal(m.nq - 7)
    cases.append((q, 0.3 * rng.standard_normal(m.nv), rng.uniform(-0.3, 0.3, m.nu)))
    return cases


def test_humanoid_single_step(engines, oracles):
    """Humanoid (nv = 27, generic kernel path): pyramidal cones, tendon-limit rows, joint springs, 3 hinges per body."""
    m = get_model("humanoid")
    e, o = engines("humanoid", N=64, H=32), oracles("humanoid", 64)
    for k, (q, v, u) in enumerate(_humanoid_poses(m)):
        g = e.step_debug(q, v, u, np.zeros(0))
        r = o.forward_debug(q, v, u, np.zeros(0))
        assert g["ncon"] == r["ncon"] and g["nefc"] == r["nefc"], (k, g["ncon"], r["ncon"], g["nefc"], r["nefc"])
        assert np.abs(g["qM"] - r["qM"]).max() < 2e-5 * np.abs(r["qM"]).max()
        scale = np.abs(r["qacc"]).max() + 1.0
        assert np.abs(g["qacc"] - r["qacc"]).max() < 2e-3 * scale, (k, np.abs(g["qacc"] - r["qacc"]).max(), scale)
        assert np.abs(g["next_qpos"] - r["next_qpos"]).max() < 1e-4
        assert np.abs(g["residual"] - r["residual"][: m.task_num_residual]).max() < 2e-4


def test_humanoid_rollout_returns(engines, oracles):
    m = get_model("humanoid")
    e = engines("humanoid", N=64, H=32)
    N, H = 32, 24
    rng = np.random.default_rng(5)
    state = np.concatenate([m.qpos0, np.zeros(m.nv)])
    knots = np.clip(0.05 * rng.standard_normal((N, 3, m.nu)), -1, 1); knots[0] = 0
    kt = np.array([0.0, 0.1725, 0.345])
    ret, fail, order = e.rollout_spline(state, 0.0, np.zeros(0), knots, kt, 2, H)
    r64 = oracles("humanoid", 64).rollout_spline(state, 0.0, np.zeros(0), knots, kt, 2, H, nthreads=8, full=True)
    r32 = oracles("humanoid", 32).rollout_spline(state, 0.0, np.zeros(0), knots, kt, 2, H, nthreads=8, full=False)
    assert not fail.any() and not r64["failure"].any()
    rel64 = np.abs(ret - r64["returns"]) / np.abs(r64["returns"])
    rel32 = np.abs(ret - r32["returns"]) / np.abs(r32["returns"])
    print("humanoid: max rel return error vs fp32 oracle %.2e, vs fp64 oracle %.2e" % (rel32.max(), rel64.max()))
    assert np.minimum(rel32, rel64).max() < 5e-4 and np.median(rel64) < 5e-5
    tr = e.fetch_all()
    np.testing.assert_allclose(tr["states"][:N, :6, : m.nq], r64["states"][:, :6, : m.nq], atol=5e-4)
    np.testing.assert_allclose(tr["actions"][:N, :H], r64["actions"], atol=2e-5)


def _track_mocap(m):
    return np.concatenate([m.key_mpos[0].reshape(-1, 3), np.tile([1.0, 0, 0, 0], (m.nmocap, 1))], 1).reshape(-1)


def test_humanoid_track_single_step(engines, oracles):
    """BASELINE config 3 task: 141-dim tracking residual reading the keyframe table from HBM, at several clip
    times / clips (task_state = [mode, reference_time], the clock is rebased on the device)."""
    from mujoco_mpc_b200 import task as T
    m = get_model("humanoid_track")
    e, o = engines("humanoid_track", N=64, H=128), oracles("humanoid_track", 64)
    mocap = _track_mocap(m)
    rng = np.random.default_rng(7)
    for mode, t in ((0, 0.0), (0, 1.2345), (4, 2.01), (9, 100.0), (2, 1003.7)):
        ts = np.array([float(mode), 1000.0 if t > 1000 else 0.25])
        e.set_task(task_state=ts); o.set_task(task_state=ts)
        q = m.key_qpos[sum(T.TRACK_MOTION_LENGTHS[:mode]) + 7].copy()
        q[7:] += 0.03 * rng.standard_normal(m.nq - 7)
        v = 0.3 * rng.standard_normal(m.nv); u = rng.uniform(-0.5, 0.5, m.nu)
        g = e.step_debug(q, v, u, mocap, time=t)
        r = o.forward_debug(q, v, u, mocap, time=t)
        assert g["ncon"] == r["ncon"] and g["nefc"] == r["nefc"]
        scale = np.abs(r["qacc"]).max() + 1.0
        assert np.abs(g["qacc"] - r["qacc"]).max() < 2e-3 * scale
        # marker velocities scale with |qvel| * lever arms; positions with metres: 2e-4 absolute covers both in fp32
        assert np.abs(g["residual"] - r["residual"][:141]).max() < 3e-4, (mode, t, np.abs(g["residual"] - r["residual"][:141]).max())
    ts = np.asarray(m.task_state, float)
    e.set_task(task_state=ts); o.set_task(task_state=ts)


def test_humanoid_track_rollout_returns(engines, oracles):
    """Config-3 shaped rollouts (16 cubic knots, dt 0.005) at a size the oracle finishes in seconds."""
    m = get_model("humanoid_track")
    e = engines("humanoid_track", N=64, H=128)
    N, H, P = 24, 101, 16
    rng = np.random.default_rng(11)
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    knots = np.clip(0.15 * 0.3 * rng.standard_normal((N, P, m.nu)), -1, 1); knots[0] = 0
    kt = np.arange(P) * (H - 1) * 0.005 / (P - 1)
    mocap = _track_mocap(m)
    ret, fail, order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    r64 = oracles("humanoid_track", 64).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=True)
    r32 = oracles("humanoid_track", 32).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=False)
    assert not fail.any() and not r64["failure"].any()
    rel64 = np.abs(ret - r64["returns"]) / np.abs(r64["returns"])
    rel32 = np.abs(ret - r32["returns"]) / np.abs(r32["returns"])
    print("humanoid track: max rel return error vs fp32 oracle %.2e, vs fp64 oracle %.2e" % (rel32.max(), rel64.max()))
    assert np.minimum(rel32, rel64).max() < 1e-3 and np.median(rel64) < 1e-4
    tr = e.fetch_all()
    np.testing.assert_allclose(tr["residual"][:N, 0], r64["residual"][:, 0], atol=3e-4)
    np.testing.assert_allclose(tr["actions"][:N, :H], r64["actions"], atol=2e-5)


def test_noisy_rollout_matches_oracle(engines, oracles, quadruped):
    """NoisyRollout (trajectory.cc:100-210): in-kernel Ornstein-Uhlenbeck xfrc noise from the injected Philox stream
    (fp32 Box-Muller on the device, fp64 in the oracle) -> same perturbed trajectories as the oracle."""
    m = quadruped
    e, o = engines("quadruped"), oracles("quadruped", 64)
    N, H = 16, 32
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    clean, _, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    e.set_xfrc_noise(2.0, 0.1, 77); o.set_xfrc_noise(2.0, 0.1, 77)
    try:
        ret, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
        tr = e.fetch_all()
        ref = o.rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=True)
    finally:
        e.set_xfrc_noise(0.0); o.set_xfrc_noise(0.0)
    assert not fail.any()
    assert np.abs(ret - clean).max() > 1e-4                       # the perturbation is visible in the returns
    np.testing.assert_allclose(tr["states"][:N, :6], ref["states"][:, :6], atol=2e-4)   # first steps: free flight + noise
    rel = np.abs(ret - ref["returns"]) / np.abs(ref["returns"])
    print("noisy rollouts: max rel return error vs fp64 oracle %.2e" % rel.max())
    assert rel.max() < 2e-3 and np.median(rel) < 2e-4
    again, _, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    np.testing.assert_allclose(again, clean, rtol=1e-6)           # switched off again


def test_noisy_rollout_equals_equivalent_controls_on_device(engines):
    """Same construction as tests/test_planners_cpu.py: on the particle a Cartesian force is exactly a control."""
    from mujoco_mpc_b200.planner import philox4x32
    m = get_model("particle")
    e = engines("particle", N=8, H=16)
    H, std, rate_s, seed = 12, 0.05, 0.2, 1234
    body = int(m.jnt_bodyid[0])
    state = np.array([0.05, -0.02, 0.1, 0.0])
    kt = np.arange(H) * m.opt_timestep - 1e-6
    e.set_xfrc_noise(std, rate_s, seed)
    try:
        e.rollout_spline(state, 0.0, mocap_of(m), np.zeros((2, H, m.nu)), kt, 0, H)
        noisy = e.fetch_trajectory(1)
    finally:
        e.set_xfrc_noise(0.0)
    rate = np.exp(-m.opt_timestep / rate_s); scale = std * np.sqrt(1 - rate * rate)
    x = np.zeros(6 * m.nbody); forces = np.zeros((H, 2))
    for t in range(H - 1):
        ctr = np.array([[t, 1, el, 0x58465243] for el in range(6 * m.nbody)], np.uint32)
        r = philox4x32(ctr, (seed, 1))
        u1 = (r[:, 0].astype(np.float64) + 0.5) / 4294967296.0; u2 = (r[:, 1].astype(np.float64) + 0.5) / 4294967296.0
        x = rate * x + scale * np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2)
        forces[t] = x[6 * body: 6 * body + 2]
    e.rollout_spline(state, 0.0, mocap_of(m), forces[None], kt, 0, H)
    clean = e.fetch_trajectory(0)
    np.testing.assert_allclose(noisy["states"], clean["states"], atol=2e-6)


def test_cpp_robust_planner_matches_python_mirror(engines, quadruped):
    """Robust planner (robust_planner.cc:91-157): C++ host class vs the Python mirror on the same engine ABI."""
    from mujoco_mpc_b200.engine import CppRobustPlanner
    from mujoco_mpc_b200.planner import RobustPlanner
    m = quadruped
    state = np.concatenate([m.key_qpos[0], np.zeros(m.nv)])
    mocap = mocap_of(m)
    N, H = 40, 32
    cpp = CppRobustPlanner(m, N, H, ncandidates=5, nrepetitions=4, xfrc_std=1.0, xfrc_rate=0.1)
    py = RobustPlanner(m, engines("quadruped"), num_trajectory=N, horizon=H, ncandidates=5, nrepetitions=4,
                       xfrc_std=1.0, xfrc_rate=0.1)
    cpp.reset(np.zeros(m.nu)); py.reset(np.zeros(m.nu))
    cpp.set_state(state, 0.0, mocap); py.set_state(state, 0.0, mocap)
    for it in range(3):
        rc = cpp.optimize_policy()
        ret, fail = py.optimize_policy()
        np.testing.assert_allclose(rc["returns"], ret, rtol=1e-5)
        np.testing.assert_allclose(rc["scores"], py.scores, rtol=1e-5)
        assert rc["winner"] == py.winner, it
        np.testing.assert_allclose(rc["knots"], py.delegate.values, atol=1e-6)
    cpp.close()
