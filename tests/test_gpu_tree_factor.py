"""GPU: the static rollout kernels' leaves-first factorisation along the dof tree (csrc/dev_data.cuh
warp_tree_factor_solve) against fp64, on the Quadruped:
  * airborne and floor rollouts: every state against the fp64 oracle, as close as the generic kernel's dense factor;
  * rollouts from a floor state (one-sided contacts: the Hessian keeps qM's tree pattern) and from a state whose legs
    touch each other (contacts between two moving bodies: the dense fallback), static kernel against the generic one
    and against the oracles."""
import numpy as np
import pytest

from conftest import get_model, quadruped_inputs

pytestmark = pytest.mark.gpu


def _oracle(oracle_lib, m, precision=64):
    from mujoco_mpc_b200.blob import to_blob
    return oracle_lib.Oracle(to_blob(m), m, precision)


def _self_contact_states(m, rng, B):
    q = np.tile(np.asarray(m.key_qpos[0], float), (B, 1))
    q[:, 2] = 3.0                                                      # far above the floor
    lo = np.array([m.jnt_range[j][0] for j in range(1, m.njnt)]); hi = np.array([m.jnt_range[j][1] for j in range(1, m.njnt)])
    q[:, 7:] = lo + (hi - lo) * rng.uniform(0.0, 1.0, (B, m.nq - 7))   # anywhere inside the joint ranges
    v = np.zeros((B, m.nv)); v[:, 6:] = 0.5 * rng.standard_normal((B, m.nv - 6))
    return q, v


@pytest.mark.parametrize("start", ["airborne", "floor"])
def test_rollout_states_match_fp64(oracle_lib, monkeypatch, start):
    """Every state of 32 candidates over 24 steps against the fp64 oracle, static kernel (tree factor) and generic
    kernel (dense factor): airborne, the solves are qM, the Euler matrix and a Hessian with only friction-loss
    diagonals; on the floor, the Hessian adds one-sided contacts."""
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 32, 24
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    if start == "airborne":
        state = state.copy(); state[2] = 3.0
    ref = _oracle(oracle_lib, m).rollout_spline(state, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=True)["states"]
    scale = np.abs(ref).reshape(N, -1).max(1) + 1.0
    e = Engine(m, N, H)
    try:
        err = {}
        for kind in ("static", "generic"):
            if kind == "generic":
                monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
            e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
            assert e.last_kernel_static == (kind == "static")
            st = e.fetch_all()["states"]
            err[kind] = np.abs(st[:, :8] - ref[:, :8]).reshape(N, -1).max(1) / scale
        monkeypatch.delenv("MJPC_B200_NO_STATIC")
    finally:
        e.close()
    print("%s: first 8 states, err / scale vs fp64: tree median %.2e max %.2e, dense median %.2e max %.2e"
          % (start, np.median(err["static"]), err["static"].max(), np.median(err["generic"]), err["generic"].max()))
    assert err["static"].max() < 5e-3 and np.median(err["static"]) <= 2 * np.median(err["generic"]) + 1e-6
    if start == "airborne":   # no contact to make or break: the two factors' errors are both rounding
        assert err["static"].max() <= 4 * err["generic"].max() + 1e-6


def test_rollouts_with_and_without_the_dense_fallback(oracle_lib, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 32, 24
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    # a self-contact start: the first state of a seeded sweep whose legs touch each other in the air
    rng = np.random.default_rng(3)
    qs, vs = _self_contact_states(m, rng, 256)
    ref = _oracle(oracle_lib, m).step_batch(qs, vs, np.zeros((len(qs), m.nu)), mocap, np.zeros(len(qs)), nthreads=8)
    k = int(np.flatnonzero((ref["ncon"] >= 2) & (ref["warning"] == 0))[0])
    starts = {"floor": state, "self-contact": np.concatenate([qs[k], vs[k]])}
    e = Engine(m, N, H)
    try:
        for name, s in starts.items():
            r_static, f_static, _ = e.rollout_spline(s, 0.0, mocap, knots, kt, 2, H)
            assert e.last_kernel_static
            monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
            r_generic, f_generic, _ = e.rollout_spline(s, 0.0, mocap, knots, kt, 2, H)
            assert not e.last_kernel_static
            monkeypatch.delenv("MJPC_B200_NO_STATIC")
            r32 = _oracle(oracle_lib, m, 32).rollout_spline(s, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=False)["returns"]
            r64 = _oracle(oracle_lib, m, 64).rollout_spline(s, 0.0, mocap, knots, kt, 2, H, nthreads=8, full=False)["returns"]
            rel_g = np.abs(r_static - r_generic) / np.abs(r_generic)
            rel = np.minimum(np.abs(r_static - r32) / np.abs(r32), np.abs(r_static - r64) / np.abs(r64))
            print("%s start: static vs generic max rel %.2e; vs the nearer oracle max %.2e median %.2e"
                  % (name, rel_g.max(), rel.max(), np.median(rel)))
            assert not f_static.any() and (f_static == f_generic).all()
            np.testing.assert_allclose(r_static, r_generic, rtol=2e-4)
            assert np.median(rel) < 5e-5 and (rel > 5e-4).sum() <= 2
    finally:
        e.close()
