"""The helper-warp rollout assembles each Newton Hessian on its helper warps while the main warp forms the gradient and
the termination test (csrc/dev_physics.cuh, k_solve).  When the test stops the solve, the assembly in flight is met and
dropped.  With a loose solver tolerance most solves stop at the first test, right after the first Hessian was posted;
every recorded array must still be bitwise that of the one-warp kernel (MJPC_B200_SHAPE=plain)."""
import numpy as np
import pytest

from conftest import get_model, quadruped_inputs


@pytest.mark.gpu
@pytest.mark.parametrize("tolerance", [1e-2, 1.0])
def test_solve_stopping_with_a_hessian_in_flight_is_bitwise(tolerance, monkeypatch):
    from mujoco_mpc_b200.engine import Engine
    base = get_model("quadruped")
    m = type(base)(base)                 # a shallow copy: only the option below differs
    m.opt_tolerance = tolerance          # a float option: the static kernels stay selected
    N, H = 24, 24
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    newton = {}
    for name, model in (("default", base), ("loose", m)):
        e = Engine(model, N, H)
        out = {}
        for shape, code in (("wide", 1), ("plain", 2)):
            monkeypatch.setenv("MJPC_B200_SHAPE", shape)
            ret, fail, _ = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
            assert e.last_kernel_shape == code
            out[shape] = dict(e.fetch_all(), returns=ret, failure=fail)
            if shape == "wide":
                newton[name] = e.fetch_stats()[:, 1].sum()
        e.close()
        assert not out["wide"]["failure"].any()
        for k in out["wide"]:
            assert np.array_equal(out["wide"][k], out["plain"][k]), (name, k)
    assert newton["loose"] < newton["default"]   # the loose tolerance did stop solves earlier
