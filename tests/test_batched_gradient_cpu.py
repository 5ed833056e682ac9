"""CPU: the entry points of the batched Gradient and iLQS planners and of the device gradient sweep, without a device:
the creates fail with MJPC_B200_ERR_CUDA and leave *out NULL, NULL handles are refused, and the host reference of the
sweep (mjpc_b200_host_gradient_sweep) equals the fp64 Python mirror."""
import ctypes as C

import numpy as np
import pytest

BAD_ARGUMENT, CUDA = -1, -4


def test_create_without_a_device_fails_and_leaves_out_null():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from conftest import get_model
    from mujoco_mpc_b200.engine import _model_blob, load_library
    lib = load_library()
    m = get_model("particle")
    buf, mb = _model_blob(m)
    cr = np.ascontiguousarray(np.asarray(m.actuator_ctrlrange, float).reshape(-1))
    out = C.c_void_p(12345)
    rc = lib.mjpc_b200_batch_gradient_planner_create(C.byref(mb), 2, 8, 5, 1, C.c_double(1e-3), C.c_double(0.01),
                                                     cr.ctypes.data_as(C.POINTER(C.c_double)), 16, 0, C.byref(out))
    assert rc == CUDA
    assert out.value is None
    seeds = np.array([1, 2], np.uint32)
    out = C.c_void_p(12345)
    rc = lib.mjpc_b200_batch_ilqs_planner_create(C.byref(mb), 2, 8, 3, 2, C.c_double(0.1), C.c_double(0.01),
                                                 cr.ctypes.data_as(C.POINTER(C.c_double)),
                                                 seeds.ctypes.data_as(C.POINTER(C.c_uint32)), 6, 1, C.c_double(1e-3), 16,
                                                 0, C.byref(out))
    assert rc == CUDA
    assert out.value is None
    del buf


def test_null_batch_handles_are_refused():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    d = C.c_double
    assert lib.mjpc_b200_batch_gradient_planner_create(None, 2, 8, 5, 1, d(1e-3), d(0.01), None, 16, 0, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_gradient_planner_get_result(None, 0, None, None, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_fd(None, d(1e-3), 0, 0) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ilqs_planner_create(None, 2, 8, 3, 2, d(0.1), d(0.01), None, None, 6, 1, d(1e-3), 16, 0,
                                                   None) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ilqs_planner_get_result(None, 0, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_ilqs_planner_set_exploration(None, d(0.1)) == BAD_ARGUMENT
    a = (C.c_double * 8)()
    assert lib.mjpc_b200_batch_planner_action_from_policy(None, 0, a, a, d(0.0), 0) == BAD_ARGUMENT
    v = (C.c_double * 8)()
    f = (C.c_float * 8)()
    assert lib.mjpc_b200_gradient_batched(None, 1, f, f, v, None, None, None, None, f, 2, 0, C.c_float(1e-3), 0, v,
                                          v) == BAD_ARGUMENT


def _chain(rng, T, n, m):
    A = (0.9 * np.eye(n) + 0.1 * rng.standard_normal((T, n, n)) / np.sqrt(n)).astype(np.float32)   # a transition
    B = rng.standard_normal((T, n, m)).astype(np.float32)
    cx = rng.standard_normal((T, n)).astype(np.float32)
    cu = rng.standard_normal((T, m)).astype(np.float32)
    return A, B, cx, cu


@pytest.mark.parametrize("T,n,m", [(2, 4, 1), (2, 36, 12), (3, 7, 3), (32, 36, 12), (64, 54, 21)])
def test_host_gradient_sweep_equals_python_mirror(T, n, m):
    from mujoco_mpc_b200.engine import host_gradient_sweep
    from mujoco_mpc_b200.gradient import gradient_sweep
    rng = np.random.default_rng(T * 1000 + n)
    A, B, cx, cu = _chain(rng, T, n, m)
    k, dV0 = host_gradient_sweep(A, B, cx, cu)
    k_ref, dV0_ref = gradient_sweep(A, B, cx, cu)
    scale = np.abs(k_ref).max()
    np.testing.assert_allclose(k, k_ref, rtol=0, atol=1e-12 * scale)
    assert abs(dV0 - dV0_ref) <= 1e-12 * abs(dV0_ref)
    np.testing.assert_array_equal(k[T - 1], k[T - 2])           # the last row repeats the one before
    assert dV0 < 0
