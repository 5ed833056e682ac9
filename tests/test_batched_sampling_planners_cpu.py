"""CPU: the entry points of the batched Predictive Sampling, Cross-Entropy, Robust and Sample Gradient planners, of the
generic batch family and of per-problem noise keys, without a device: creates fail with MJPC_B200_ERR_CUDA and leave
*out NULL, and NULL handles are refused."""
import ctypes as C

import numpy as np
import pytest

BAD_ARGUMENT, CUDA = -1, -4


def _no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")


def _create_args(crp, sp):
    """Each kind's batch create arguments between the model and out, with ctrlrange crp and seeds sp."""
    d = C.c_double
    return {
        "sampling": (2, 8, 3, 2, d(0.1), d(0.01), crp, sp, 11, 0),
        "ce": (2, 8, 0, 3, 2, d(0.1), d(0.01), d(0.0), d(0.01), crp, sp, 11, 0),
        "sg": (2, 8, 2, 3, 2, d(0.1), d(0.5), d(0.01), crp, sp, 11, 0),
        "robust": (2, 10, 3, 2, d(0.1), d(0.01), crp, sp, -1, 5, d(0.1), d(0.1), 11, 0),
    }


def test_creates_without_a_device_fail_and_leave_out_null():
    _no_device()
    from conftest import get_model
    from mujoco_mpc_b200.engine import _model_blob, load_library
    lib = load_library()
    m = get_model("particle")
    buf, mb = _model_blob(m)
    cr = np.ascontiguousarray(np.asarray(m.actuator_ctrlrange, float).reshape(-1))
    crp = cr.ctypes.data_as(C.POINTER(C.c_double))
    seeds = np.array([1, 2], np.uint32)
    sp = seeds.ctypes.data_as(C.POINTER(C.c_uint32))
    for kind, args in _create_args(crp, sp).items():
        out = C.c_void_p(12345)
        rc = getattr(lib, f"mjpc_b200_batch_{kind}_planner_create")(C.byref(mb), *args, C.byref(out))
        assert rc == CUDA, (kind, rc)
        assert out.value is None, kind
    del buf


def test_null_batch_family_handles_are_refused_at_header_arity():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    seeds = (C.c_uint32 * 2)(1, 2)
    assert lib.mjpc_b200_set_xfrc_noise_batched(None, C.c_double(0.1), C.c_double(0.1), 2, seeds) == BAD_ARGUMENT
    assert lib.mjpc_b200_planner_set_task(None, None) == BAD_ARGUMENT
    for kind, args in _create_args(None, None).items():
        assert getattr(lib, f"mjpc_b200_batch_{kind}_planner_get_result")(None, 0, *([None] * 9)) == BAD_ARGUMENT, kind
        assert getattr(lib, f"mjpc_b200_batch_{kind}_planner_create")(None, *args, None) == BAD_ARGUMENT, kind
    v = (C.c_double * 8)()
    generic = {"reset": (0, 8, None), "set_state": (0, v, C.c_double(0.0), None), "set_task": (0, None, None, None),
               "optimize_policy": (8, None), "action_from_policy": (0, v, None, C.c_double(0.0), 0)}
    for name, args in generic.items():
        assert getattr(lib, f"mjpc_b200_batch_planner_{name}")(None, *args) == BAD_ARGUMENT, name
