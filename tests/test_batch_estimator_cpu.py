"""CPU: the batched estimator's entry points refuse a NULL handle with MJPC_B200_ERR_BAD_ARGUMENT instead of
dereferencing it, and its create refuses, before it asks for a device, a bad argument, a bad blob, a sensor range
outside the model's sensors and more step rows than one handle holds (no device needed)."""
import ctypes

BAD_ARGUMENT, BAD_BLOB, CAPACITY = -1, -2, -3   # MJPC_B200_ERR_*


def test_batch_estimator_entry_points_refuse_null_handle():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    v = (ctypes.c_double * 8)()
    status = (ctypes.c_int * 8)()
    calls = {"destroy": (), "reset": (0, None, ctypes.c_double(0.0), ctypes.c_double(1e-4), ctypes.c_double(1e-4),
                                      ctypes.c_double(1e-4)),
             "set_noise": (0, None, None), "set": (0, None, None, ctypes.c_double(0.0)), "update": (v, v, None, status),
             "get": (0, None, None, None, None)}
    for name, args in calls.items():
        assert getattr(lib, f"mjpc_b200_batch_estimator_{name}")(None, *args) == BAD_ARGUMENT, name
    lib.mjpc_b200_batch_estimator_last_error.restype = ctypes.c_char_p
    assert lib.mjpc_b200_batch_estimator_last_error(None) == b""


def test_batch_estimator_create_refusals_before_the_device():
    from mujoco_mpc_b200 import models
    from mujoco_mpc_b200.engine import ModelBlob, _model_blob, load_library
    lib = load_library()
    create = lib.mjpc_b200_batch_estimator_create
    m = models.load("quadruped")
    _, mb = _model_blob(m)
    h = ctypes.c_void_p()
    dt = ctypes.c_double(0.005)
    for kind, prm in ((1, (1e-3, 1.0)), (2, (1.0, 2.0))):
        s = (ctypes.c_double * 2)(*prm)
        assert create(ctypes.byref(mb), kind, 2, 9, m.nsensor, dt, s, 0, ctypes.byref(h)) == BAD_ARGUMENT
        assert create(ctypes.byref(mb), kind, 2, -1, 2, dt, s, 0, ctypes.byref(h)) == BAD_ARGUMENT
        assert create(ctypes.byref(mb), kind, 0, 9, 21, dt, s, 0, ctypes.byref(h)) == BAD_ARGUMENT
        assert create(ctypes.byref(mb), kind, 2, 9, 21, ctypes.c_double(0.0), s, 0, ctypes.byref(h)) == BAD_ARGUMENT
        # 73 step rows per Quadruped filter (Unscented 2 ndstate + 1, centred Kalman the same): 898 filters exceed 65536
        assert create(ctypes.byref(mb), kind, 65536 // 73 + 1, 9, 21, dt, s, 0, ctypes.byref(h)) == CAPACITY
        assert not h.value
        junk = ctypes.create_string_buffer(b"not a model blob", 16)
        bad = ModelBlob(ctypes.cast(junk, ctypes.c_void_p), 16)
        assert create(ctypes.byref(bad), kind, 2, 9, 21, dt, s, 0, ctypes.byref(h)) == BAD_BLOB
        assert not h.value
    s = (ctypes.c_double * 2)(1.0, 2.0)
    assert create(ctypes.byref(mb), 3, 2, 9, 21, dt, s, 0, ctypes.byref(h)) == BAD_ARGUMENT        # unknown kind
    assert create(ctypes.byref(mb), 1, 2, 9, 21, dt, (ctypes.c_double * 2)(0.0, 1.0), 0, ctypes.byref(h)) == BAD_ARGUMENT
    assert create(ctypes.byref(mb), 2, 2, 9, 21, dt, None, 0, ctypes.byref(h)) == BAD_ARGUMENT
