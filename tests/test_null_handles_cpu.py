"""CPU: the planner and estimator entry points refuse a NULL handle with MJPC_B200_ERR_BAD_ARGUMENT instead of
dereferencing it (no device needed)."""
import ctypes

BAD_ARGUMENT = -1   # MJPC_B200_ERR_BAD_ARGUMENT


def test_planner_entry_points_refuse_null_handle():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    v = (ctypes.c_double * 8)()
    generic = {"destroy": (), "reset": (8, None), "set_state": (v, 0.0, None), "optimize_policy": (8,),
               "nominal_trajectory": (8,), "action_from_policy": (v, None, 0.0, 0), "set_fd": (1e-3, 1, 0)}
    for name, args in generic.items():
        assert getattr(lib, f"mjpc_b200_planner_{name}")(None, *args) == BAD_ARGUMENT, name
    # the kind-specific calls on a handle refuse it too
    assert lib.mjpc_b200_sampling_planner_set_exploration(None, 0.1, 0.0) == BAD_ARGUMENT
    assert lib.mjpc_b200_ilqs_planner_set_exploration(None, ctypes.c_double(0.1)) == BAD_ARGUMENT
    for kind in ("sampling", "ce", "sg", "robust", "ilqg", "gradient", "ilqs"):
        assert getattr(lib, f"mjpc_b200_{kind}_planner_get_result")(None, *([None] * 9)) == BAD_ARGUMENT, kind


def test_estimator_entry_points_refuse_null_handle():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    v = (ctypes.c_double * 8)()
    generic = {"destroy": (), "reset": (None, 0.0, 1e-4, 1e-4, 1e-4), "set_noise": (None, None),
               "set": (None, None, 0.0), "update": (v, v, None), "get": (None, None, None, None)}
    for name, args in generic.items():
        assert getattr(lib, f"mjpc_b200_estimator_{name}")(None, *args) == BAD_ARGUMENT, name
    assert lib.mjpc_b200_estimator_last_error(None) == b""
    assert lib.mjpc_b200_kalman_update_measurement(None, v, v, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_kalman_update_prediction(None) == BAD_ARGUMENT
