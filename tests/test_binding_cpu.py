"""CPU: the ctypes prototypes the binding parses from include/mjpc_b200.h (no device)."""
import ctypes as C
import re

import numpy as np
import pytest


@pytest.fixture(scope="module")
def header():
    from mujoco_mpc_b200.engine import HEADER
    with open(HEADER) as f:
        return f.read()


def test_every_declaration_has_a_prototype_of_its_arity(header):
    from mujoco_mpc_b200.engine import parse_header
    protos = parse_header(header)
    declared = set(re.findall(r"\b(mjpc_b200_[a-z_]+)\s*\(", header))
    assert declared and set(protos) == declared
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    for name in declared:
        params = re.search(r"\b" + name + r"\s*\(([^)]*)\)", code).group(1).strip()
        arity = 0 if params == "void" else params.count(",") + 1
        assert len(protos[name][1]) == arity, name


def test_non_int_returns(header):
    from mujoco_mpc_b200.engine import parse_header
    protos = parse_header(header)
    expect = {"mjpc_b200_version": C.c_char_p, "mjpc_b200_last_error": C.c_char_p,
              "mjpc_b200_estimator_last_error": C.c_char_p, "mjpc_b200_batch_estimator_last_error": C.c_char_p,
              "mjpc_b200_stream": C.c_void_p, "mjpc_b200_device_returns": C.c_void_p,
              "mjpc_b200_quadruped_transition_create": C.c_void_p, "mjpc_b200_track_transition_create": C.c_void_p,
              "mjpc_b200_shadow_transition_create": C.c_void_p, "mjpc_b200_launch_count": C.c_int64,
              "mjpc_b200_last_kernel_ms": C.c_float, "mjpc_b200_host_philox_normal": C.c_double,
              "mjpc_b200_destroy": None, "mjpc_b200_batch_planner_destroy": None, "mjpc_b200_agent_reset": None}
    for name, restype in expect.items():
        assert protos[name][0] is restype, name


def test_unknown_type_raises_naming_it():
    from mujoco_mpc_b200.engine import parse_header
    with pytest.raises(TypeError, match=r"long double.*mjpc_b200_scale\(long double s, int n\)"):
        parse_header("/* a comment */\nint mjpc_b200_scale(long double s,\n                     int n);\n")
    assert parse_header("int mjpc_b200_scale(const double *s, int n);")["mjpc_b200_scale"] == \
        (C.c_int, [C.POINTER(C.c_double), C.c_int])


def test_scalars_convert_through_the_prototype():
    """A numpy float64 time0 and a Python int timestep are converted to the header's double."""
    from mujoco_mpc_b200 import engine
    nodes = np.array([0.0, 1.5, 3.0, 4.5, 6.0])
    H = 5
    times, upper, frac = np.zeros(H), np.zeros(H, np.int32), np.zeros(H, np.float32)
    engine.load_library().mjpc_b200_host_policy_intervals(
        nodes.ctypes.data_as(C.POINTER(C.c_double)), len(nodes), np.float64(0.25), 1, H,
        times.ctypes.data_as(C.POINTER(C.c_double)), upper.ctypes.data_as(C.POINTER(C.c_int)),
        frac.ctypes.data_as(C.POINTER(C.c_float)))
    ref = engine.host_policy_intervals(nodes, 0.25, 1.0, H)
    for a, b in zip((times, upper, frac), ref):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(times, 0.25 + np.arange(H))
