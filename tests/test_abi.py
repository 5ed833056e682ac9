"""CPU: the C-ABI library loads and exports every symbol include/mjpc_b200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest


def test_header_symbols_exported():
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.engine import EXPORTS
    so = build.build()
    lib = ctypes.CDLL(so)
    hdr = open(os.path.join(os.path.dirname(build.HERE), "include", "mjpc_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(mjpc_b200_[a-z_]+)\s*\(", hdr)))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert sorted(EXPORTS) == declared
    lib.mjpc_b200_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.mjpc_b200_version()


def test_no_cpu_fallback():
    """Without a CUDA device create() must fail loudly with MJPC_B200_ERR_CUDA."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from conftest import get_model
    from mujoco_mpc_b200.engine import Engine, EngineError
    with pytest.raises(EngineError) as e:
        Engine(get_model("particle"), 4, 8)
    assert "-4" in str(e.value) or "CUDA" in str(e.value)


def test_product_does_not_import_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "mujoco_mpc_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and '"oracle/' not in txt and "../oracle" not in txt, f


def test_cpp_host_spline_and_noise_match_python_mirror():
    """The C++ host layer (TimeSpline::Sample restatement, injected Philox noise) vs the reference's spline known
    answers (spline_test.cc:115-158) and the Python mirror - no GPU needed."""
    import numpy as np
    from mujoco_mpc_b200 import build
    from mujoco_mpc_b200.planner import philox_normal, sample_spline
    lib = ctypes.CDLL(build.build())
    lib.mjpc_b200_host_philox_normal.restype = ctypes.c_double
    dp = ctypes.POINTER(ctypes.c_double)

    def sample(times, values, interp, t):
        times = np.ascontiguousarray(times, float); values = np.ascontiguousarray(values, float)
        out = np.zeros(values.shape[1])
        lib.mjpc_b200_host_spline_sample(times.ctypes.data_as(dp), values.ctypes.data_as(dp), len(times), values.shape[1],
                                         interp, ctypes.c_double(t), out.ctypes.data_as(dp))
        return out
    np.testing.assert_allclose(sample([1, 2], [[1.0, 2], [3, 4]], 0, 1.5), [1, 2])
    np.testing.assert_allclose(sample([1, 2], [[1.0, 2], [3, 4]], 1, 1.5), [2, 3])
    np.testing.assert_allclose(sample([0, 1, 2, 3], [[1.0, 2], [1, 2], [3, 4], [3, 4]], 2, 1.5), [2, 3])
    for x in np.arange(0.0, 1.0001, 0.125):
        np.testing.assert_allclose(sample([-1, 0, 1], [[1.0], [0.0], [1.0]], 2, x), [-x ** 3 + 2 * x ** 2], atol=1e-12)
    rng = np.random.default_rng(2)
    times = np.cumsum(rng.uniform(0.1, 0.4, 5)); vals = rng.normal(size=(5, 3))
    for interp in (0, 1, 2):
        for t in np.linspace(times[0] - 0.2, times[-1] + 0.2, 23):
            np.testing.assert_allclose(sample(times, vals, interp, t), sample_spline(times, vals, interp, t), atol=1e-12)
    z = philox_normal(7, 4, 3, 12)
    for (i, k, d) in ((0, 0, 0), (3, 2, 11), (1, 1, 5)):
        zc = lib.mjpc_b200_host_philox_normal(ctypes.c_uint32(0x5EED), ctypes.c_uint32(7), ctypes.c_uint32(i),
                                              ctypes.c_uint32(k), ctypes.c_uint32(d))
        assert abs(zc - z[i, k, d]) < 1e-12


def test_agent_steps_rule():
    """agent.cc:107,292-293: steps_ = max(min(horizon / timestep + 1, 512), 1) truncated to int (SURVEY.md App. B.9)."""
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    st = lib.mjpc_b200_agent_steps
    assert st(0.47, 0.01) == 47          # 0.47 / 0.01 + 1 = 47.99999999999999 -> 47
    assert st(0.4701, 0.01) == 48        # the Shadow-Hand workaround of SURVEY.md 8d
    assert st(0.63, 0.01) == 64 and st(0.31, 0.01) == 32 and st(0.635, 0.005) == 128
    assert st(100.0, 0.01) == 512 and st(0.0, 0.01) == 1
