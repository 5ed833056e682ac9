"""CPU: the host definition of a model ensemble's score (mjpc_b200_host_ensemble_score), which the device's
ensemble_score_kernel must equal bit for bit, against a numpy restatement: the member returns sorted in descending
order with ties to the lower member, the first `worst` summed left to right in double, divided once by worst and
rounded to float; any failed member fails the candidate with exactly 1e6.  Also the NULL-handle refusals of the new
entry points."""
import ctypes as C

import numpy as np
import pytest

BAD_ARGUMENT = -1


def _restated(r, f, worst):
    r = np.asarray(r, np.float32)
    if np.any(np.asarray(f) != 0):
        return np.float32(1.0e6), 1
    order = sorted(range(len(r)), key=lambda k: (-float(r[k]), k))
    total = 0.0
    for k in order[:worst]:
        total += float(r[k])
    return np.float32(total / worst), 0


def _score(r, f, worst):
    from mujoco_mpc_b200.engine import host_ensemble_score
    return host_ensemble_score(r, f, worst)


def _check(r, f, worst):
    s, fl = _score(r, f, worst)
    e, ef = _restated(r, f, worst)
    assert fl == ef
    assert np.float32(s).tobytes() == e.tobytes(), (r, f, worst, s, e)
    return s


@pytest.mark.parametrize("K", [1, 3, 32])
def test_score_matches_the_restatement(K):
    rng = np.random.default_rng(K)
    for trial in range(50):
        # returns spread over decades, so that the order and the double sum both matter
        r = (rng.standard_normal(K) * 10.0 ** rng.integers(-3, 4, K)).astype(np.float32)
        for worst in sorted({1, min(2, K), K}):
            _check(r, np.zeros(K, np.uint8), worst)


@pytest.mark.parametrize("K", [3, 32])
def test_ties_take_the_lower_member(K):
    r = np.full(K, 0.25, np.float32)
    r[K // 2] = 7.0
    r[-1] = 7.0
    for worst in sorted({1, 2, K}):
        _check(r, np.zeros(K, np.uint8), worst)
    assert _score(r, np.zeros(K, np.uint8), 2)[0] == np.float32(7.0)


def test_a_worst_subset_is_the_largest_returns():
    r = np.array([1.0, 5.0, 3.0], np.float32)
    assert _score(r, np.zeros(3, np.uint8), 1)[0] == np.float32(5.0)
    assert _score(r, np.zeros(3, np.uint8), 2)[0] == np.float32(4.0)
    assert _score(r, np.zeros(3, np.uint8), 3)[0] == np.float32(3.0)


def test_the_sum_is_in_double_and_divided_once():
    # in float, 1e8 + 1 - 1e8 loses the 1; in double the mean of the three is exactly (2e8 + 1) / 3 rounded once
    r = np.array([1.0e8, 1.0, 1.0e8], np.float32)
    s = _check(r, np.zeros(3, np.uint8), 3)
    assert s == np.float32((1.0e8 + 1.0e8 + 1.0) / 3.0)


@pytest.mark.parametrize("K", [1, 3, 32])
def test_failed_members_fail_the_candidate(K):
    rng = np.random.default_rng(5)
    r = rng.standard_normal(K).astype(np.float32)
    one = np.zeros(K, np.uint8)
    one[K - 1] = 1
    r[K - 1] = 1.0e6   # what a failed rollout returns
    for worst in sorted({1, min(2, K), K}):
        s, f = _score(r, one, worst)
        assert f == 1 and s == np.float32(1.0e6)
        s, f = _score(r, np.ones(K, np.uint8), worst)
        assert f == 1 and s == np.float32(1.0e6)


def test_one_member_is_the_identity():
    rng = np.random.default_rng(9)
    for x in np.concatenate([rng.standard_normal(200) * 1e3, [0.0, 1e-30, 3.4e38, 1.0e6]]).astype(np.float32):
        s, f = _score([x], [0], 1)
        assert f == 0 and np.float32(s).tobytes() == np.float32(x).tobytes()


def test_out_of_range_arguments_write_nothing():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    r = np.ones(33, np.float32)
    fl = np.zeros(33, np.uint8)
    for K, worst in ((0, 1), (33, 1), (3, 0), (3, 4)):
        s, f = np.full(1, -7.0, np.float32), np.full(1, 9, np.uint8)
        lib.mjpc_b200_host_ensemble_score(r.ctypes.data_as(C.POINTER(C.c_float)), fl.ctypes.data_as(C.POINTER(C.c_uint8)),
                                          K, worst, s.ctypes.data_as(C.POINTER(C.c_float)),
                                          f.ctypes.data_as(C.POINTER(C.c_uint8)))
        assert s[0] == -7.0 and f[0] == 9


def test_null_handles_are_refused():
    from mujoco_mpc_b200.engine import load_library
    lib = load_library()
    assert lib.mjpc_b200_set_model_ensemble(None, None, 2, 1) == BAD_ARGUMENT
    assert lib.mjpc_b200_fetch_ensemble(None, None, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_fetch_trajectory_member(None, 0, 0, None, None, None, None, None, None) == BAD_ARGUMENT
    assert lib.mjpc_b200_planner_set_ensemble(None, None, 2, 1) == BAD_ARGUMENT
    assert lib.mjpc_b200_batch_planner_set_ensemble(None, None, 2, 1) == BAD_ARGUMENT
