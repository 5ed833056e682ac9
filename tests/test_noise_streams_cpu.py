"""CPU: the noise streams' integer words and fp64 normals, pinned to the published Philox4x32-10 known-answer vectors
(Salmon et al. 2011, Random123 kat_vectors), so that every fp64 truth of tests/test_gpu_noise_streams.py rests on a
checked restatement; the counter search those GPU tests draw at; and the host twin of the state-ensemble draws on
positive semi-definite, rank-deficient covariances."""
import numpy as np
import pytest

import plant_noise as PN
from conftest import get_model

KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


@pytest.mark.parametrize("case", range(len(KAT)))
def test_philox_restatements_reproduce_the_known_answers(case):
    from mujoco_mpc_b200.planner import philox4x32
    ctr, key, want = KAT[case]
    assert philox4x32(np.array([ctr], np.uint32), key)[0].tolist() == list(want)
    # the key-vectorised restatement, on counters (step, 0, element, tag): only the zero-c1 vector fits its layout
    if ctr[1] == 0:
        assert PN.philox_words([key[0]], ctr[0], ctr[2], ctr[3], key1=key[1])[0].tolist() == list(want)


def test_the_vectorised_words_are_the_planner_words():
    from mujoco_mpc_b200.planner import philox4x32
    seeds = np.array([0, 1, 0x5EED, 0xFFFFFFFF, 123456789], np.uint32)
    for tag in (PN.TAG_CTRL, PN.TAG_XFRC, PN.TAG_SENS):
        for step, e in ((0, 0), (7, 3), (0xFFFFFFFF, 83)):
            got = PN.philox_words(seeds, step, e, tag)
            for i, s in enumerate(seeds):
                ref = philox4x32(np.array([[step, 0, e, tag]], np.uint32), (int(s), 2))[0]
                assert got[i].tolist() == ref.tolist()


def test_the_host_knot_stream_is_the_restated_stream():
    """mjpc_b200_host_philox_normal (the host planners' knot noise, key (seed, 0), counter (iteration, candidate,
    knot, dof)) against fp64 Box-Muller on the restated words: the same words give the same double to 1e-15."""
    import ctypes
    from mujoco_mpc_b200.engine import load_library
    from mujoco_mpc_b200.planner import philox4x32
    lib = load_library()
    lib.mjpc_b200_host_philox_normal.restype = ctypes.c_double
    rng = np.random.default_rng(0)
    ctr = rng.integers(0, 1 << 32, (512, 4), dtype=np.uint64).astype(np.uint32)
    ctr[:8, 0] = 0xFFFFFFFF
    seeds = rng.integers(0, 1 << 32, 512, dtype=np.uint64).astype(np.uint32)
    for c, s in zip(ctr, seeds):
        z = PN.box_muller(philox4x32(c[None], (int(s), 0)))[0]
        got = lib.mjpc_b200_host_philox_normal(*(ctypes.c_uint32(int(v)) for v in (s, *c)))
        assert abs(got - z) <= 1e-15 * max(1.0, abs(z)), (c, s, got, z)


def test_the_belief_stream_is_the_restated_stream():
    """host_state_member on an identity covariance is mean + z in the velocity half: z restated from the words with
    key (seed + problem, 3), counter (iteration, k, e, 'BELF')."""
    from mujoco_mpc_b200.engine import host_state_member
    from mujoco_mpc_b200.planner import philox4x32
    m = get_model("quadruped")
    n = 2 * m.nv
    x = np.concatenate([np.asarray(m.key_qpos[0], float), np.zeros(m.nv)])
    for seed, it, b, k in ((7, 0, 0, 1), (0xFFFFFFFF, 3, 2, 31), (11, 0xFFFFFFFF, 0, 5)):
        out = host_state_member(m, x, np.eye(n), seed, it, b, k)
        ctr = np.array([[it, k, e, 0x42454C46] for e in range(n)], np.uint32)
        z = PN.box_muller(philox4x32(ctr, ((seed + b) & 0xFFFFFFFF, 3)))
        np.testing.assert_allclose(out[m.nq:], z[m.nv:], rtol=0, atol=1e-15 * 8)


@pytest.mark.parametrize("region", list(PN.REGIONS))
def test_the_counter_search_lands_in_its_regions(region):
    found = _search()
    cases = found[region]
    assert len(cases) >= 2, region
    i, lo, hi = PN.REGIONS[region]
    for seed, e in cases:
        w = int(PN.philox_words([seed], 0, e, PN.TAG_CTRL)[0, i])
        assert lo <= w < hi and 0 <= e < 12, (region, seed, e, hex(w))


_FOUND = {}


def _search():
    if not _FOUND:
        _FOUND.update(PN.search_counters(PN.TAG_CTRL, 12, per_region=2))
    return _FOUND


# ------------------------------------------------------------------------------------------ rank-deficient covariances
def _deficient(n, rank, scale, seed, m=None):
    """J J^T for J [n][rank] in general position (Gaussian columns), and an orthonormal basis of its range.  With a
    model, the rows of free and ball rotations are scaled so that their std stays below 0.1 rad: a member's tangent is
    then recovered by differentiate_pos, which wraps rotations to pi."""
    rng = np.random.default_rng(seed)
    J = rng.standard_normal((n, rank)) * np.sqrt(scale / n)
    if m is not None:
        for j in range(m.njnt):
            if m.jnt_type[j] in (0, 1):
                d = int(m.jnt_dofadr[j]) + (3 if m.jnt_type[j] == 0 else 0)
                J[d:d + 3] *= min(1.0, 0.1 / np.sqrt(scale))
    Q, _ = np.linalg.qr(J)
    return J @ J.T, Q


CASES = [(d, s, seed) for d in (1, 3) for s in (1e-6, 1e-2, 1e2) for seed in (0, 1)]


def _tangent(m, x, out):
    from mujoco_mpc_b200 import estimator
    return np.concatenate([estimator.differentiate_pos(m, x[:m.nq], out[:m.nq]), out[m.nq:] - x[m.nq:]])


@pytest.mark.parametrize("deficiency,scale,seed", CASES)
def test_a_rank_deficient_psd_covariance_is_accepted_and_drawn_in_its_range(deficiency, scale, seed):
    """The host twin accepts J J^T (rank n - 1 and n - 3, not axis-aligned) and draws L z in range(J): the component
    outside it is below 1e-9 of the draw.  Before the pivot tolerance, the factorisation refused most such matrices
    (a rounded pivot of about -1e-13 relative) and accepted rounded positive pivots with a division by their root."""
    from mujoco_mpc_b200.engine import host_state_member
    m = get_model("quadruped")
    n = 2 * m.nv
    P, Q = _deficient(n, n - deficiency, scale, seed, m)
    x = np.concatenate([np.asarray(m.key_qpos[0], float), np.zeros(m.nv)])
    worst = 0.0
    for k in range(1, 8):
        dx = _tangent(m, x, host_state_member(m, x, P, 5, 0, 0, k))
        out = dx - Q @ (Q.T @ dx)
        worst = max(worst, np.linalg.norm(out) / np.linalg.norm(dx))
    print("rank n-%d scale %g: largest share outside range(J) %.1e" % (deficiency, scale, worst))
    assert worst <= 1e-9


@pytest.mark.parametrize("deficiency", [1, 3])
def test_a_rank_deficient_covariance_is_drawn_with_its_covariance(deficiency):
    """About 4k draws: the sample covariance equals P to 5 standard errors (the bar of test_state_ensemble_cpu.py)."""
    from mujoco_mpc_b200.engine import host_state_member
    m = get_model("quadruped")
    n = 2 * m.nv
    P, _ = _deficient(n, n - deficiency, 1e-3, 7, m)
    x = np.concatenate([np.asarray(m.key_qpos[0], float), np.zeros(m.nv)])
    count = 31 * 132
    D = np.array([_tangent(m, x, host_state_member(m, x, P, 5, i // 31, 0, i % 31 + 1)) for i in range(count)])
    S = D.T @ D / count
    se = np.sqrt((np.outer(np.diag(P), np.diag(P)) + P ** 2) / count)
    assert np.all(np.abs(S - P) < 5 * se), np.max(np.abs(S - P) / se)


def test_the_tolerance_keeps_the_refusals():
    """A pivot below -tau, a pivot within tau of zero with a real coupling below it and a non-finite entry are still
    refused, at every scale; an exactly zero direction alone is still a zero column."""
    from mujoco_mpc_b200.engine import EngineError, host_state_member
    m = get_model("quadruped")
    n = 2 * m.nv
    x = np.concatenate([np.asarray(m.key_qpos[0], float), np.zeros(m.nv)])
    for s in (1e-6, 1.0, 1e2):
        P = np.eye(n) * s
        P[5, 5] = -1e-9 * s    # far below -tau_j = -n 2^-40 P_jj
        with pytest.raises(EngineError, match="not positive semi-definite"):
            host_state_member(m, x, P, 1, 0, 0, 1)
        P = np.eye(n) * s
        P[3, 3] = 0.0
        P[3, 4] = P[4, 3] = 1e-4 * s
        with pytest.raises(EngineError, match="not positive semi-definite"):
            host_state_member(m, x, P, 1, 0, 0, 1)
        P = np.eye(n) * s
        P[3, 3] = 1e-14 * s    # within tau of zero, but coupled far above rounding: an eigenvalue of -1e-8 s
        P[3, 4] = P[4, 3] = 1e-4 * s
        with pytest.raises(EngineError, match="not positive semi-definite"):
            host_state_member(m, x, P, 1, 0, 0, 1)
    P = np.eye(n)
    P[2, 2] = np.inf
    with pytest.raises(EngineError, match="non-finite"):
        host_state_member(m, x, P, 1, 0, 0, 1)
    P = np.eye(n) * 1e-3
    P[m.nv + 3, m.nv + 3] = 0.0
    out = host_state_member(m, x, P, 1, 0, 0, 1)
    assert out[m.nq + 3] == x[m.nq + 3] and out[m.nq + 4] != x[m.nq + 4]


def test_an_ill_conditioned_pd_covariance_is_factored_as_cholesky():
    """cond 1e10 is below 2^40 / n: every pivot is above its tau and the factor is numpy's Cholesky to rounding; so is
    a diagonal covariance of any spread."""
    from mujoco_mpc_b200.engine import host_state_member
    from mujoco_mpc_b200.planner import philox4x32
    m = get_model("quadruped")
    n = 2 * m.nv
    rng = np.random.default_rng(3)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    P = 1e-2 * (Q * np.logspace(0, -10, n)) @ Q.T
    P = 0.5 * (P + P.T)
    x = np.concatenate([np.asarray(m.key_qpos[0], float), np.zeros(m.nv)])
    out = host_state_member(m, x, P, 4, 1, 0, 2)
    ctr = np.array([[1, 2, e, 0x42454C46] for e in range(n)], np.uint32)
    dx = np.linalg.cholesky(P) @ PN.box_muller(philox4x32(ctr, (4, 3)))
    np.testing.assert_allclose(out[m.nq:] - x[m.nq:], dx[m.nv:], rtol=0, atol=1e-12)
    P = np.diag(10.0 ** np.linspace(2, -30, n))
    out = host_state_member(m, x, P, 4, 1, 0, 2)
    dx = np.sqrt(np.diag(P)) * PN.box_muller(philox4x32(ctr, (4, 3)))
    np.testing.assert_allclose(out[m.nq:] - x[m.nq:], dx[m.nv:], rtol=1e-15, atol=0)
