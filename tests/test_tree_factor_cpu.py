"""The leaves-first tree factorisation of csrc/dev_data.cuh (warp_tree_factor_solve), restated in numpy lane by lane
and checked against numpy.linalg in fp64: the elimination schedule (DofTree), the right-hand side carried as one more
row, the kMinVal pivot clamp, and the fill check that sends Hessians with cross-branch couplings to the dense factor."""
import os
import re

import numpy as np
import pytest

from conftest import get_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_MIN_VAL = 1e-15


def ancestors(parent, j):
    out, a = [], parent[j]
    while a >= 0:
        out.append(a)
        a = parent[a]
    return out


def schedule(parent):
    """DofTree::col: by height above the leaves (leaves first), within one height by descending index."""
    n = len(parent)
    h = [0] * n
    for k in range(n - 1, -1, -1):
        if parent[k] >= 0:
            h[parent[k]] = max(h[parent[k]], h[k] + 1)
    return [j for lvl in range(max(h) + 1) for j in range(n - 1, -1, -1) if h[j] == lvl]


def tree_solve(A, b, parent):
    """warp_tree_factor_solve lane by lane: row[lane][k] = A[k][lane] (lane < n), row[n] = b."""
    n = len(parent)
    row = np.vstack([A.T, b[None, :]]).astype(np.float64)   # lanes 0..n
    il = np.zeros(n)
    for j in schedule(parent):
        p = max(row[j, j], K_MIN_VAL)
        il[j] = 1.0 / np.sqrt(p)
        row[:, j] *= il[j]
        for a in ancestors(parent, j):
            row[:, a] -= row[:, j] * row[a, j]
    xs = row[n, :].copy()   # y, the solution of G y = b
    for j in range(n):      # G^T x = y, root to leaves
        t = xs[j]
        for i in sorted(ancestors(parent, j)):
            t -= row[i, j] * xs[i]
        xs[j] = t * il[j]
    return xs


def fill_free(J, parent):
    """No constraint row couples two dofs of which neither is an ancestor of the other."""
    n = len(parent)
    anc = [set(ancestors(parent, j)) for j in range(n)]
    for r in J:
        nz = np.flatnonzero(r)
        if any(a != c and a not in anc[c] and c not in anc[a] for a in nz for c in nz):
            return False
    return True


def chain(parent, d):
    return [d] + ancestors(parent, d)


def tree_spd(parent, rng, scale=1.0):
    """A random SPD matrix with exactly the (dof, ancestor) pattern: sum of chain outer products plus a diagonal."""
    n = len(parent)
    A = np.diag(rng.uniform(0.5, 2.0, n) * scale)
    for d in range(n):
        v = np.zeros(n)
        v[chain(parent, d)] = rng.normal(size=len(chain(parent, d)))
        A += np.outer(v, v)
    return A


def model_parent(name):
    return [int(x) for x in np.asarray(get_model(name).dof_parentid)]


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_schedule_is_leaves_first_and_shorter_than_nv(name):
    parent = model_parent(name)
    order = schedule(parent)
    assert sorted(order) == list(range(len(parent)))
    pos = {j: t for t, j in enumerate(order)}
    for j in range(len(parent)):
        assert all(pos[a] > pos[j] for a in ancestors(parent, j))   # every dof before its ancestors
    levels = max(len(chain(parent, d)) for d in range(len(parent)))
    assert levels < len(parent)
    if name == "quadruped":
        assert levels == 9   # 6 base dofs + one 3-dof leg


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_generated_spec_holds_the_model_tree(name):
    text = open(os.path.join(ROOT, "mujoco_mpc_b200", "csrc", f"spec_{name}.h")).read()
    body = re.search(r"kDofParent\[64\] = \{([^}]*)\}", text).group(1)
    words = [int(x) for x in body.replace("\n", " ").split(",") if x.strip()]
    parent = model_parent(name)
    assert words[:len(parent)] == parent and all(w == -1 for w in words[len(parent):])


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_tree_solve_matches_numpy(name):
    parent = model_parent(name)
    rng = np.random.default_rng(7)
    for _ in range(20):
        A = tree_spd(parent, rng)
        b = rng.normal(size=len(parent))
        x = tree_solve(A, b, parent)
        ref = np.linalg.solve(A, b)
        assert np.allclose(x, ref, rtol=1e-10, atol=1e-10 * np.abs(ref).max())
        # G G^T = A: the Cholesky factor of the index-reversed matrix, reversed back
        L = np.linalg.cholesky(A[::-1, ::-1])
        assert np.allclose(L @ L.T, A[::-1, ::-1])


def test_tree_solve_ignores_entries_outside_the_pattern():
    parent = model_parent("quadruped")
    rng = np.random.default_rng(3)
    A = tree_spd(parent, rng)
    b = rng.normal(size=len(parent))
    junk = A.copy()
    anc = [set(ancestors(parent, j)) for j in range(len(parent))]
    for r in range(len(parent)):
        for c in range(len(parent)):
            if r != c and r not in anc[c] and c not in anc[r]:
                junk[r, c] = np.nan   # the device reads these words but never uses them
    assert np.array_equal(tree_solve(junk, b, parent), tree_solve(A, b, parent))


def test_near_singular_pivot_is_clamped_like_the_dense_factor():
    parent = model_parent("quadruped")
    n = len(parent)
    rng = np.random.default_rng(11)
    A = tree_spd(parent, rng)
    # make the ankle of the first leg (dof 8) a zero-mass leaf: its pivot is 0 and is clamped to kMinVal
    A[8, :] = 0.0
    A[:, 8] = 0.0
    b = rng.normal(size=n)
    b[8] = 0.0
    x = tree_solve(A, b, parent)
    assert np.all(np.isfinite(x)) and x[8] == 0.0
    keep = [d for d in range(n) if d != 8]
    ref = np.linalg.solve(A[np.ix_(keep, keep)], b[keep])
    assert np.allclose(x[keep], ref, rtol=1e-10, atol=1e-12)


def contact_row(parent, dofs, rng):
    r = np.zeros(len(parent))
    r[dofs] = rng.normal(size=len(dofs))
    return r


def test_fill_check_accepts_world_contacts_and_rejects_cross_branch_contacts():
    parent = model_parent("quadruped")
    n = len(parent)
    rng = np.random.default_rng(5)
    M = tree_spd(parent, rng)
    b = rng.normal(size=n)
    feet = [8, 11, 14, 17]
    # one-sided (floor) contacts at every foot: rows on one root-to-foot chain each
    J = np.array([contact_row(parent, chain(parent, f), rng) for f in feet for _ in range(3)])
    H = M + J.T @ np.diag(rng.uniform(0.1, 5.0, len(J))) @ J
    assert fill_free(J, parent)
    assert np.allclose(tree_solve(H, b, parent), np.linalg.solve(H, b), rtol=1e-10, atol=1e-10)
    # a contact between two feet: the row holds both legs' dofs (the common base dofs cancel)
    cross = contact_row(parent, [6, 7, 8, 9, 10, 11], rng)
    Jx = np.vstack([J, cross])
    Hx = M + Jx.T @ np.diag(rng.uniform(0.1, 5.0, len(Jx))) @ Jx
    assert not fill_free(Jx, parent)
    # the tree path would drop the fill the two legs create: the check is what keeps it exact
    assert not np.allclose(tree_solve(Hx, b, parent), np.linalg.solve(Hx, b), rtol=1e-6)
