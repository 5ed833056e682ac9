"""CPU: the fp64 oracle's contact constraint solve (oracle/physics.h make_constraint, update_constraint, line_search,
solve_constraints) against an independent fp64 restatement of its convex problem, on the scenes of
tests/solver_scenes.py, for both cones and impratio 1, 10 and 100.

The device and the oracle were written from the same description, so an error they share passes every parity test.
solver_scenes.Problem restates the problem without the oracle's recursions: J from refmath's world-frame body
Jacobians and the oracle's contact frame, diagApprox from body_invweight0, the impedance, K, B and aref from solref
and solimp, R with the impratio and friction-ratio scaling, pyramidal edges J_n +- mu_k J_t,k, and the cost, its
gradient and a generalised Hessian derived by hand from MuJoCo's published convex formulation.  It takes the oracle's
contact geometry (dist, pos, frame: pinned by tests/test_oracle_contacts.py) and qacc_smooth (pinned by
tests/test_smooth_dynamics_cpu.py) as input.

Stated, not derived: the pyramidal edges' R = 2 mu^2 R_0 with mu = friction[0] / sqrt(impratio) is transcribed from
the implementation; MuJoCo is not vendored, so the rule is not checked against its source.

Asserted:
  rows         every row of Oracle.efc_debug matches the restatement: type, id and friction loss exactly, J to 1e-12
               of each row's largest entry, every scalar to 1e-12 of itself; also on the Quadruped's stance, sliding
               and self-contact states (joint limits, friction loss, parameter mixing);
  optimality   with tolerance 1e-15 and 1000 iterations, the restated gradient M (a - a_smooth) - J' f at the oracle's
               qacc is below OPT_BAR = 1e-8 of the force scale.  Not 1e-10: the fp64 line search accepts a step on
               the published cost comparison, and near the optimum the decrease a Newton step buys (~ g' H^-1 g) falls
               below the rounding of the cost (~ eps |cost|) while the gradient is still ~ 1e-9 of its scale; the
               solve then stops with alpha = 0 (measured worst 2.9e-9, an elliptic condim-4 box sliding at
               impratio 100; tolerance 0 stops at the same point);
  minimiser    scipy's trust-region Newton on the restated cost, from qacc_smooth, lands within 1e-8 of the oracle,
               or within the strong-convexity bound (|g(scipy)| + |g(oracle)|) / lambda_min(M) where both stop on the
               cost's resolution (1 of 156 cases); both gradients are bounded;
  closed forms a contact in the elliptic cone zone lies on the cone, sum_j (f_j / friction_j)^2 = f_N^2; the
               quadratic zone has f = -D jar, the separated zone f = 0; pyramidal edge forces are >= 0 and sum to the
               contact's normal force in the restated problem; the resting box's normal forces sum to m g at the
               closed-form equilibrium penetration (solver_scenes.rest_penetration), where qacc = 0;
  warm starts  the explicit starts the GPU stepped solves use cost less than qacc_smooth and, over the elliptic
               scenes, put contacts in every zone; two starts on the resting box have a tangential jar of exactly 0
               with N < 0 and with N >= 0 (the two Tn <= 0 branches of the update).
"""
import numpy as np
import pytest

import solver_scenes as S

SCENES = S.scenes()
VARIANTS = S.variants()
IDS = [f"{k}-{c}-{i}" for k, c, i in VARIANTS]
_CACHE = {}
OPT_BAR = 1e-8
BEYOND_1E8 = {True: 0, False: 0}   # minimiser cases that needed the strong-convexity bound / met 1e-8


def _oracle(key, cone, impratio, option="", precision=64):
    ck = (key, cone, impratio, option, precision)
    if ck not in _CACHE:
        from mujoco_mpc_b200.blob import to_blob
        from oracle import pyoracle
        m = S.compile_scene(SCENES[key].xml(cone, impratio, option))
        _CACHE[ck] = (m, pyoracle.Oracle(to_blob(m), m, precision))
    return _CACHE[ck]


def _rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-300) if b.size else 0.0


def _solve(o, m, q, v):
    return o.efc_debug(q, v, np.zeros(m.nu), np.zeros(0))


def _paths(key, cone, m, r):
    sc = SCENES[key]
    assert S.model_path(m) == sc.path, (key, S.model_path(m))
    assert (S.line_search_items(m, r) <= 32) == sc.is_cached(cone), (key, S.line_search_items(m, r))


@pytest.mark.parametrize("key,cone,impratio", VARIANTS, ids=IDS)
def test_rows_match_restatement(oracle_lib, key, cone, impratio):
    m, o = _oracle(key, cone, impratio)
    for name, q, v in SCENES[key].states(m, cone, impratio):
        r = _solve(o, m, q, v)
        assert r["warning"] == 0 and r["ncon"] > 0, (name, r["warning"], r["ncon"])
        _paths(key, cone, m, r)
        p = S.Problem(m, q, v, r)
        assert p.ne == r["nefc"]
        assert np.array_equal(p.type, r["efc_type"]) and np.array_equal(p.id, r["efc_id"]), name
        assert np.array_equal(p.floss, r["efc_frictionloss"]), name
        # per row: J against its own largest entry, every scalar against itself
        Jrow = np.abs(r["efc_J"]).max(1, keepdims=True) + 1e-300
        assert (np.abs(p.J - r["efc_J"]) <= 1e-12 * Jrow).all(), (name, (np.abs(p.J - r["efc_J"]) / Jrow).max())
        for k, mine in (("efc_pos", p.pos), ("efc_margin", p.margin), ("efc_diagApprox", p.diag), ("efc_R", p.R),
                        ("efc_D", p.D), ("efc_aref", p.aref)):
            err = np.abs(mine - r[k]) / (np.abs(r[k]) + 1e-300)
            assert (err < 1e-12).all() or (np.abs(mine - r[k]) <= 1e-12 * np.abs(r[k])).all(), (name, k, err.max())
        assert _rel(p.M, r["qM"]) < 1e-12, name
        mu = np.array([c["mu"] for c in p.contacts])
        assert _rel(mu, r["mu"]) < 1e-12 and np.array_equal([c["adr"] for c in p.contacts], r["efc_address"])


def _optimal(key, cone, impratio):
    return _oracle(key, cone, impratio, ' tolerance="1e-15" iterations="1000"')


@pytest.mark.parametrize("key,cone,impratio", VARIANTS, ids=IDS)
def test_oracle_qacc_is_optimal(oracle_lib, key, cone, impratio):
    m, o = _optimal(key, cone, impratio)
    for name, q, v in SCENES[key].states(m, cone, impratio):
        r = _solve(o, m, q, v)
        p = S.Problem(m, q, v, r)
        g = p.grad(r["qacc"])
        scale = p.grad_scale(r["qacc"]).max() + np.abs(r["qfrc_smooth"]).max()
        assert np.abs(g).max() < OPT_BAR * scale, (name, np.abs(g).max(), scale)
        assert _rel(p.force(r["qacc"]), r["efc_force"]) < 1e-9, name


@pytest.mark.parametrize("key,cone,impratio", VARIANTS, ids=IDS)
def test_independent_minimiser_agrees(oracle_lib, key, cone, impratio):
    m, o = _optimal(key, cone, impratio)
    for name, q, v in SCENES[key].states(m, cone, impratio):
        r = _solve(o, m, q, v)
        p = S.Problem(m, q, v, r)
        a = p.minimise()
        scale = p.grad_scale(a).max() + np.abs(r["qfrc_smooth"]).max()
        assert np.abs(p.grad(a)).max() < 10 * OPT_BAR * scale, name     # scipy's own stop (worst 1.04e-8)
        assert np.abs(p.grad(r["qacc"])).max() < OPT_BAR * scale, name
        # the cost is lambda_min(M)-strongly convex (the constraint cost is convex), so each point lies within
        # |g| / lambda_min(M) of the optimum; that bound, from the two measured gradients, is what the issue's 1e-8
        # gives way to on the stiffest problems (impratio 100, where both solvers stop on the cost's resolution)
        lam = np.linalg.eigvalsh(p.M)[0]
        bound = (np.linalg.norm(p.grad(a)) + np.linalg.norm(p.grad(r["qacc"]))) / lam
        err = np.linalg.norm(a - r["qacc"])
        assert err < max(1e-8 * (np.abs(r["qacc"]).max() + 1), bound), (name, err, bound)
        BEYOND_1E8[err > 1e-8 * (np.abs(r["qacc"]).max() + 1)] += 1


@pytest.mark.parametrize("key,cone,impratio", VARIANTS, ids=IDS)
def test_forces_closed_forms(oracle_lib, key, cone, impratio):
    m, o = _optimal(key, cone, impratio)
    for name, q, v in SCENES[key].states(m, cone, impratio):
        r = _solve(o, m, q, v)
        p = S.Problem(m, q, v, r)
        f, jar = r["efc_force"], r["efc_J"] @ r["qacc"] - r["efc_aref"]
        fs = np.abs(f).max() + 1e-300
        # rounding of jar recomputed here: eps x the terms it is the difference of, times D
        fr_tol = 1e-13 * r["efc_D"] * (np.abs(r["efc_J"]) @ np.abs(r["qacc"]) + np.abs(r["efc_aref"])) + 1e-12 * fs
        zones = p.zones(r["qacc"])
        for c, cd in enumerate(p.contacts):
            a, dim = cd["adr"], cd["dim"]
            rows = slice(a, a + cd["nrow"])
            if p.kind[a] == "edge":
                assert (f[rows] >= -1e-12 * fs).all(), (name, f[rows])
                # every edge pushes along n +- f_k t_k, so the contact's normal force is the sum of its edge forces:
                # against the normal force of the restated problem at the same qacc
                fn = p.force(r["qacc"])[rows].sum()
                assert abs(f[rows].sum() - fn) <= 1e-9 * fs, (name, c, f[rows].sum(), fn)
            elif p.kind[a] == "cone":
                st = r["efc_state"][a]
                if zones[a] == "cone":
                    assert st == 4
                    ft = f[a + 1:a + dim] / cd["friction"][:dim - 1]
                    assert abs(np.sum(ft ** 2) - f[a] ** 2) < 1e-12 * f[a] ** 2 + 1e-24, (name, c)
                elif zones[a] == "bottom":
                    assert st == 1 and (np.abs(f[rows] + r["efc_D"][rows] * jar[rows]) <= fr_tol[rows]).all()
                else:
                    assert st == 0 and (f[rows] == 0).all()
        for i in range(r["nefc"]):
            if p.kind[i] in ("edge", "one"):
                assert (f[i] == 0) == (jar[i] >= 0) and (jar[i] >= 0 or abs(f[i] + r["efc_D"][i] * jar[i]) <= fr_tol[i])


@pytest.mark.parametrize("cone", S.CONES)
@pytest.mark.parametrize("impratio", S.IMPRATIOS)
def test_resting_box_carries_its_weight(oracle_lib, cone, impratio):
    """At the closed-form equilibrium penetration (solver_scenes.rest_penetration: the soft-contact law of
    test_oracle_invariants' resting sphere, with the box's four corners and, for the pyramid, its edges' R) the box
    is in equilibrium: qacc = 0 and the normal forces carry m g."""
    m, o = _oracle("box", cone, impratio)
    name, q, v = SCENES["box"].states(m, cone, impratio)[0]
    assert name == "rest"
    r = _solve(o, m, q, v)
    assert r["ncon"] == 4 and np.abs(r["qacc"]).max() < 1e-9 * S.G, r["qacc"]
    f = r["efc_force"]
    normal = f.sum() if cone == "pyramidal" else f[r["efc_address"]].sum()
    assert abs(normal - S.BOX_MASS * S.G) < 1e-9 * S.BOX_MASS * S.G, normal


def warm_starts(m, o, key, cone, impratio):
    """[(state name, qpos, qvel, start name, start)] for the stepped solves: perturbations of the fp64 optimum, and on
    the resting elliptic box two starts whose tangential jar is exactly 0 (N < 0 and N >= 0)."""
    out = []
    for si, (name, q, v) in enumerate(SCENES[key].states(m, cone, impratio)):
        r = _solve(o, m, q, v)
        p = S.Problem(m, q, v, r)
        for k, a in enumerate(S.optimum_starts(p, r["qacc"], seed=1000 * si + 17)):
            out.append((name, q, v, f"perturbed{k}", a))
        if key == "box" and cone == "elliptic" and name == "rest":
            aref = r["efc_aref"][r["efc_address"][0]]
            for sname, z in (("tangent0_pressing", -0.5 * S.G), ("tangent0_lifting", 2.0 * aref)):
                a = np.zeros(m.nv); a[2] = z
                out.append((name, q, v, sname, a))
    return out


def test_warm_starts_cover_the_zones(oracle_lib):
    seen = set()
    branches = set()
    for key, cone, impratio in VARIANTS:
        m, o = _optimal(key, cone, impratio)
        for name, q, v, sname, a in warm_starts(m, o, key, cone, impratio):
            r = _solve(o, m, q, v)
            p = S.Problem(m, q, v, r)
            assert p.cost(a) < p.cost(p.a_smooth), (key, cone, impratio, name, sname)
            if cone == "elliptic":
                seen.update(z for z in p.zones(a) if z is not None)
            if sname.startswith("tangent0"):
                x = p.J @ a - p.aref
                for c in p.contacts:
                    ad = c["adr"]
                    assert (x[ad + 1:ad + 3] == 0).all()
                    branches.add("N<0" if x[ad] < 0 else "N>=0")
    assert {"top", "bottom", "cone"} <= seen, seen
    assert branches == {"N<0", "N>=0"}, branches


def test_quadruped_rows_and_optimality(oracle_lib):
    """The Quadruped's stance, sliding and self-contact states (tests/test_gpu_constraint_solve.py): its joint-limit,
    friction-loss and contact rows match the restatement, and the oracle's qacc minimises the restated problem."""
    from conftest import get_model, mocap_of
    from mujoco_mpc_b200.blob import to_blob
    m = get_model("quadruped")
    mc = mocap_of(m)
    o = oracle_lib.Oracle(to_blob(m), m, 64)
    for name, q, v in S.quadruped_states(m) + [S.self_contact_state(m, o)]:
        r = o.efc_debug(q, v, np.zeros(m.nu), mc)
        assert r["warning"] == 0 and r["ncon"] >= 2, name
        if name == "self_contact":     # a contact between two moving bodies: the dense-fallback factor on the device
            assert any(m.geom_bodyid[g1] > 0 and m.geom_bodyid[g2] > 0 for g1, g2 in zip(r["geom1"], r["geom2"]))
        p = S.Problem(m, q, v, r, mocap=mc)
        assert np.array_equal(p.type, r["efc_type"]) and np.array_equal(p.id, r["efc_id"]), name
        Jrow = np.abs(r["efc_J"]).max(1, keepdims=True) + 1e-300
        assert (np.abs(p.J - r["efc_J"]) <= 1e-12 * Jrow).all(), name
        for k, mine in (("efc_pos", p.pos), ("efc_R", p.R), ("efc_aref", p.aref)):
            assert (np.abs(mine - r[k]) <= 1e-12 * np.abs(r[k]) + 1e-300).all(), (name, k)
        g = np.abs(p.grad(r["qacc"])).max()
        assert g < OPT_BAR * (p.grad_scale(r["qacc"]).max() + np.abs(r["qfrc_smooth"]).max()), (name, g)


def test_zz_minimiser_report():
    """How many minimiser cases met the issue's 1e-8 directly (printed with -s)."""
    print("independent minimiser: %d cases within 1e-8, %d within the strong-convexity bound only"
          % (BEYOND_1E8[False], BEYOND_1E8[True]))
