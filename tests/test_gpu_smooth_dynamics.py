"""GPU: the device's smooth dynamics (k_kinematics, k_com_pos, k_crb, k_com_vel, the RNE bias of k_smooth_forces and the
position update of k_euler) against the fp64 oracle on the scenes of tests/smooth_scenes.py.  The oracle's smooth
dynamics are pinned to an independent fp64 restatement by tests/test_smooth_dynamics_cpu.py.

Bars.  Per case and quantity the bar is 4 x the error of the oracle's fp32 instantiation against its fp64 one plus a
floor of 16 fp32 ulps of the quantity's scale (max |fp64| + 1), for qM, qacc, next_qvel, the non-quaternion entries of
next_qpos and the quaternion entries of next_qpos.  The fp32 error at one input is one draw of its round-off, and
where M is ill-conditioned (cond(qM) ~ 4e3 on the forest scene) draws differ by 6x: the forest's first case met an fp32
oracle error of 9e-5 in qacc where the same case with inputs one ulp away gives up to 6e-4, and the device 7e-4.  So
the fp32 error taken is the largest over the case and NEIGHBOURS copies of it whose fp32 inputs differ from it by one
ulp in some entries, each against the fp64 oracle at the same input.  Every quaternion the device returns is unit-norm
to 4 ulps.

Translation invariance.  The far cases (x = 1e2 and 1e3 m) are compared on the device with their twin at the origin.
The state is stored in fp32, so x itself carries up to half an ulp of x (3e-5 m at 1e3) and every offset the kinematics
forms as a difference of two world positions (body com to subtree com, joint anchor to subtree com) carries up to
one ulp of x.  To first order that is a relative error of 2 ulp(x) / L in qM, qacc and next_qvel, L = 0.02 m being the
smallest such offset in the scene: that is their bar (of the quantity's scale, max |origin twin| + 1), h^2 / 2 of the
qacc bar plus 16 ulps is the quaternions', and next_qpos must move by x to 2 ulps of x.  These bars come from the fp32
state, not from the fp32 oracle; on the H100 the x = 1e3 case used under 5 % of them.

Static instances.  The Quadruped and Humanoid Track run their own kernel instances: step_batch with the dense factor
and rollout_spline with the dof-tree factor.  Airborne extreme states (fast trunk spin, large joint velocities, a
non-unit base quaternion, x = 1e3) go through both and through the generic instance (MJPC_B200_NO_STATIC=1), each
against the fp64 oracle with the fp32-oracle bar; the oracle's qM and qfrc_bias at the same states are pinned to the
restatement on the CPU.  test_zz_report prints the largest error as a fraction of its bar per group.
"""
import numpy as np
import pytest

import smooth_scenes as S
from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -23
RATIOS = {}
_CACHE = {}
SCENES = S.scenes()
CASES = [(k, c) for k, s in SCENES.items() for c in s.cases]


def _ratio(group, err, bar):
    RATIOS[group] = max(RATIOS.get(group, 0.0), float(err) / bar)
    return err <= bar


def _get(key):
    if key not in _CACHE:
        from mujoco_mpc_b200.blob import to_blob
        from mujoco_mpc_b200.engine import Engine
        from oracle import pyoracle
        m = SCENES[key].compile()
        _CACHE[key] = (m, Engine(m, 8, 4), pyoracle.Oracle(to_blob(m), m, 64), pyoracle.Oracle(to_blob(m), m, 32))
    return _CACHE[key]


def _mocap(m, mocap):
    if mocap is not None:
        return np.asarray(mocap, float)
    return mocap_of(m)


def quat_slots(m):
    from mujoco_mpc_b200.mjcf import JNT_BALL, JNT_FREE
    out = []
    for j in range(m.njnt):
        if m.jnt_type[j] in (JNT_FREE, JNT_BALL):
            a = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == JNT_FREE else 0)
            out += list(range(a, a + 4))
    return np.array(out, int)


def _split(m, x):
    """name -> array: qM, qacc, next_qvel, next_qpos (non-quaternion entries), next_quat."""
    qs = quat_slots(m)
    rest = np.setdiff1d(np.arange(m.nq), qs)
    return dict(qM=np.asarray(x["qM"], float), qacc=np.asarray(x["qacc"], float),
                next_qvel=np.asarray(x["next_qvel"], float), next_qpos=np.asarray(x["next_qpos"], float)[rest],
                next_quat=np.asarray(x["next_qpos"], float)[qs])


NEIGHBOURS = 4


def _neighbour(x, k):
    """Copy k of input x: its fp32 rounding moved by one ulp up or down in about two thirds of its non-zero entries."""
    x32 = np.atleast_1d(np.asarray(x, np.float32))
    sgn = np.random.default_rng(k).integers(-1, 2, x32.size) * (x32 != 0)
    out = np.where(sgn > 0, np.nextafter(x32, np.float32(np.inf)), np.where(sgn < 0, np.nextafter(x32, np.float32(-np.inf)), x32))
    return out.astype(float).reshape(np.shape(x))


def _fp32_pairs(run, *args):
    """[(fp64 result, fp32 result)] of run(precision, *inputs) on the case and its NEIGHBOURS copies."""
    out = []
    for k in range(NEIGHBOURS + 1):
        a = args if k == 0 else [_neighbour(x, k) for x in args]
        out.append((run(64, *a), run(32, *a)))
    return out


def _check(group, m, dev, r64, pairs, keys=None):
    d, a = _split(m, dev), _split(m, r64)
    sp = [(_split(m, x), _split(m, y)) for x, y in pairs]
    out = {}
    for k in keys or d:
        if d[k].size == 0:
            continue
        err = np.abs(d[k] - a[k]).max()
        err32 = max(np.abs(y[k] - x[k]).max() for x, y in sp)
        bar = 4 * err32 + 16 * ULP * (np.abs(a[k]).max() + 1)
        out[k] = (err, err32, bar)
        assert _ratio(f"{group} {k}", err, bar), (group, k, err, err32, bar)
    return out


def _unit_quats(group, m, qpos):
    qs = quat_slots(m).reshape(-1, 4)
    for s in qs:
        e = abs(np.linalg.norm(np.asarray(qpos, float)[s]) - 1)
        assert _ratio(group + " |quat| - 1", e, 4 * ULP), (group, s, e)


# ---------------------------------------------------------------------------------------------- generic instance
@pytest.mark.parametrize("key,case", CASES, ids=[f"{k}-{c[0]}" for k, c in CASES])
def test_step_debug_matches_fp64(key, case):
    m, e, o64, o32 = _get(key)
    name, q, v, mocap = case
    mc = _mocap(m, mocap)
    u = np.zeros(m.nu)
    g = e.step_debug(q, v, u, mc)
    r64 = o64.forward_debug(q, v, u, mc)
    pairs = _fp32_pairs(lambda p, q, v: (o64 if p == 64 else o32).forward_debug(q, v, u, mc), q, v)
    assert g["warning"] == r64["warning"] == 0 and g["nefc"] == r64["nefc"] == 0 and g["ncon"] == 0
    res = _check(key, m, g, r64, pairs)
    print("%s %s: " % (key, name) + ", ".join("%s %.2e (fp32 oracle %.2e, bar %.2e)" % (k, *x) for k, x in res.items()))
    _unit_quats(key, m, g["next_qpos"])


@pytest.mark.parametrize("key", list(SCENES))
def test_step_batch_matches_fp64(key):
    m, e, o64, o32 = _get(key)
    cases = SCENES[key].cases
    for mc in {None if c[3] is None else tuple(c[3]) for c in cases}:
        sub = [c for c in cases if (None if c[3] is None else tuple(c[3])) == mc]
        q = np.stack([c[1] for c in sub]); v = np.stack([c[2] for c in sub]); u = np.zeros((len(sub), m.nu))
        mca, t = _mocap(m, mc), np.zeros(len(sub))
        g, r64 = e.step_batch(q, v, u, mca, t), o64.step_batch(q, v, u, mca, t)
        assert not g["warning"].any() and not r64["warning"].any()
        for i in range(len(sub)):
            pick = lambda x: {k: x[k][i] for k in ("qacc", "next_qpos", "next_qvel")} | {"qM": np.zeros(0)}
            pairs = _fp32_pairs(lambda p, q, v: (o64 if p == 64 else o32).forward_debug(q, v, u[i], mca), q[i], v[i])
            _check(key + " (step_batch)", m, pick(g), pick(r64), pairs, ("qacc", "next_qvel", "next_qpos", "next_quat"))
            _unit_quats(key + " (step_batch)", m, g["next_qpos"][i])


def test_far_cases_match_their_twin_at_the_origin():
    m, e, _, _ = _get("far")
    cases = {c[0]: c for c in SCENES["far"].cases}
    base = cases["origin"]
    g0 = e.step_debug(base[1], base[2], np.zeros(0), np.zeros(0))
    L = 0.02
    for name, q, v, _ in SCENES["far"].cases:
        x = S.far_twin(name)
        if not x:
            continue
        g = e.step_debug(q, v, np.zeros(0), np.zeros(0))
        ulpx = np.spacing(np.float32(x))
        for k in ("qM", "qacc", "next_qvel"):
            err = np.abs(g[k] - g0[k]).max()
            bar = 2 * ulpx / L * (np.abs(g0[k]).max() + 1)
            print("far %s %s: device vs origin twin %.2e (bar %.2e)" % (name, k, err, bar))
            assert _ratio(f"far translation {k}", err, bar), (name, k, err, bar)
        d = g["next_qpos"].astype(float) - g0["next_qpos"]
        qs = quat_slots(m)
        rest = np.setdiff1d(np.arange(m.nq), qs)
        dx = np.abs(d[0] - x)
        other = np.abs(d[rest[1:]]).max()
        assert _ratio("far translation next_qpos x", dx, 2 * ulpx), (name, dx)
        assert _ratio("far translation next_qpos other", other, 2 * ulpx), (name, other)
        # the quaternion moves by h^2 / 2 times the angular qacc's difference
        h = m.opt_timestep
        err = np.abs(d[qs]).max()
        bar = 0.5 * h * h * 2 * ulpx / L * (np.abs(g0["qacc"]).max() + 1) + 16 * ULP
        assert _ratio("far translation next_quat", err, bar), (name, err, bar)


# ---------------------------------------------------------------------------------------------- static instances
STATIC = ["quadruped", "humanoid_track"]


@pytest.fixture(scope="module")
def static_rigs():
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200.engine import Engine
    from oracle import pyoracle
    out = {}
    for name in STATIC:
        m = get_model(name)
        out[name] = (m, Engine(m, 8, 8), pyoracle.Oracle(to_blob(m), m, 64), pyoracle.Oracle(to_blob(m), m, 32))
    yield out
    for m, e, _, _ in out.values():
        e.close()


def _step_batch(e, m, q, v, u, mc):
    return e.step_batch(q[None], v[None], u[None], mc, np.zeros(1))


def _first(x):
    return {k: x[k][0] for k in ("qacc", "next_qpos", "next_qvel")} | {"qM": np.zeros(0)}


@pytest.mark.parametrize("name", STATIC)
def test_static_instances_match_fp64_on_extreme_states(static_rigs, name, monkeypatch):
    m, e, o64, o32 = static_rigs[name]
    mc = mocap_of(m)
    H, P = 4, 2
    keys = ("qacc", "next_qvel", "next_qpos", "next_quat")
    for case, q, v in S.extreme_states(m):
        u = np.zeros(m.nu)
        r64 = _step_batch(o64, m, q, v, u, mc)
        pairs = _fp32_pairs(lambda p, q, v: _first(_step_batch(o64 if p == 64 else o32, m, q, v, u, mc)), q, v)
        assert not r64["warning"].any() and int(r64["ncon"][0]) == 0
        monkeypatch.delenv("MJPC_B200_NO_STATIC", raising=False)
        st = _step_batch(e, m, q, v, u, mc)
        assert e.last_kernel_shape == 1 and not st["warning"].any()
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
        ge = _step_batch(e, m, q, v, u, mc)
        assert e.last_kernel_shape == 0
        monkeypatch.delenv("MJPC_B200_NO_STATIC")
        for inst, g in (("static", st), ("generic", ge)):
            res = _check(f"{name} step_batch ({inst})", m, _first(g), _first(r64), pairs, keys)
            print("%s %s step_batch %s: " % (name, case, inst) +
                  ", ".join("%s %.2e (fp32 oracle %.2e, bar %.2e)" % (k, *x) for k, x in res.items()))
            _unit_quats(f"{name} step_batch ({inst})", m, g["next_qpos"][0])
        # the first steps of a rollout (dof-tree factor in the static instance), zero-order hold of ctrl 0
        state = np.concatenate([q, v])
        knots = np.zeros((1, P, m.nu))
        kt = np.arange(P) * (H - 1) * m.opt_timestep
        ro64 = o64.rollout_spline(state, 0.0, mc, knots, kt, 0, H, nthreads=1, full=True)
        rpairs = _fp32_pairs(lambda p, s: (o64 if p == 64 else o32).rollout_spline(s, 0.0, mc, knots, kt, 0, H, nthreads=1,
                                                                                    full=True)["states"][0], state)
        for inst in ("static", "generic"):
            if inst == "generic":
                monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
            ret, fail, _ = e.rollout_spline(state, 0.0, mc, knots, kt, 0, H)
            assert e.last_kernel_shape == (1 if inst == "static" else 0) and not fail.any()
            tr = e.fetch_all()
            monkeypatch.delenv("MJPC_B200_NO_STATIC", raising=False)
            for k in range(1, H):
                pick = lambda s: {"next_qpos": s[:m.nq], "next_qvel": s[m.nq:], "qacc": np.zeros(m.nv),
                                  "qM": np.zeros(0)}
                res = _check(f"{name} rollout ({inst}) step {k}", m, pick(tr["states"][0, k]),
                             pick(ro64["states"][0, k]), [(pick(a[k]), pick(b[k])) for a, b in rpairs],
                             ("next_qvel", "next_qpos", "next_quat"))
                _unit_quats(f"{name} rollout ({inst})", m, tr["states"][0, k, :m.nq])
            print("%s %s rollout %s step %d: " % (name, case, inst, H - 1) +
                  ", ".join("%s %.2e (fp32 oracle %.2e, bar %.2e)" % (k, *x) for k, x in res.items()))


def test_zz_report():
    """Largest error as a fraction of its bar, per group (printed with -s)."""
    for k in sorted(RATIOS):
        print(f"{k:60s} {RATIOS[k]:.3f}")
    assert all(v <= 1 for v in RATIOS.values())
    for m, e, _, _ in _CACHE.values():
        e.close()
    _CACHE.clear()
