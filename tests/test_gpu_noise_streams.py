"""GPU: the device's randomness against fp64 restatements at its edges: philox_normal one draw at a time (plant control
and sensor noise, at counters where fp32 Box-Muller is fragile and over about 1e6 ordinary draws) and its distribution;
the Ornstein-Uhlenbeck coefficients of the plants' control and force noise and of the rollouts' force noise at time
constants from dt / 100 to 1e6 s; and the state-ensemble members against mean (+) L64 z64 with numpy's Cholesky and
scipy's rotations, including rank-deficient covariances.

The words are restated by tests/plant_noise.py, which tests/test_noise_streams_cpu.py pins to the published
Philox4x32-10 known answers."""
import numpy as np
import pytest

import plant_noise as PN
from conftest import get_model, mocap_of
from test_gpu_plant import QUAD_SENSORS, _bank, _start

pytestmark = pytest.mark.gpu

WORST = {}   # group -> largest error / bar, printed by test_zz_report


def _record(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), float(ratio))


def _z_bar(z64):
    """|z_dev - z64| <= 2^-19 (1 + |z64|): u1's and u2's rounding to fp32 (2^-24 relative each; the top counters'
    log1p of the exact complement), __logf / log1pf / cospif / sqrtf to a few ulps, and a phase error of at most
    2 pi 2^-25 times the radius sqrt(-2 log u1) < 6 on the cosine"""
    return 2.0 ** -19 * (1.0 + np.abs(z64))


def _white_bank(m, seeds, sensors=(None, 0)):
    """plants whose control noise is white and unit: ctrl_rate << dt gives r = 0, s = 1, so that the applied ctrl of
    commanded ctrl 0 is exactly the device's z"""
    bank = _bank(m, len(seeds), sensors)
    q, v = _start(m, 1)[0]
    for b, s in enumerate(seeds):
        bank.reset(b, q, np.zeros_like(v), 0.0, mocap_of(m))
        bank.set_disturbance(b, ctrl_std=1.0, ctrl_rate=m.opt_timestep / 1e3, seed=int(s))
    return bank


# ------------------------------------------------------------------------------------------ 1. normals, one at a time
_SEARCH = {}


def _searched():
    if not _SEARCH:
        _SEARCH.update(PN.search_counters(PN.TAG_CTRL, 12, per_region=4))
    return _SEARCH


def test_device_normals_at_fragile_counters():
    m = get_model("quadruped")
    assert m.nu == 12
    found = _searched()
    cases = [(k, s, e) for k, v in found.items() for s, e in v]
    bank = _white_bank(m, [s for _, s, _ in cases])
    o = bank.step(np.zeros((len(cases), m.nu), np.float32))
    bank.close()
    bad = []
    for b, (region, s, e) in enumerate(cases):
        z64 = PN.box_muller(PN.philox_words([s], 0, e, PN.TAG_CTRL))[0]
        err = abs(float(o["ctrl"][b, e]) - z64)
        _record("normals at fragile counters", err / _z_bar(z64))
        if err > _z_bar(z64):
            bad.append((region, s, e, float(o["ctrl"][b, e]), z64, err))
    assert not bad, "device z off the fp64 Box-Muller: (region, seed, element, z_dev, z64, err) %s" % bad[:8]


_DRAWS = {}


def _ordinary():
    """[steps][plants][nu] device z and fp64 z of 4096 Quadruped plants over 20 steps (983k draws)"""
    if not _DRAWS:
        m = get_model("quadruped")
        B, steps = 4096, 20
        seeds = np.arange(B, dtype=np.uint64) * 7919 + 11
        bank = _white_bank(m, seeds)
        dev = np.zeros((steps, B, m.nu))
        for k in range(steps):
            o = bank.step(np.zeros((B, m.nu), np.float32))
            assert (o["status"] == 0).all()
            dev[k] = o["ctrl"]
        bank.close()
        ref = np.stack([np.stack([PN.box_muller(PN.philox_words(seeds, k, e, PN.TAG_CTRL)) for e in range(m.nu)], 1)
                        for k in range(steps)])
        _DRAWS.update(dev=dev, ref=ref, seeds=seeds)
    return _DRAWS


def test_device_normals_over_a_million_draws():
    d = _ordinary()
    r = np.abs(d["dev"] - d["ref"]) / _z_bar(d["ref"])
    _record("ordinary normals", r.max())
    assert r.max() <= 1.0, np.unravel_index(r.argmax(), r.shape)


def test_device_sensor_noise_one_draw_at_a_time():
    """sd = 1: the noisy reading minus the twin bank's noiseless reading is z, up to the rounding of y + z and of the
    subtraction (2^-24 |y + z| each)"""
    m = get_model("quadruped")
    B, steps = 512, 4
    seeds = np.arange(B, dtype=np.uint64) * 31 + 5
    noisy, clean = _white_bank(m, seeds, QUAD_SENSORS), _white_bank(m, seeds, QUAD_SENSORS)
    for b in range(B):
        noisy.set_sensor_noise(b, 1.0)
    worst = 0.0
    for k in range(steps):
        a = noisy.step(np.zeros((B, m.nu), np.float32))
        c = clean.step(np.zeros((B, m.nu), np.float32))
        dim = a["sensordata"].shape[1]
        z64 = np.stack([PN.box_muller(PN.philox_words(seeds, k, e, PN.TAG_SENS)) for e in range(dim)], 1)
        diff = a["sensordata"].astype(float) - c["sensordata"].astype(float)
        bar = _z_bar(z64) + 2.0 ** -23 * (np.abs(c["sensordata"]) + np.abs(z64))
        worst = max(worst, float((np.abs(diff - z64) / bar).max()))
    noisy.close(); clean.close()
    _record("sensor normals", worst)
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------ 2. distribution
def test_distribution_of_the_device_normals():
    from scipy import stats
    d = _ordinary()
    z = d["dev"]
    x = z.reshape(-1)
    n = x.size
    p = stats.kstest(x, "norm").pvalue
    assert p > 1e-4, p
    assert abs(x.mean()) < 5 / np.sqrt(n)
    assert abs(x.var() - 1) < 5 * np.sqrt(2 / n)
    for t in (3.0, 4.0):
        q = 2 * stats.norm.sf(t)
        c = int((np.abs(x) > t).sum())
        assert abs(c - n * q) < 5 * np.sqrt(n * q * (1 - q)) + 1, (t, c, n * q)
    for axis in range(3):   # lag-1 across step, plant, element
        a = np.moveaxis(z, axis, 0)
        rho = float((a[1:] * a[:-1]).mean())
        cnt = a[1:].size
        assert abs(rho) < 5 / np.sqrt(cnt), (axis, rho)
    # the tags of one counter draw different words
    seeds = d["seeds"][:64]
    w = [PN.philox_words(seeds, 3, 5, t) for t in (PN.TAG_CTRL, PN.TAG_XFRC, PN.TAG_SENS)]
    assert not (w[0] == w[1]).all(1).any() and not (w[0] == w[2]).all(1).any() and not (w[1] == w[2]).all(1).any()


# ------------------------------------------------------------------------------------------ 3. OU coefficients
RATE_FACTORS = ("dt/100", "dt", 0.05, 2.0, 1e2, 1e4, 1e6)


def _rate(m, f):
    return {"dt/100": m.opt_timestep / 100, "dt": m.opt_timestep}.get(f, f)


def _truth(dt, std, rate):
    """r and s in fp64 from the fp32 values the device holds"""
    dt, std, rate = (float(np.float32(v)) for v in (dt, std, rate))
    return np.exp(-dt / rate), std * np.sqrt(-np.expm1(-2 * dt / rate))


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
def test_plant_ou_coefficients_at_their_edges(name):
    """s from the first committed step (n1 = s z1, z1 the twin's with r = 0, s = 1), r from the second on elements with
    |z1| > 2 and |z2| < 0.5.  Bars: s within 8 fp32 ulps relative; r within 2 ulps of max(r, 1/2) (r = 1 + expm1f(x)
    is accurate in absolute terms, which is what r n is, and expm1f(x) ~ -1 below r = 1/2) plus the recovery's
    rounding, 2^-23 (r + |z2| / |z1|); r <= 1 up to that recovery rounding."""
    m = get_model(name)
    per, stds = 48, (0.7, 3.0)                  # plants per rate; ctrl std, xfrc std
    seeds = np.arange(per, dtype=np.uint64) * 101 + 3
    B = per * len(RATE_FACTORS)
    q, v = _start(m, 1)[0]
    noisy, twin = _bank(m, B), _bank(m, B)
    for i, f in enumerate(RATE_FACTORS):
        for j in range(per):
            b = i * per + j
            for bk in (noisy, twin):
                bk.reset(b, q, v, 0.0, _mocap(m))
            noisy.set_disturbance(b, stds[0], _rate(m, f), stds[1], _rate(m, f), int(seeds[j]))
            twin.set_disturbance(b, 1.0, m.opt_timestep / 1e3, 1.0, m.opt_timestep / 1e3, int(seeds[j]))
    n, z = [], []
    U = np.zeros((B, m.nu), np.float32)
    for k in range(2):
        a, c = noisy.step(U), twin.step(U)
        assert (a["status"] == 0).all() and (c["status"] == 0).all()
        n.append([np.concatenate([noisy.disturbance(b)["ctrl_noise"], noisy.disturbance(b)["xfrc_noise"].reshape(-1)])
                  for b in range(B)])
        z.append([np.concatenate([twin.disturbance(b)["ctrl_noise"], twin.disturbance(b)["xfrc_noise"].reshape(-1)])
                  for b in range(B)])
    noisy.close(); twin.close()
    n1, n2, z1, z2 = (np.asarray(a, float) for a in (n[0], n[1], z[0], z[1]))
    nu = m.nu
    bad = []
    for i, f in enumerate(RATE_FACTORS):
        rows = slice(i * per, (i + 1) * per)
        for kind, cols, std in (("ctrl", slice(0, nu), stds[0]), ("xfrc", slice(nu, None), stds[1])):
            r64, s64 = _truth(m.opt_timestep, std, _rate(m, f))
            a1, a2, y1, y2 = n1[rows, cols], n2[rows, cols], z1[rows, cols], z2[rows, cols]
            s_dev = a1 / y1
            es = float(np.abs(s_dev / s64 - 1).max()) / (8 * 2.0 ** -24)
            pick = (np.abs(y1) > 2) & (np.abs(y2) < 0.5)
            r_dev = (a2[pick] - s_dev[pick] * y2[pick]) / a1[pick]
            r_bar = 2 * 2.0 ** -24 * max(r64, 0.5) + 2.0 ** -23 * (r64 + np.abs(y2[pick] / y1[pick]))
            er = float((np.abs(r_dev - r64) / r_bar).max()) if pick.any() else 0.0
            _record("plant OU s", es); _record("plant OU r", er)
            print("%s %s rate %s: s err %.2f of bar, r err %.2f of bar over %d elements, r64 %.9f" % (
                name, kind, f, es, er, int(pick.sum()), r64))
            if es > 1 or er > 1 or not pick.any() or (r_dev > 1 + r_bar - 2 * 2.0 ** -24 * max(r64, 0.5)).any():
                bad.append((kind, f, es, er, int(pick.sum())))
    assert not bad, bad


def _mocap(m):
    from test_gpu_plant import _mocap as mc
    return mc(m)


@pytest.mark.parametrize("factor", RATE_FACTORS)
def test_rollout_force_noise_at_its_edges(factor):
    """On the particle (two slide joints on one body, unit-gear motors) a force on the body is exactly a control: a
    noisy rollout must equal a clean rollout driven by the fp64 OU forces (test_gpu_parity's construction).  The std
    is chosen per rate so that s = 0.05 N: at 1e6 s, 1 - r^2 cancels in fp32 and the previous formula added no force."""
    from mujoco_mpc_b200.engine import Engine
    from mujoco_mpc_b200.planner import philox4x32
    m = get_model("particle")
    H, seed = 12, 4321
    rate = _rate(m, factor)
    _, s_unit = _truth(m.opt_timestep, 1.0, rate)
    std = 0.05 / s_unit
    r64, s64 = _truth(m.opt_timestep, std, rate)
    body = int(m.jnt_bodyid[0])
    state = np.array([0.05, -0.02, 0.1, 0.0])
    kt = np.arange(H) * m.opt_timestep - 1e-6
    e = Engine(m, 8, H)
    e.set_xfrc_noise(std, rate, seed)
    try:
        e.rollout_spline(state, 0.0, mocap_of(m), np.zeros((2, H, m.nu)), kt, 0, H)
        noisy = e.fetch_trajectory(1)
    finally:
        e.set_xfrc_noise(0.0)
    x = np.zeros(6 * m.nbody); forces = np.zeros((H, 2))
    for t in range(H - 1):
        ctr = np.array([[t, 1, el, PN.TAG_XFRC] for el in range(6 * m.nbody)], np.uint32)
        x = r64 * x + s64 * PN.box_muller(philox4x32(ctr, (seed, 1)))
        forces[t] = x[6 * body: 6 * body + 2]
    assert np.abs(forces).max() < 1   # inside ctrlrange: the control is not clamped
    e.rollout_spline(state, 0.0, mocap_of(m), forces[None], kt, 0, H)
    clean = e.fetch_trajectory(0)
    e.close()
    err = np.abs(noisy["states"] - clean["states"]).max()
    moved = np.abs(clean["states"] - _free_states(m, state, H, kt)).max()
    _record("rollout OU states", err / 2e-6)
    print("rate %s: |noisy - force-as-control| %.2e, displacement by the noise %.2e" % (factor, err, moved))
    assert moved > 1e-4
    assert err <= 2e-6


def _free_states(m, state, H, kt):
    """the particle's states with no force at all"""
    from mujoco_mpc_b200.engine import Engine
    e = Engine(m, 8, H)
    e.rollout_spline(state, 0.0, mocap_of(m), np.zeros((1, H, m.nu)), kt, 0, H)
    out = e.fetch_trajectory(0)["states"]
    e.close()
    return out


# ------------------------------------------------------------------------------------------ 4. state-ensemble draws
def _restated(m, mean, L, seed, iteration, b, k):
    """mean (+) L z64 in fp64: free and ball quaternions through scipy's Rotation (q times exp(w / 2), normalised, as
    mju_quatIntegrate: a rotation below mjMINVAL = 1e-15 only normalises q, and one of exactly zero keeps q's bits)"""
    from scipy.spatial.transform import Rotation
    n = 2 * m.nv
    ctr = np.array([[iteration, k, e, 0x42454C46] for e in range(n)], np.uint32)
    from mujoco_mpc_b200.planner import philox4x32
    dx = L @ PN.box_muller(philox4x32(ctr, ((seed + b) & 0xFFFFFFFF, 3)))
    out = np.array(mean, float)
    for j in range(m.njnt):
        t, qa, da = int(m.jnt_type[j]), int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        if t == 0:
            out[qa:qa + 3] += dx[da:da + 3]
        if t in (0, 1):
            a = qa + (3 if t == 0 else 0)
            w = dx[da + (3 if t == 0 else 0): da + (3 if t == 0 else 0) + 3]
            q = out[a:a + 4]
            if np.any(w != 0) and np.linalg.norm(w) < 1e-15:   # below mjMINVAL: normalised, not rotated
                out[a:a + 4] = q / np.linalg.norm(q)
            elif np.any(w != 0):
                r = Rotation.from_quat([q[1], q[2], q[3], q[0]], scalar_first=False) * Rotation.from_rotvec(w)
                x, y, zz, s = r.as_quat(canonical=False)
                out[a:a + 4] = np.array([s, x, y, zz]) / np.linalg.norm([s, x, y, zz])
        elif t >= 2:
            out[qa] += dx[da]
    out[m.nq:] += dx[m.nv:]
    return out, dx


def _covariances(m, kind, B):
    n = 2 * m.nv
    rng = np.random.default_rng(17)
    out = []
    for b in range(B):
        if kind == "diagonal":
            P = np.diag(10.0 ** rng.uniform(-5, -2, n))
        elif kind == "correlated":
            A = rng.standard_normal((n, n))
            P = 1e-3 * (A @ A.T / n + 0.1 * np.eye(n))
        elif kind == "cond1e10":
            Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
            P = 1e-2 * (Q * np.logspace(0, -10, n)) @ Q.T
        else:   # orientation: rotation variances giving |w| from 1e-16 to past 3 pi
            sig = (1e-16, 1e-8, np.pi, 3 * np.pi)[b % 4] / np.sqrt(3)
            P = np.diag(np.full(n, 1e-4))
            for j in range(m.njnt):
                if m.jnt_type[j] in (0, 1):
                    d = int(m.jnt_dofadr[j]) + (3 if m.jnt_type[j] == 0 else 0)
                    P[d:d + 3, d:d + 3] = sig ** 2 * np.eye(3)
        out.append(0.5 * (P + P.T))
    return np.stack(out)


def _launch(m, covs, K=8, seed=9, iteration=3):
    from test_gpu_batched import _problems
    from test_gpu_model_variants import _engine
    from test_gpu_state_ensemble import _belief, _member_states
    B, N, H = len(covs), 2, 4
    pr = _problems(m, N, H, B=B)
    e = _engine(m, B * K * N, H)
    try:
        _belief(e, pr, covs, H, K, 1, seed=seed, iteration=iteration)
        dev = _member_states(e, B, K, N)
    finally:
        e.close()
    return pr, dev


def _ulps(a, b):
    from test_gpu_state_ensemble import _ulps as u
    return u(a, b)


@pytest.mark.parametrize("name", ["quadruped", "humanoid_track"])
@pytest.mark.parametrize("kind", ["diagonal", "correlated", "cond1e10", "orientation"])
def test_state_members_against_the_fp64_restatement(name, kind):
    """member k of problem b is mean (+) L64 z64 rounded to float, to 2 ulps per entry (a quaternion's sign is the
    rotation's, so the restatement takes the device's hemisphere)"""
    m = get_model(name)
    B, K = 4, 8
    covs = _covariances(m, kind, B)
    pr, dev = _launch(m, covs, K)
    worst = 0
    for b in range(B):
        mean = np.asarray(pr["states"][b], np.float32).astype(float)
        L = np.linalg.cholesky(covs[b])
        for k in range(1, K):
            ref, _ = _restated(m, mean, L, 9, 3, b, k)
            for j in range(m.njnt):
                if m.jnt_type[j] in (0, 1):
                    a = int(m.jnt_qposadr[j]) + (3 if m.jnt_type[j] == 0 else 0)
                    if np.dot(ref[a:a + 4], dev[b, k, a:a + 4]) < 0:
                        ref[a:a + 4] *= -1
            u = _ulps(dev[b, k], ref.astype(np.float32))
            # a quaternion component is a coordinate of a unit vector: both fp64 computations of it are good to a
            # few fp64 ulps of 1, which exceeds the float ulp of a component within ~1e-8 of zero
            near = np.abs(dev[b, k].astype(float) - ref) <= 16 * 2.0 ** -53
            u = np.where(near, 0, u)
            if u.max() > 2:
                i = int(u.argmax())
                print("problem %d member %d entry %d: device %r restated %r" % (b, k, i, float(dev[b, k, i]), ref[i]))
            worst = max(worst, int(u.max()))
    _record("state members (ulp / 2)", worst / 2)
    print("%s %s: largest distance of a member state from the restatement: %d ulp" % (name, kind, worst))
    assert worst <= 2


@pytest.mark.parametrize("deficiency", [1, 3])
@pytest.mark.parametrize("scale", [1e-6, 1e-2, 1e2])
def test_rank_deficient_members_agree_with_the_host_and_lie_in_range(deficiency, scale):
    """The device and the host twin accept the J J^T of tests/test_noise_streams_cpu.py, and the device's draws lie in
    range(J) up to the float rounding of the member states (the projection outside range(J) of a rounding vector is
    at most its norm).  A pivot that lands within the device's fused multiply-add rounding of -tau can be accepted on
    one side and refused on the other; these cases are not at that edge."""
    from mujoco_mpc_b200 import estimator
    from mujoco_mpc_b200.engine import EngineError, host_state_member
    m = get_model("quadruped")
    n = 2 * m.nv
    B, K = 2, 8
    from test_noise_streams_cpu import _deficient
    covs, Qs = zip(*(_deficient(n, n - deficiency, scale, b, m) for b in range(B)))
    covs = np.stack(covs)
    host_ok = []
    from test_gpu_batched import _problems
    pr = _problems(m, 2, 4, B=B)
    for b in range(B):
        try:
            host_state_member(m, np.asarray(pr["states"][b], np.float32).astype(float), covs[b], 9, 3, b, 1)
            host_ok.append(True)
        except EngineError:
            host_ok.append(False)
    try:
        _, dev = _launch(m, covs, K)
        dev_ok = True
    except EngineError:
        dev_ok = False
    assert dev_ok == all(host_ok), (dev_ok, host_ok)
    assert dev_ok
    worst = 0.0
    for b in range(B):
        mean = np.asarray(pr["states"][b], np.float32).astype(float)
        for k in range(1, K):
            x = dev[b, k].astype(float)
            dx = np.concatenate([estimator.differentiate_pos(m, mean[:m.nq], x[:m.nq]), x[m.nq:] - mean[m.nq:]])
            out = np.linalg.norm(dx - Qs[b] @ (Qs[b].T @ dx))
            bar = 4 * np.linalg.norm(np.spacing(np.abs(x).astype(np.float32)).astype(float))
            worst = max(worst, out / bar)
    _record("rank-deficient members outside range(J)", worst)
    assert worst <= 1.0


def test_zz_report():
    for k, v in sorted(WORST.items()):
        print("worst error / bar: %-45s %.3g" % (k, v))
