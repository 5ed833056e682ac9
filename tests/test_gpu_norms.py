"""GPU: the device norms (norm_value in csrc/dev_task.cuh, norm_full in csrc/ilqg_kernels.cuh), the risk transform and
the cost-derivative kernel against the fp64 oracle (oracle/task.h, itself pinned to norm_test.cc), at every norm type
and at the inputs where fp32 fast-math code goes wrong: exact zeros (zero exponents of __powf), softplus overflow,
cosh near the top of fp32's range, risk cancellation, more than 32 terms and terms wider than 32.

Models: deep copies of the humanoid (46 residuals: Height 1, Balance 1, CoM Vel 2, Joint Vel 21, Control 21) with the
task's norm specification rewritten; each variant gets its own Engine and fp64 Oracle.

Bars.  Inputs are rounded to fp32 before both calls, so what remains is device arithmetic:
  - sums and products: every output entry is a sum of products over at most 46 residual entries and 46 terms, so its
    round-off is bounded by ~2 * 46 * 2^-24 < 32 * 2^-22 relative to the sum of the |products| (M below);
  - fast-math transcendentals: __powf(a, b) = ex2(b * lg2(a)) and __expf(z) = ex2(z * log2 e) carry a relative error
    of about |b log2 a| * 2^-22 (resp. |z| * 2^-22), the error of the product in the exponent; Z is the largest such
    exponent over the entries of the row, and the per-entry bar is (32 + 2 Z) * 2^-22 * M;
  - risk R: the derivatives are scaled by s = exp(R c) (c = sum of w y / H, Cmag its summed magnitudes), whose relative error adds
    |R| Cmag times the bar, and |R c| 2^-22 for the exponential itself; the value transform expm1(R c) / R has slope
    e^(R c), so the value bar is (32 + 2 Z) * 2^-22 * e^(R c) * V + 4 * 2^-22 * |value| (V: the summed magnitudes);
  - an absolute floor of 1e-30: products of the +-1e-30 residual entries underflow fp32 (x^2 = 1e-60) and lose
    contributions below that size.
M is computed in fp64 from the oracle's own norm gradients and Hessians with every factor replaced by its magnitude,
and every difference in a norm's formula by the sum of its operands' magnitudes (sqrt(x^2 + p^2) - p, cosh(z) - 1,
1 - g^2, ...): fp32 evaluates such a difference to a few ulps of its operands, not of the result.

Points excluded (the fp64 reference is not a finite fp32 number there):
  - the PowerLoss Hessian at an exact zero with p < 2 (0^(p-2) is infinite; p = 1 gives 0 * inf): cxx, cxu and cuu
    of those rows are non-finite in fp64 and dropped; L22 and SmoothAbs2 with q < 2 are not exercised;
  - rows with |R c| > 80 at risk R != 0: e^(R c) leaves fp32's range (cosh at |x/p| = 80 makes c ~ 1e33).
Everywhere else a device NaN or inf where fp64 is finite is a failure.
"""
import copy

import numpy as np
import pytest

from conftest import get_model, mocap_of

pytestmark = pytest.mark.gpu

NULL, QUAD, L22, L2, COSH, POWER, SABS, SABS2, RECT = -1, 0, 1, 2, 3, 5, 6, 7, 8
TYPE_NAME = {NULL: "Null", QUAD: "Quadratic", L22: "L22", L2: "L2", COSH: "Cosh", POWER: "PowerLoss",
             SABS: "SmoothAbs", SABS2: "SmoothAbs2", RECT: "Rectify"}
HUMANOID_DIMS = [1, 1, 2, 21, 21]
U22 = 2.0 ** -22
H = 8


def _uniform(ntype, params):
    w = [1.0, 0.5, 2.0, 0.3, 0.7]
    return [(d, ntype, list(params), w[i]) for i, d in enumerate(HUMANOID_DIMS)]


def _mixed46():
    cyc = [(QUAD, []), (L22, [0.1, 2]), (L2, [0.01]), (COSH, [0.3]), (POWER, [1]), (POWER, [1.5]), (POWER, [2]),
           (SABS, [0.1]), (SABS2, [0.1, 2]), (SABS2, [0.2, 4]), (RECT, [0.01]), (RECT, [1]), (NULL, []),
           (L22, [0.3, 4]), (POWER, [3]), (COSH, [1])]
    return [(1, t, p, 0.2 + 0.1 * (i % 7)) for i, (t, p) in enumerate(cyc[i % len(cyc)] for i in range(46))]


VARIANTS = {
    "quadratic": _uniform(QUAD, []),
    "l22_q2": _uniform(L22, [0.1, 2]),
    "l22_q4": _uniform(L22, [0.3, 4]),
    "l2_p0.01": _uniform(L2, [0.01]),
    "l2_p0.1": _uniform(L2, [0.1]),
    "cosh_p0.3": _uniform(COSH, [0.3]),
    "cosh_p1": _uniform(COSH, [1]),
    "power_p1": _uniform(POWER, [1]),
    "power_p1.5": _uniform(POWER, [1.5]),
    "power_p2": _uniform(POWER, [2]),
    "power_p3": _uniform(POWER, [3]),
    "smoothabs_p0.01": _uniform(SABS, [0.01]),
    "smoothabs_p0.1": _uniform(SABS, [0.1]),
    "smoothabs2_q2": _uniform(SABS2, [0.1, 2]),
    "smoothabs2_q4": _uniform(SABS2, [0.2, 4]),
    "rectify_p0.01": _uniform(RECT, [0.01]),
    "rectify_p1": _uniform(RECT, [1]),
    "null_46x1": [(1, NULL, [], 0.5 + 0.01 * i) for i in range(46)],
    "mixed_46x1": _mixed46(),
    # terms wider than 32 residuals: the cost-derivative kernel's per-term scratch is sized from the widest term
    "wide_1_1_2_42": [(1, SABS, [0.1], 1.0), (1, RECT, [0.01], 0.5), (2, L22, [0.1, 2], 2.0), (42, L22, [0.3, 4], 0.3)],
    "wide_46": [(46, L22, [0.3, 4], 0.7)],
}


def variant_model(terms):
    """deep copy of the humanoid with its cost terms replaced by `terms` = [(dim, norm, params, weight)]"""
    base = get_model("humanoid")
    m = type(base)(copy.deepcopy(dict(base)))
    assert sum(d for d, _, _, _ in terms) == m.task_num_residual == 46
    m.task_num_term = len(terms)
    m.task_dim_norm_residual = np.array([d for d, _, _, _ in terms], np.int32)
    m.task_norm = np.array([t for _, t, _, _ in terms], np.int32)
    m.task_weight = np.array([w for _, _, _, w in terms], float)
    m.task_num_norm_parameter = np.array([len(p) for _, _, p, _ in terms], np.int32)
    m.task_norm_parameter = np.array([x for _, _, p, _ in terms for x in p], float)
    m.task_weight_names = ["term %d" % i for i in range(len(terms))]
    return m


_CTX = {}


@pytest.fixture(scope="module")
def variants(oracle_lib):
    from mujoco_mpc_b200 import build
    build.build()
    yield _CTX
    for _, e, _ in _CTX.values():
        e.close()
    _CTX.clear()


def _get(variants, oracle_lib, name):
    if name not in variants:
        from mujoco_mpc_b200.blob import to_blob
        from mujoco_mpc_b200.engine import Engine
        m = variant_model(VARIANTS[name])
        variants[name] = (m, Engine(m, 16, H), oracle_lib.Oracle(to_blob(m), m, 64))
    return variants[name]


def _entry_specs(terms):
    """per residual entry: (norm type, params) of its term"""
    out = []
    for d, t, p, _ in terms:
        out += [(t, p)] * d
    return out


def _rows(terms, seed=0):
    """hand-chosen residual rows [H, 46]: exact zeros, +-1e-30, +-1e-3, +-1, random, large (Cosh |x/p| up to 80,
    Rectify x/p = +-100), an all-zero block next to random values, and a mix of zeros and small values"""
    rng = np.random.default_rng(seed)
    spec = _entry_specs(terms)
    alt = np.where(np.arange(46) % 2 == 0, 1.0, -1.0)
    large = np.empty(46)
    for j, (t, p) in enumerate(spec):
        if t == COSH:
            large[j] = alt[j] * 80 * p[0] * (1.0 if j % 3 == 0 else 0.6)
        elif t == RECT:
            large[j] = alt[j] * 100 * p[0]
        else:
            large[j] = alt[j] * 3.0
    half = rng.normal(0, 0.5, 46)
    half[:23] = 0
    mix = np.where(np.arange(46) % 3 == 0, 0.0, np.where(np.arange(46) % 3 == 1, 1e-3 * alt, 0.3 * alt))
    R = np.stack([np.zeros(46), 1e-30 * alt, 1e-3 * alt, alt, rng.normal(0, 0.5, 46), large, half, mix])
    return R.astype(np.float32).astype(np.float64)


def _exponent_mag(x, t, p):
    """largest |b log2 a| of the __powf calls (|z| of the exponentials) that evaluate norm t on the entries x"""
    p0 = p[0] if p else 0.0
    q = p[1] if len(p) > 1 else 0.0
    ax = np.abs(x)
    lg = np.log2(ax, out=np.zeros_like(ax), where=ax > 0)
    if t in (COSH, RECT):
        return float(np.max(np.abs(x / p0)))
    if t == POWER:
        return float(np.max(max(abs(p0), abs(p0 - 1), abs(p0 - 2)) * np.abs(lg)))
    if t == SABS2:
        e = ax ** q + p0 ** q
        return float(np.max(max(q, abs(q - 2)) * np.abs(lg) + np.abs(np.log2(e)) / q))
    if t == L22:
        cc = float(np.sum(x * x))
        z = max(q / 2, abs(q / 2 - 1)) * abs(np.log2(cc)) if cc > 0 else 0.0
        return z + abs(np.log2(cc ** (q / 2) + p0 ** q)) / q
    return 0.0


def _summand_mag(x, t, p, y, g, Hh):
    """fp64 magnitudes of the summands the norm's formulas add or subtract (value, gradient, Hessian): fp32 evaluation
    of e.g. sqrt(x^2 + p^2) - p or cosh(z) - 1 is exact only to a few ulps of its operands, not of the difference"""
    p0 = p[0] if p else 0.0
    q = p[1] if len(p) > 1 else 0.0
    n = len(x)
    V, G, Hm = abs(y), np.abs(g), np.abs(Hh)
    if t in (L2, L22):
        cc = float(np.sum(x * x))
        s = np.sqrt(cc + p0 * p0) if t == L2 else (cc ** (q / 2) + p0 ** q) ** (1 / q)
        V = s + p0
        if t == L2 and s > 0:
            Hm = (np.eye(n) + np.abs(np.outer(g, g))) / s
        elif t == L22:
            a = cc ** (q / 2) + p0 ** q
            b = s / a * (cc ** (q / 2 - 1) if q != 2 else 1.0) if cc > 0 or q >= 2 else 0.0
            c2 = abs((1 - q) * (cc ** (q / 2 - 1) if cc > 0 else float(q == 2)) / a) + abs(q - 2) / max(cc, 1e-15)
            Hm = abs(b) * (np.eye(n) + np.abs(np.outer(x, x)) * c2)
    elif t in (SABS, SABS2):
        if t == SABS:
            s = np.sqrt(x * x + p0 * p0)
            Hm = np.diag(np.where(s > 0, (1 + g * g) / np.where(s > 0, s, 1), 0.0))
        else:
            a = np.abs(x)
            e = a ** q + p0 ** q
            s = e ** (1 / q)
            c2 = s * (a ** (q - 2) if q != 2 else 1.0) / e
            Hm = np.diag(np.abs(c2 * (q - 1)) * (1 + a ** q / e))
        V = float(np.sum(s + p0))
    elif t == COSH:
        V = float(np.sum(p0 * p0 * (np.cosh(x / p0) + 1)))
    return V, G, Hm


def _magnitudes(pyoracle, terms, res, C, D, risk):
    """fp64 magnitude sums M (every factor by its absolute value) for cx, cu, cxx, cuu, cxu, the per-row exponent
    bound Z, the row cost c and Cmag = sum |w y| / H"""
    Hn_, n, m = C.shape[0], C.shape[2], D.shape[2]
    Mx, Mu = np.zeros((Hn_, n)), np.zeros((Hn_, m))
    Mxx, Muu, Mxu = np.zeros((Hn_, n, n)), np.zeros((Hn_, m, m)), np.zeros((Hn_, n, m))
    Z, c, Cmag = np.zeros(Hn_), np.zeros(Hn_), np.zeros(Hn_)
    for t in range(Hn_):
        f = 0
        for d, ty, p, w in terms:
            x = res[t, f:f + d]
            y, g, Hh = pyoracle.norm(x, np.array(p, float) if p else None, ty, grad=True, hess=True)
            if ty == NULL:
                g[1:] = 0
            with np.errstate(all="ignore"):
                V, g, Hh = _summand_mag(x, ty, p, y, g, Hh)
            rx, ru = np.abs(C[t, f:f + d]), np.abs(D[t, f:f + d])
            ww = w / Hn_
            with np.errstate(all="ignore"):
                Mx[t] += ww * rx.T @ np.abs(g)
                Mu[t] += ww * ru.T @ np.abs(g)
                Mxx[t] += ww * rx.T @ np.abs(Hh) @ rx
                Muu[t] += ww * ru.T @ np.abs(Hh) @ ru
                Mxu[t] += ww * rx.T @ np.abs(Hh) @ ru
            c[t] += ww * y
            Cmag[t] += ww * V
            Z[t] = max(Z[t], _exponent_mag(x, ty, p))
            f += d
    if abs(risk) >= 1e-6:
        s = np.exp(risk * c)
        Mx, Mu = Mx * s[:, None], Mu * s[:, None]
        Mxx = Mxx * s[:, None, None] + abs(risk) * s[:, None, None] * Mx[:, :, None] * Mx[:, None, :]
        Muu = Muu * s[:, None, None] + abs(risk) * s[:, None, None] * Mu[:, :, None] * Mu[:, None, :]
        Mxu = Mxu * s[:, None, None] + abs(risk) * s[:, None, None] * Mx[:, :, None] * Mu[:, None, :]
    return (Mx, Mu, Mxx, Muu, Mxu), Z, c, Cmag


@pytest.mark.parametrize("risk", [0.0, 1.0, -0.5])
@pytest.mark.parametrize("name", list(VARIANTS))
def test_cost_derivatives_vs_fp64(variants, oracle_lib, name, risk):
    """Engine.cost_derivatives (norm_full + the Gauss-Newton products + the risk scaling) vs oracle.cost_derivatives
    on the same fp32-rounded residual rows and seeded random C, D."""
    m, e, o = _get(variants, oracle_lib, name)
    terms = VARIANTS[name]
    res = _rows(terms)
    rng = np.random.default_rng(1)
    C = rng.normal(0, 0.5, (H, 46, 2 * m.nv)).astype(np.float32).astype(np.float64)
    D = rng.normal(0, 0.5, (H, 46, m.nu)).astype(np.float32).astype(np.float64)
    e.set_task(risk=risk)
    o.set_task(risk=risk)
    try:
        dev = e.cost_derivatives(res, C, D)
        with np.errstate(all="ignore"):
            ref = o.cost_derivatives(res, C, D)
    finally:
        e.set_task(risk=0.0)
        o.set_task(risk=0.0)
    Ms, Z, c, Cmag = _magnitudes(oracle_lib, terms, res, C, D, risk)
    keep_row = np.abs(risk * c) <= 80 if risk != 0 else np.ones(H, bool)
    assert keep_row.sum() >= 4, (name, risk, c)
    spec = _entry_specs(terms)
    sing = np.array([t == POWER and p[0] < 2 for t, p in spec])
    sing_rows = ((res == 0) & sing[None, :]).any(1)
    worst = {}
    for k, (G, R, M) in enumerate(zip(dev, ref, Ms)):
        nm = ("cx", "cu", "cxx", "cuu", "cxu")[k]
        shape = (H,) + (1,) * (R.ndim - 1)
        finite_ref = np.isfinite(R) & (np.abs(R) < 3.4e38) & keep_row.reshape(shape)
        if sing_rows.any() and nm in ("cxx", "cuu", "cxu"):
            # the only reference singularity exercised: 0^(p-2) with p < 2 at the exact-zero rows
            assert not np.isfinite(R[sing_rows]).all()
            finite_ref &= ~sing_rows.reshape(shape)
        assert np.isfinite(R[keep_row & ~sing_rows]).all(), (name, nm)
        bad = finite_ref & ~np.isfinite(G)
        assert not bad.any(), "%s risk %g %s: device non-finite where fp64 is finite at rows %s" % (
            name, risk, nm, sorted(set(np.nonzero(bad)[0].tolist())))
        tol = (32 + 2 * Z) * U22 * (1 + abs(risk) * Cmag) + 2 * U22 * np.abs(risk * c)
        bar = tol.reshape(shape) * M + 1e-30
        err = np.where(finite_ref, np.abs(G.astype(np.float64) - R), 0.0)
        ratio = np.where(finite_ref & (tol.reshape(shape) * M > 1e-30), err / np.where(M > 0, M, 1.0), 0.0)
        worst[nm] = float(ratio.max())
        over = finite_ref & (err > bar)
        assert not over.any(), "%s risk %g %s: |dev - fp64| above the bar at rows %s (max %.3e vs bar %.3e)" % (
            name, risk, nm, sorted(set(np.nonzero(over)[0].tolist())), err[over].max(), bar[over].min())
    print("norms %-16s risk %4g: max |dev - fp64| / M: %s  (Z max %.1f)" % (
        name, risk, " ".join("%s %.2e" % kv for kv in worst.items()), Z.max()))


def _value_inputs(m, terms):
    """step_batch inputs that set the Control residual (ctrl) and Joint Vel residual (qvel[6:]) to exact zeros, +-1
    (the ctrl bounds), +-1e-3, the Rectify / Cosh large-argument values and random values"""
    spec = _entry_specs(terms)
    alt = np.where(np.arange(21) % 2 == 0, 1.0, -1.0)

    def large(off):
        out = np.empty(21)
        for j in range(21):
            t, p = spec[off + j]
            out[j] = alt[j] * (80 * p[0] if t == COSH else 100 * p[0] if t == RECT else 3.0)
        return out

    rng = np.random.default_rng(2)
    cr = np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    bounds = np.where(np.arange(21) % 2 == 0, cr[:, 1], cr[:, 0])
    pats = [(np.zeros(21), np.zeros(21)), (alt, bounds), (1e-3 * alt, -1e-3 * alt), (large(4), large(25)),
            (rng.normal(0, 0.5, 21), rng.normal(0, 0.5, 21)), (np.zeros(21), bounds)]
    B = len(pats)
    qpos = np.tile(m.qpos0, (B, 1))
    qvel = np.zeros((B, m.nv))
    ctrl = np.zeros((B, m.nu))
    for b, (jv, u) in enumerate(pats):
        qvel[b, 6:] = jv
        ctrl[b] = u
    return qpos, qvel, ctrl


@pytest.mark.parametrize("risk", [0.0, 1.0, 1e-3])
@pytest.mark.parametrize("name", list(VARIANTS))
def test_cost_value_vs_fp64(variants, oracle_lib, name, risk):
    """the device per-step cost (norm_value + k_cost_value through Engine.step_batch) vs oracle.cost_value of the
    device's own residual in fp64, so that only the norm and risk code is compared, not the physics; each state is
    evaluated at the variant's weights (far from zero cost) and at 1e-4 times them (near zero cost, where the risk
    transform cancels)."""
    m, e, o = _get(variants, oracle_lib, name)
    terms = VARIANTS[name]
    qpos, qvel, ctrl = _value_inputs(m, terms)
    B = qpos.shape[0]
    worst = 0.0
    for scale in (1.0, 1e-4):
        w = m.task_weight * scale
        e.set_task(weight=w, risk=risk)
        o.set_task(weight=w, risk=risk)
        try:
            out = e.step_batch(qpos, qvel, ctrl, mocap_of(m), np.zeros(B))
            res = out["residual"].astype(np.float64)
            for b in range(B):
                with np.errstate(all="ignore"):
                    ref, tv = o.cost_value(res[b], terms=True)
                    c = float(tv.sum())
                    wsum, f = 0.0, 0
                    for d, ty, p, wk in terms:
                        x = res[b, f:f + d]
                        y, g, Hh = oracle_lib.norm(x, np.array(p, float) if p else None, ty, grad=True, hess=True)
                        wsum += abs(wk * scale) * _summand_mag(x, ty, p, y, g, Hh)[0]
                        f += d
                if risk != 0 and abs(risk * c) > 80:
                    continue
                assert np.isfinite(ref)
                Z = 0.0
                f = 0
                for d, ty, p, _ in terms:
                    Z = max(Z, _exponent_mag(res[b, f:f + d], ty, p))
                    f += d
                dev = float(out["cost"][b])
                assert np.isfinite(dev), "%s risk %g scale %g state %d: device cost %r, fp64 %r" % (name, risk, scale, b, dev, ref)
                growth = np.exp(max(risk * c, 0.0)) if risk != 0 else 1.0
                bar = (32 + 2 * Z) * U22 * growth * wsum + 4 * U22 * abs(ref) + 1e-30
                err = abs(dev - ref)
                worst = max(worst, err / max(growth * wsum, 1e-300))
                assert err <= bar, "%s risk %g scale %g state %d: device %.9g fp64 %.9g (|err| %.3e > bar %.3e)" % (
                    name, risk, scale, b, dev, ref, err, bar)
        finally:
            e.set_task(weight=m.task_weight, risk=0.0)
            o.set_task(weight=m.task_weight, risk=0.0)
    print("cost value %-16s risk %6g: max |dev - fp64| / (e^(Rc) sum|w y|) = %.2e" % (name, risk, worst))

