"""GPU: measurement noise on the closed-loop plants (mjpc_b200_plant_set_sensor_noise, CppPlantBank.set_sensor_noise).

A zero std must leave every output bitwise as a plant without the call; noise must change only the returned sensordata
(state, cost, warm start and status bitwise unchanged); the noise of a noisy plant against its clean twin in the same
bank must have mean about 0 and std about std[e], match the numpy restatement of its draw, replay after reset and not
depend on the plant's index.  Refusals leave the plant unchanged."""
import ctypes as C

import numpy as np
import pytest

from conftest import get_model
from test_gpu_model_variants import _variants
from test_gpu_plant import QUAD_SENSORS, _bank, _ctrl, _eq, _mocap, _run, _start

pytestmark = pytest.mark.gpu

BAD_ARGUMENT, UNSUPPORTED = -1, -5
TAG_SENS = 0x53454E53   # 'SENS'


def _std(bank, seed=0):
    """a std per sensordata element, spread over two decades"""
    return (10.0 ** np.random.default_rng(seed).uniform(-3, -1, bank.nsensordata)).astype(np.float32)


@pytest.mark.parametrize("case", ["quadruped", "quadruped-generic"])
def test_zero_std_is_bitwise_a_plant_without_the_call(case, monkeypatch):
    if case.endswith("generic"):
        monkeypatch.setenv("MJPC_B200_NO_STATIC", "1")
    m = get_model("quadruped")
    B, steps = 3, 30
    mc, starts, U = _mocap(m), _start(m, B), _ctrl(m, B, steps, seed=4)
    plain, zero, cleared = _bank(m, B, QUAD_SENSORS), _bank(m, B, QUAD_SENSORS), _bank(m, B, QUAD_SENSORS)
    for b in range(B):
        zero.set_disturbance(b, seed=30 + b)
        zero.set_sensor_noise(b, 0.0)
        cleared.set_sensor_noise(b, _std(cleared))
        cleared.set_sensor_noise(b, None)
    ref = _run(plain, starts, mc, U)
    for bank, what in ((zero, "zero std"), (cleared, "cleared")):
        got = _run(bank, starts, mc, U)
        for k in range(steps):
            for f in ("state", "cost", "time", "status", "sensordata", "ctrl"):
                _eq(got[k][f], ref[k][f], f"{case} {what} step {k} {f}")
        for b in range(B):
            g, r = bank.get(b), plain.get(b)
            for f in g:
                _eq(g[f], r[f], f"{case} {what} plant {b} {f}")
        bank.close()
    plain.close()


def test_noise_changes_only_the_measurement_and_has_its_std():
    from plant_noise import plant_normal
    m = get_model("quadruped")
    steps = 2000
    bank = _bank(m, 2, QUAD_SENSORS)
    std = _std(bank, 1)
    std[::5] = 0.0                       # some elements without noise
    q, v = _start(m, 1)[0]
    mc = _mocap(m)
    seed = 77
    for b in range(2):
        bank.reset(b, q, v, 0.0, mc)
        bank.set_disturbance(b, seed=seed)
    bank.set_sensor_noise(0, std)        # plant 1 is the clean twin
    noise = np.zeros((steps, bank.nsensordata))
    u = np.zeros((2, m.nu), np.float32)
    for k in range(steps):
        o = bank.step(u)
        assert (o["status"] == 0).all()
        for f in ("state", "cost", "time", "ctrl"):
            _eq(o[f][0], o[f][1], f"step {k} {f}")
        noise[k] = o["sensordata"][0].astype(float) - o["sensordata"][1].astype(float)
        _eq(o["sensordata"][0][std == 0], o["sensordata"][1][std == 0], f"step {k}: elements with std 0")
        if k < 20:   # the draw: the numpy restatement of the counter (committed step count, 0, element, 'SENS')
            z = plant_normal(seed, k, bank.nsensordata, TAG_SENS)
            clean = np.abs(o["sensordata"][1]) + np.abs(std * z)
            tol = 2 * np.spacing(clean.astype(np.float32)).astype(float) + 1e-4 * np.abs(std * z)
            assert np.all(np.abs(noise[k] - std * z) <= tol), np.max(np.abs(noise[k] - std * z) / tol)
    g0, g1 = bank.get(0), bank.get(1)
    for f in g0:
        _eq(g0[f], g1[f], f"plant fields {f}")
    on = std > 0
    mean, sd = noise[:, on].mean(0), noise[:, on].std(0)
    assert np.all(np.abs(mean) < 4 * std[on] / np.sqrt(steps)), np.max(np.abs(mean) / std[on])
    assert np.all(np.abs(sd / std[on] - 1) < 0.08), (sd / std[on]).round(3)
    print("noise std / std: min %.3f max %.3f over %d steps" % ((sd / std[on]).min(), (sd / std[on]).max(), steps))
    bank.close()


def test_noise_replays_after_reset_and_does_not_depend_on_the_plant_index():
    m = get_model("quadruped")
    steps = 40
    bank = _bank(m, 3, QUAD_SENSORS)
    std = _std(bank, 2)
    q, v = _start(m, 1)[0]
    mc = _mocap(m)
    U = np.zeros((steps, 3, m.nu), np.float32)
    for b in range(3):
        bank.set_disturbance(b, seed=5 if b != 1 else 6)
        bank.set_sensor_noise(b, std)
    first = _run(bank, [(q, v)] * 3, mc, U)
    again = _run(bank, [(q, v)] * 3, mc, U)
    for k in range(steps):
        _eq(first[k]["sensordata"][0], first[k]["sensordata"][2], f"step {k}: plants 0 and 2 share a seed")
        _eq(first[k]["sensordata"], again[k]["sensordata"], f"step {k}: replay after reset")
        assert not np.array_equal(first[k]["sensordata"][0], first[k]["sensordata"][1])
    bank.close()


def test_refusals_leave_the_plant_unchanged():
    from mujoco_mpc_b200.engine import EngineError
    m = get_model("quadruped")
    steps = 10
    bank, ref = _bank(m, 2, QUAD_SENSORS), _bank(m, 2, QUAD_SENSORS)
    std = _std(bank, 3)
    for b in range(2):
        bank.set_sensor_noise(b, std)
        ref.set_sensor_noise(b, std)
    for bad in (-1e-3, np.nan, np.inf):
        s = std.copy()
        s[4] = bad
        with pytest.raises(EngineError, match="plant_set_sensor_noise: std\\[4\\]"):
            bank.set_sensor_noise(1, s)
    lib = bank.lib
    fp = C.POINTER(C.c_float)
    assert lib.mjpc_b200_plant_set_sensor_noise(bank.h, 2, std.ctypes.data_as(fp)) == BAD_ARGUMENT
    assert lib.mjpc_b200_set_model_ensemble(bank.h, *_ensemble(2)) == 0
    assert lib.mjpc_b200_plant_set_sensor_noise(bank.h, 0, None) == UNSUPPORTED
    assert lib.mjpc_b200_set_model_ensemble(bank.h, None, 0, 0) == 0
    starts, mc, U = _start(m, 2), _mocap(m), _ctrl(m, 2, steps, seed=9)
    got, want = _run(bank, starts, mc, U), _run(ref, starts, mc, U)
    for k in range(steps):
        for f in ("state", "sensordata", "cost"):
            _eq(got[k][f], want[k][f], f"step {k} {f} after the refusals")
    bank.close(); ref.close()


def _ensemble(K):
    from mujoco_mpc_b200.engine import _model_blobs
    bufs, arr, n = _model_blobs(_variants("quadruped")[:K])
    _ensemble.keep = bufs
    return arr, n, 1
