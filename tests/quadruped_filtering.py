"""The Quadruped filtering scenario shared by tests/test_estimator_cpu.py (which derives the bar from the oracle-backed
filters) and tests/test_gpu_estimator.py (which holds the engine-backed filters to it).

Plant: the fp64 oracle from the home keyframe at estimator_timestep (0.005 s), driven by a joint PD law towards the home
pose plus a seeded sinusoid and Gaussian torque noise that lifts and replants the feet (contacts make and break).  The
21 measured sensors (5 framepos, 12 jointpos, 4 touch) get seeded Gaussian noise of std SENSOR_SD, and the filter's
sensor noise variance is SENSOR_SD^2.  The error is the RMS over steps 50 .. 199 of the filtered qpos / qvel against
the plant's state after the step.
"""
import numpy as np

from estimator_backends import simulate

SENSOR_SD = 1e-3
STEPS = 200


def plant(m):
    k = m.key_names.index("home")
    home = m.key_qpos[k]
    rng = np.random.default_rng(5)
    kicks = 0.3 * rng.normal(size=(STEPS + 1, m.nu))

    def ctrl(t, x):
        return np.clip(2.0 * (home[7:] - x[7:m.nq]) - 0.1 * x[m.nq + 6:] + 0.6 * np.sin(0.1 * t + np.arange(m.nu))
                       + kicks[t], -1, 1)
    x0 = np.concatenate([home, np.zeros(m.nv)])
    return simulate(m, x0[:m.nq], x0[m.nq:], STEPS + 1, timestep=0.005, ctrl=ctrl, start=9, count=21, noise=SENSOR_SD,
                    seed=6)


def run_filter(m, f, X, Y, U, mocap):
    """Filter the plant's measurements; returns (rms qpos error, rms qvel error, max asymmetry, min eigenvalue)."""
    f.reset(state=X[0])
    f.set_noise(sensor=np.full(f.nsensordata, SENSOR_SD ** 2))
    eq, ev, asym, mineig = [], [], 0.0, np.inf
    for t in range(STEPS):
        f.update(U[t], Y[t], mocap)
        s, P = f.state, f.covariance
        eq.append(s[:m.nq] - X[t + 1, :m.nq]); ev.append(s[m.nq:] - X[t + 1, m.nq:])
        asym = max(asym, float(np.abs(P - P.T).max()))
        mineig = min(mineig, float(np.linalg.eigvalsh(0.5 * (P + P.T)).min()))
    return (float(np.sqrt(np.mean(np.square(eq[50:])))), float(np.sqrt(np.mean(np.square(ev[50:])))), asym, mineig)
