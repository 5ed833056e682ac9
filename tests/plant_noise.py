"""The plants' disturbance noise restated in numpy (the definition of plant_disturb in csrc/rollout_kernels.cuh and of
mjpc_b200_plant_set_disturbance in include/mjpc_b200.h), in fp64:
  z    Philox4x32-10, key (seed, 2), counter (the plant's committed step count, 0, element, tag), Box-Muller on the
       first two words; tag 'CTRL' for the control noise, 'XFRC' for the body-force noise
  OU   n <- r n + s z with r = exp(-timestep / rate), s = std sqrt(1 - r^2), from n = 0 at the episode's start"""
import numpy as np

from mujoco_mpc_b200.planner import philox4x32

TAG_CTRL = 0x4354524C   # 'CTRL'
TAG_XFRC = 0x58465243   # 'XFRC'


def plant_normal(seed, step, n, tag):
    """The n standard normals of one plant step: z[element] for element 0 .. n-1."""
    ctr = np.array([[step, 0, e, tag] for e in range(n)], np.uint32).reshape(n, 4)
    r = philox4x32(ctr, (seed, 2))
    u1 = (r[:, 0].astype(np.float64) + 0.5) / 4294967296.0
    u2 = (r[:, 1].astype(np.float64) + 0.5) / 4294967296.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def ou_states(seed, steps, n, std, rate, timestep, tag):
    """[steps][n]: the OU state after each of the first `steps` committed steps (row k is the noise step k applied)."""
    r = np.exp(-timestep / rate)
    s = std * np.sqrt(1.0 - r * r)
    x, out = np.zeros(n), np.zeros((steps, n))
    for k in range(steps):
        x = r * x + s * plant_normal(seed, k, n, tag)
        out[k] = x
    return out
