"""The plants' disturbance noise restated in numpy (the definition of plant_disturb in csrc/rollout_kernels.cuh and of
mjpc_b200_plant_set_disturbance in include/mjpc_b200.h), in fp64:
  z    Philox4x32-10, key (seed, 2), counter (the plant's committed step count, 0, element, tag), Box-Muller on the
       first two words; tag 'CTRL' for the control noise, 'XFRC' for the body-force noise
  OU   n <- r n + s z with r = exp(-timestep / rate), s = std sqrt(1 - r^2) = std sqrt(-expm1(-2 timestep / rate)),
       from n = 0 at the episode's start"""
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
    s = std * np.sqrt(-np.expm1(-2.0 * timestep / rate))
    x, out = np.zeros(n), np.zeros((steps, n))
    for k in range(steps):
        x = r * x + s * plant_normal(seed, k, n, tag)
        out[k] = x
    return out


# ------------------------------------------------------------------------------------------ counters where fp32 breaks
TAG_SENS = 0x53454E53   # 'SENS'


def philox_words(seeds, step, element, tag, key1=2):
    """Philox4x32-10 words [len(seeds)][4] of counter (step, 0, element, tag) under keys (seed, key1), one key per row:
    planner.philox4x32 with the key vectorised.  tests/test_noise_streams_cpu.py pins both to the published vectors."""
    s = np.asarray(seeds, np.uint64)
    c = np.zeros((len(s), 4), np.uint64)
    c[:, 0], c[:, 2], c[:, 3] = step, element, tag
    k0, k1 = s.copy(), np.full(len(s), key1, np.uint64)
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[:, 0]
        p1 = np.uint64(0xCD9E8D57) * c[:, 2]
        c = np.stack([(p1 >> np.uint64(32)) ^ c[:, 1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[:, 3] ^ k1, p0 & m32], 1)
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return c.astype(np.uint32)


def box_muller(words):
    """fp64 Box-Muller on the first two words: the exact standard normal the stream defines"""
    u1 = (words[..., 0].astype(np.float64) + 0.5) / 4294967296.0
    u2 = (words[..., 1].astype(np.float64) + 0.5) / 4294967296.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


# where the fp32 Box-Muller is fragile: (word, lo, hi) with lo <= word < hi
REGIONS = {
    "far tail c0 < 2^8": (0, 0, 1 << 8),
    "u1 rounds to 1, c0 >= 2^32 - 2^8": (0, (1 << 32) - (1 << 8), 1 << 32),
    "c0 around 2^24": (0, (1 << 24) - (1 << 10), (1 << 24) + (1 << 10)),
    "c0 around 2^31": (0, (1 << 31) - (1 << 10), (1 << 31) + (1 << 10)),
    "c1 at a quarter turn": (1, (1 << 30) - (1 << 10), (1 << 30) + (1 << 10)),
    "c1 at a half turn": (1, (1 << 31) - (1 << 10), (1 << 31) + (1 << 10)),
    "c1 at three quarter turns": (1, 3 * (1 << 30) - (1 << 10), 3 * (1 << 30) + (1 << 10)),
}


def search_counters(tag, elements, per_region=4, chunk=1 << 20, max_seeds=1 << 24):
    """{region: [(seed, element), ...]}: up to per_region plant seeds whose step-0 draw of `element` (< elements) under
    `tag` lands in each region of REGIONS, searching seeds 0, 1, 2, ... until every region has per_region cases (or
    max_seeds seeds were tried).  Each region has probability 2^-24 or 2^-21 per draw."""
    found = {k: [] for k in REGIONS}
    for s0 in range(0, max_seeds, chunk):
        seeds = np.arange(s0, s0 + chunk, dtype=np.uint64)
        for e in range(elements):
            w = philox_words(seeds, 0, e, tag).astype(np.int64)
            for k, (i, lo, hi) in REGIONS.items():
                if len(found[k]) < per_region:
                    hit = np.nonzero((w[:, i] >= lo) & (w[:, i] < hi))[0][:per_region - len(found[k])]
                    found[k] += [(int(seeds[h]), e) for h in hit]
        if all(len(v) >= per_region for v in found.values()):
            break
    return found
