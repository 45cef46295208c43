"""Host oracle of the sampler's counter-based noise (``ns2vc_b200/csrc/philox.cuh``): Philox4x32-10 in numpy uint32 arithmetic and
the fp64 Box-Muller transform of the same (u, v).

Layout: key = the 64-bit seed (lo, hi), counter = (t >> 2, c, step, 0); frames t & 3 = 0, 1 take z0, z1 of the output pair
(x, y), frames 2, 3 those of (z, w).  ``XT_STEP`` is the step reserved for an utterance's x_T."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
XT_STEP = 0xFFFFFFFF
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key) -> np.ndarray:
    """counter [..., 4] and key [..., 2] (uint32, broadcast against each other) -> the four uint32 outputs [..., 4]."""
    ctr = np.asarray(counter, dtype=np.uint32)
    k = np.asarray(key, dtype=np.uint32)
    shape = np.broadcast_shapes(ctr.shape[:-1], k.shape[:-1])
    ctr, k = np.broadcast_to(ctr, shape + (4,)), np.broadcast_to(k, shape + (2,))
    c0, c1, c2, c3 = (ctr[..., i].astype(np.uint64) for i in range(4))
    k0, k1 = k[..., 0].copy(), k[..., 1].copy()
    with np.errstate(over="ignore"):
        for r in range(10):
            if r > 0:
                k0 = k0 + W0
                k1 = k1 + W1
            p0, p1 = M0 * c0, M1 * c2
            n0 = (p1 >> np.uint64(32)) ^ c1 ^ k0.astype(np.uint64)
            n2 = (p0 >> np.uint64(32)) ^ c3 ^ k1.astype(np.uint64)
            c1, c3 = p1 & _LO, p0 & _LO
            c0, c2 = n0, n2
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def uv(a, b):
    """The Box-Muller inputs of the output pair (a, b) as the device forms them: u = fp32((a >> 8) + 0.5) * 2^-24 in (0, 1]
    (the sum needs 25 bits from 2^23 up and is rounded once, to nearest even) and v = (b >> 8) * 2^-24 in [0, 1) (exact)."""
    a, b = np.asarray(a, dtype=np.uint32), np.asarray(b, dtype=np.uint32)
    u = ((a >> 8).astype(np.float64) + 0.5).astype(np.float32).astype(np.float64) * 2.0 ** -24
    return u, (b >> 8).astype(np.float64) * 2.0 ** -24


def box_muller(a, b):
    """(z0, z1, r) in fp64 of the output pair (a, b)."""
    u, v = uv(a, b)
    r = np.sqrt(-2.0 * np.log(u))
    return r * np.cos(2.0 * np.pi * v), r * np.sin(2.0 * np.pi * v), r


def seed_key(seeds) -> np.ndarray:
    s = np.asarray(seeds, dtype=np.uint64)
    return np.stack([(s & _LO).astype(np.uint32), (s >> np.uint64(32)).astype(np.uint32)], -1)


def normal(seed: int, step: int, C: int, T: int):
    """(noise, r) [C, T] in fp64: the normal at (seed, step, c, t) for every c < C, t < T, and its Box-Muller radius."""
    c = np.arange(C, dtype=np.uint32)[:, None]
    t = np.arange(T, dtype=np.uint32)[None, :]
    ctr = np.stack(np.broadcast_arrays(t >> 2, c, np.uint32(step), np.uint32(0)), -1)
    o = philox4x32_10(ctr, seed_key(seed))
    second = (t & 2) != 0
    a = np.where(second, o[..., 2], o[..., 0])
    b = np.where(second, o[..., 3], o[..., 1])
    z0, z1, r = box_muller(a, b)
    return np.where((t & 1) != 0, z1, z0), r
