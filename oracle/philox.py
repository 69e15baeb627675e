"""TEST INFRASTRUCTURE ONLY -- Philox4x32-10 on the host, with curand's conventions, so that a test knows every
uniform the sampling kernel (``lade_sample_verify``) will draw before it launches it.

The kernel calls ``curand_init(seed, 0, offset, &state)`` and then ``curand_uniform`` once per draw.  In curand
(``curand_kernel.h``, ``curand_philox4x32_x.h``):

* key = (seed lo, seed hi);
* counter = (c0, c1, c2, c3) = (offset/4 lo, offset/4 hi, subsequence lo, subsequence hi), carried as one 128-bit
  little-endian integer: word n of the stream is output word n % 4 of Philox(counter of n // 4);
* ten rounds; each round maps (c0, c1, c2, c3) to (hi(M1*c2) ^ c1 ^ k0, lo(M1*c2), hi(M0*c0) ^ c3 ^ k1, lo(M0*c0)),
  then the key is bumped by (W0, W1) between rounds;
* ``curand_uniform(x) = float(x) * 2^-32 + 2^-33`` in fp32 (the product is exact, so one rounding), range (0, 1].

Everything is vectorised over counters: the probe searches scan millions of offsets.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key) -> np.ndarray:
    """ctr: (..., 4) uint32 counters, key: (2,) uint32 -> (..., 4) uint32 outputs."""
    c = np.asarray(ctr, dtype=np.uint32).astype(np.uint64)
    c0, c1, c2, c3 = c[..., 0], c[..., 1], c[..., 2], c[..., 3]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c0, M1 * c2                      # < 2^64: exact in uint64
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & _MASK32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & _MASK32)
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def _key(seed: int):
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return (seed & 0xFFFFFFFF, seed >> 32)


def words(seed: int, offset, n: int, subsequence: int = 0) -> np.ndarray:
    """The n 32-bit words curand returns after ``curand_init(seed, subsequence, offset)``.
    `offset` may be an int (-> shape (n,)) or an integer array (-> shape offset.shape + (n,))."""
    if np.ndim(offset) == 0:                                         # one run of words: each block computed once
        o = int(offset)
        q0, q1 = o >> 2, (o + n + 3) >> 2
        q = np.arange(q1 - q0, dtype=np.uint64) + np.uint64(q0)
        ctr = np.stack([q & _MASK32, q >> np.uint64(32), np.full_like(q, subsequence & 0xFFFFFFFF),
                        np.full_like(q, (subsequence >> 32) & 0xFFFFFFFF)], -1)
        return philox4x32_10(ctr, _key(seed)).reshape(-1)[o & 3:(o & 3) + n]
    off = np.asarray(offset, dtype=np.uint64)
    idx = off[..., None] + np.arange(n, dtype=np.uint64)            # absolute word index in the subsequence
    q = idx >> np.uint64(2)
    ctr = np.stack([q & _MASK32, q >> np.uint64(32),
                    np.full_like(q, subsequence & 0xFFFFFFFF), np.full_like(q, (subsequence >> 32) & 0xFFFFFFFF)], -1)
    out = philox4x32_10(ctr, _key(seed))
    return np.take_along_axis(out, (idx & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]


def to_uniform(x) -> np.ndarray:
    """curand_uniform of 32-bit words: fp32, in (0, 1]."""
    f = np.asarray(x, dtype=np.uint32).astype(np.float32)           # round to nearest, like cvt.rn.f32.u32
    return f * np.float32(2.0 ** -32) + np.float32(2.0 ** -33)


def uniforms(seed: int, offset, n: int) -> np.ndarray:
    """The n fp32 uniforms the kernel draws from rng_state = (seed, offset)."""
    return to_uniform(words(seed, offset, n))


def advance(n_draws: int) -> int:
    """How far the kernel moves rng_state[1] after n_draws draws: whole Philox blocks of 4 words."""
    return (int(n_draws) + 3) & ~3
