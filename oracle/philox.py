"""Independent reference of the dropout RNG of the library: Random123's Philox4x32-10 and the element -> multiplier mapping the
C-ABI documents (pnp_dropout_cfg in include/pnp_b200.h, the comments above pnp_dropout_bits8 / pnp_make_drop in common.cuh).

    element i of a tensor draws Philox block i >> 3 with counter (lo(i >> 3), hi(i >> 3), lo(stream), hi(stream)) and key
    (lo(seed), hi(seed)); it reads 32-bit word (i & 7) >> 1 of the block, its low 16 bits when i is even and its high 16 bits
    when i is odd; it is kept iff that 16-bit draw is below thresh = clamp(uint(fl32(fl32(keep * 65536) + 0.5f)), 0, 65536),
    and a kept element is multiplied by fl32(1 / keep), a dropped one by 0.  keep >= 1 or no seed disables dropout.
    pnp_seed_advance replaces the seed by seed * 6364136223846793005 + 1442695040888963407 mod 2^64.

Everything is numpy over uint64 (products of two 32-bit words fit), vectorised over blocks; no GPU is needed."""
import numpy as np

PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
LCG_MUL, LCG_INC = 6364136223846793005, 1442695040888963407
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11; Random123 philox4x32 with 10 rounds).  ctr [..., 4] and key [..., 2] are arrays of
    32-bit words (any integer dtype, broadcastable against each other); returns the [..., 4] uint32 output block."""
    ctr = np.asarray(ctr, dtype=np.uint64) & _M32
    key = np.asarray(key, dtype=np.uint64) & _M32
    c0, c1, c2, c3 = (ctr[..., j] for j in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    m0, m1 = np.uint64(PHILOX_M[0]), np.uint64(PHILOX_M[1])
    w0, w1 = np.uint64(PHILOX_W[0]), np.uint64(PHILOX_W[1])
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2                         # exact: both factors < 2^32
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _M32, p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), axis=-1).astype(np.uint32)


def lo32(v):
    return int(v) & 0xFFFFFFFF


def hi32(v):
    return (int(v) >> 32) & 0xFFFFFFFF


def blocks(seed, stream, nblocks, first=0):
    """Philox output blocks first .. first + nblocks - 1 of (seed, stream): [nblocks, 4] uint32"""
    b = np.arange(first, first + nblocks, dtype=np.uint64)
    ctr = np.stack([b & _M32, b >> np.uint64(32), np.full_like(b, lo32(stream)), np.full_like(b, hi32(stream))], axis=-1)
    return philox4x32_10(ctr, np.array([lo32(seed), hi32(seed)], dtype=np.uint64))


def draws16(seed, stream, n):
    """the 16-bit draw of each of the elements 0 .. n-1: [n] uint32 in [0, 65536)"""
    words = blocks(seed, stream, (n + 7) // 8).reshape(-1)       # word w of block b sits at 4 b + w
    i = np.arange(n, dtype=np.int64)
    w = words[4 * (i >> 3) + ((i & 7) >> 1)]
    return np.where(i & 1, w >> np.uint32(16), w & np.uint32(0xFFFF))


def keep_threshold(keep):
    """pnp_make_drop's threshold: clamp(uint(fl32(fl32(keep * 65536) + 0.5f)), 0, 65536), keep taken as fp32"""
    t = np.float32(np.float32(np.float32(keep) * np.float32(65536.0)) + np.float32(0.5))
    return 0 if t <= 0 else (65536 if t >= 65536 else int(t))


def inv_keep(keep):
    return np.float32(np.float32(1.0) / np.float32(keep))


def enabled(seed, keep):
    return seed is not None and np.float32(keep) < np.float32(1.0)


def dropout_mult(seed, stream, keep, n):
    """the fp32 multiplier of each of the elements 0 .. n-1 (1 everywhere when dropout is disabled)"""
    if not enabled(seed, keep):
        return np.ones(n, dtype=np.float32)
    kept = draws16(seed, stream, n) < keep_threshold(keep)
    return np.where(kept, inv_keep(keep), np.float32(0.0)).astype(np.float32)


def seed_advance(s, k=1):
    """pnp_seed_advance applied k times"""
    for _ in range(k):
        s = (int(s) * LCG_MUL + LCG_INC) % (1 << 64)
    return s
