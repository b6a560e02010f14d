"""Philox4x32-10 and the dropout keep mask, in numpy, bit for bit as the kernels draw them.

Layout (``philox4x32_10`` in csrc/common.cuh): key = seed (low word k0, high word k1); the 128-bit counter is
(ctr_lo, ctr_hi) = (offset + idx // 4, stream id); element idx of a dropout stream reads word idx % 4 of that call.
Every dropout site draws this way: ``dropout_kernel`` (inter-layer, stream = layer index), ``mlp_dropout_kernel``
(stream, stream + 1) and the four streams of ``fuse_head_kernel`` (0 / 1 text, 2 / 3 audio).

The keep test is the device's: thr = (uint32) fminf(p * 2^32, 4294967295.0f) computed in fp32 (saturating, so p = 1
drops everything), keep iff word >= thr; kept values are scaled by 1 / (1 - p) in fp32 (0 at p = 1).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed, ctr_lo, ctr_hi):
    """Four uint32 words per counter: arrays broadcast; returns uint32 [..., 4]."""
    seed = np.asarray(seed, dtype=np.uint64)
    ctr_lo = np.asarray(ctr_lo, dtype=np.uint64)
    ctr_hi = np.asarray(ctr_hi, dtype=np.uint64)
    seed, ctr_lo, ctr_hi = np.broadcast_arrays(seed, ctr_lo, ctr_hi)
    k0 = (seed & _LO).astype(np.uint32)
    k1 = (seed >> np.uint64(32)).astype(np.uint32)
    c0 = (ctr_lo & _LO).astype(np.uint32)
    c1 = (ctr_lo >> np.uint64(32)).astype(np.uint32)
    c2 = (ctr_hi & _LO).astype(np.uint32)
    c3 = (ctr_hi >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0 = k0 + W0
            k1 = k1 + W1
    return np.stack([c0, c1, c2, c3], axis=-1)


def words(seed, offset, stream, n):
    """The n uint32 words elements 0..n-1 of one dropout stream read."""
    nq = (int(n) + 3) // 4
    q = np.arange(nq, dtype=np.uint64) + np.uint64(offset)
    return philox4x32_10(np.uint64(seed), q, np.uint64(stream)).reshape(-1)[:n]


def threshold(p):
    """(uint32) fminf(p * 4294967296.0f, 4294967295.0f), every step in fp32 as on the device."""
    t = np.float32(p) * np.float32(4294967296.0)
    t = min(t, np.float32(4294967295.0))   # fp32(4294967295) == 2^32: the conversion saturates to 0xFFFFFFFF
    return np.uint32(min(int(t), 0xFFFFFFFF))


def scale(p):
    """1 / (1 - p) in fp32, 0 at p >= 1 (launch_dropout / the fuse head / mlp_dropout)."""
    p = np.float32(p)
    return np.float32(np.float32(1.0) / (np.float32(1.0) - p)) if p < np.float32(1.0) else np.float32(0.0)


def keep_mask(seed, offset, stream, n, p):
    """bool [n]: element i of stream `stream` is kept."""
    return words(seed, offset, stream, n) >= threshold(p)


def dropout_factor(seed, offset, stream, n, p):
    """fp32 [n]: the factor the kernels multiply element i by (scale or 0)."""
    return np.where(keep_mask(seed, offset, stream, n, p), scale(p), np.float32(0.0)).astype(np.float32)
