"""The rounding bound of the fp16-pair input projection (gemm_f16x3_kernel, csrc/gemm_tc.cu) and a numpy emulation of its
arithmetic, shared by tests/test_gemm_h16_bound_cpu.py (the emulation meets the bound, and misses it without a
correction product) and tests/test_gpu_gemm_h16.py (the kernel meets it element by element).

Every element of C = A W^T + b must satisfy

    |C - C64| <= kappa * u * S + F,    S = (|A| |W|^T)_mn + |b_n|,  u = 2^-24,

with C64 the float64 result. kappa counts rounding stages, as oracle/grad_gemm.py does for the 3xTF32 GEMMs:

  split       a row of A is scaled by 2^e_m per k-block of 64 and a row of W by 2^e_n (exact powers of 2, so that the row's
              max lies in [2^14, 2^15)), then x = hi + lo with hi = RN_f16(x), lo = RN_f16(x - hi). |x - hi| <= 2^-11 |x|
              and lo's own rounding costs <= 2^-11 |x - hi| <= 2^-22 |x| while lo is a normal fp16; the dropped lo*lo is
              <= 2^-22 |a w|. The three products hi*hi + lo*hi + hi*lo are exact in the MMA: 3 * 2^-22 = 12u |a w| per
              product, summed linearly.
  floor       where hi or lo falls below the fp16 normal range (elements 2^-28 or more below the row's max) the rounding
              is absolute: <= 2^-24 in scaled units, i.e. 2^-24 2^-e per element. F = 2^-24 (2^-e_A sum_k |w| + 2^-e_W
              sum_k |a|) with e_A, e_W the exponents of the whole rows (a k-block's e is at least its row's).
  in-block    12 MMAs chain on the tensor core's truncating accumulator per k-block: 4u per MMA, linearly: 48u.
  cross-block the k-blocks' sums go into a register total with fma(acc, 2^-e_m, total): one round-to-nearest per k-block,
              a chain of K / 64; sqrt(depth) taken LAMBDA = 3 times (Higham & Mary), plus the unscale by 2^-e_n (exact)
              and the two bias additions (2u of S).

    kappa = 3 (sqrt(K / 64) + 1) + 1 + 2 + 48 + 12

A lost correction product costs ~2^-11 of every product of positive operands (hi*lo is not small against u): the sharp
operands of oracle.grad_gemm (a = h (1 + 2^-12)) give lo = 2^-12 hi for TF32-exact h; in fp16 the same operands put
h's bits below fp16's 11 into lo, which the tests use.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
LAMBDA = 3.0
BK = 64


def kappa(K: int) -> float:
    nkb = max(1, (K + BK - 1) // BK)
    return LAMBDA * (math.sqrt(nkb) + 1.0) + 1.0 + 2.0 + 48.0 + 12.0


def scale_exp(m):
    """h16::scale_exp elementwise: 2^e m in [2^14, 2^15); 0 for a zero or non-finite max; e <= 112"""
    m = np.asarray(m, np.float64)
    ok = (m > 0) & np.isfinite(m)
    _, x = np.frexp(np.where(ok, m, 1.0))
    return np.where(ok, np.minimum(15 - x, 112), 0).astype(np.int64)


def split16(x, e):
    """x * 2^e (exact) -> (hi, lo) fp16 values as float64, hi = RN_f16, lo = RN_f16(x 2^e - hi)"""
    v = (np.asarray(x, np.float32).astype(np.float64) * np.exp2(e)).astype(np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def trunc_f32(x):
    x = np.asarray(x, np.float64)
    r = x.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(x)
    return np.where(over, np.nextafter(r, np.float32(0)), r).astype(np.float64)


def emulate(A, W, bias=None, drop=None):
    """C = A[M,K] W[N,K]^T + bias as gemm_f16x3_kernel computes it. drop: "lo_hi" or "hi_lo" leaves that product out"""
    A = np.asarray(A, np.float32)
    W = np.asarray(W, np.float32)
    M, K = A.shape
    N = W.shape[0]
    ew = scale_exp(np.abs(W).max(axis=1))
    wh, wl = split16(W, ew[:, None])
    total = np.zeros((M, N), np.float32)
    for k0 in range(0, K, BK):
        a = A[:, k0:k0 + BK]
        ea = scale_exp(np.abs(a).max(axis=1))
        ah, al = split16(a, ea[:, None])
        acc = np.zeros((M, N))
        for s in range(0, a.shape[1], 16):
            sl = slice(s, s + 16)
            ws = slice(k0 + s, k0 + s + 16)
            for name, x, y in (("lo_hi", al, wh), ("hi_lo", ah, wl), ("hi_hi", ah, wh)):
                if name != drop:
                    acc = trunc_f32(acc + x[:, sl] @ y[:, ws].T)
        # total = fma(acc, 2^-e_m, total): one rounding
        total = (total.astype(np.float64) + acc * np.exp2(-ea)[:, None]).astype(np.float32)
    out = (total.astype(np.float64) * np.exp2(-ew)[None, :]).astype(np.float32)
    if bias is not None:
        out = (out + np.asarray(bias, np.float32)[None, :]).astype(np.float32)
    return out


def bound(A, W, bias=None):
    """(C64, kappa u S + F) in float64"""
    A64 = np.asarray(A, np.float64)
    W64 = np.asarray(W, np.float64)
    C64 = A64 @ W64.T
    S = np.abs(A64) @ np.abs(W64).T
    if bias is not None:
        b = np.asarray(bias, np.float64)
        C64 = C64 + b[None, :]
        S = S + np.abs(b)[None, :]
    ea = scale_exp(np.abs(A64).max(axis=1))
    ew = scale_exp(np.abs(W64).max(axis=1))
    F = 2.0 ** -24 * (np.exp2(-ea)[:, None] * np.abs(W64).sum(axis=1)[None, :] +
                      np.exp2(-ew)[None, :] * np.abs(A64).sum(axis=1)[:, None])
    return C64, kappa(A64.shape[1]) * U * S + F


def max_ratio(C, A, W, bias=None) -> float:
    C64, bnd = bound(A, W, bias)
    return float((np.abs(np.asarray(C, np.float64) - C64) / bnd).max())
