"""ORACLE — test infrastructure only (never imported by the product path).

The rounding bound of the backward's gradient GEMMs (csrc/api.cu run_grad_gemm) and a numpy emulation of their
tensor-core arithmetic with the same k-block structure, so that the bound's sharpness can be checked without a GPU
(tests/test_grad_gemm_bound_cpu.py) and then applied element by element to the kernels (tests/test_gpu_grad_gemm_f64.py).

Every element of C = A B (+ C0) must satisfy

    |C - C64| <= kappa * u * S,    S = (|A| |B|)_ij (+ |C0_ij| when accumulating),  u = 2^-24,

with C64 the float64 product of the operands as the GEMM addresses them (TF32 mode: the operands rounded to TF32 first,
as split_tf32_kernel rounds them, so that only the accumulation error is left). kappa counts rounding stages:

  split       3xTF32 only: a*b = ah*bh + al*bh + ah*bl with ah = rna_tf32(a), al = a - ah exact, |al| <= 2^-11 |a|.
              The dropped al*bl is <= 2^-22 |a b| = 4u |a b|; the MMA reads al and bl as TF32 (the low 13 bits are
              ignored), which costs <= 2^-10 |al| |bh| <= 2^-21 |a b| = 8u |a b| for each of the two correction products:
              20u |a b| per product, worst case, summed linearly.
  in-block    within one k-block of 32 the MMAs chain on the tensor core's accumulator (12 in 3xTF32, 4 in TF32), which
              adds with truncation: per MMA at most 2 ulps = 4u of the block's |terms| (one for the truncated result,
              one for the alignment of the addends). Truncation is biased, so this is counted linearly: 48u (3xTF32) or
              16u (TF32) of S.
  cross-block each k-block's sum is added into a register total with round-to-nearest, `chain` times per split (the
              FFMA path: one fmaf per K value, `chain` = K values per split); then the split-K reduce adds `splitk`
              partials, and accumulating adds C0 once. An accumulation chain of depth d errs by sqrt(d) u S with high
              probability when the roundings are independent (Higham & Mary, SIAM J. Sci. Comput. 41(5), 2019); the
              maximum is taken over up to 10^7 elements here, so the sqrt(d) is taken LAMBDA = 3 times.

    kappa = 3 (sqrt(chain) + sqrt(splitk)) + 1  [+ 48 + 20 on 3xTF32 tensor cores, + 16 on TF32 ones]

A lost correction product shifts every output of positive TF32-exact operands a = h (1 + 2^-12) by 2^-12 S = 4096 u S:
at K = 15360 on one split the 3xTF32 kappa is 3 (sqrt(480) + 1) + 69 = 138, thirty times smaller. On random operands
the loss is a random-sign sum, ~2^-11 / sqrt(3 K) of S, which the bound catches at small K.
"""
from __future__ import annotations

import math

import numpy as np

from .tf32 import round_tf32

U = 2.0 ** -24
LAMBDA = 3.0
BK = 32               # k-block of the tensor-core GEMM (gemm_tc.cu)
MMAS_PER_BLOCK = {False: 12, True: 4}   # 3xTF32 / single-pass TF32
SPLIT_3XTF32 = 20.0
TRUNC_PER_MMA = 4.0


def kappa(path: str, tf32: bool, chain: int, splitk: int) -> float:
    """chain: k-blocks per split (path "tc") or K values per split (path "ffma")"""
    k = LAMBDA * (math.sqrt(max(chain, 1)) + math.sqrt(max(splitk, 1))) + 1.0
    if path == "tc":
        k += TRUNC_PER_MMA * MMAS_PER_BLOCK[bool(tf32)] + (0.0 if tf32 else SPLIT_3XTF32)
    return k


# ---- numpy emulation of the tensor-core GEMM ------------------------------------------------------------------------

def trunc_tf32(x) -> np.ndarray:
    """what the MMA reads of an fp32 value: its 13 low mantissa bits ignored (toward zero). Returns float64."""
    a = np.ascontiguousarray(np.asarray(x, dtype=np.float32))
    return (a.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def trunc_f32(x) -> np.ndarray:
    """float64 -> float32 rounded toward zero (the tensor core's accumulator), returned as float64"""
    x = np.asarray(x, dtype=np.float64)
    r = x.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(x)
    r = np.where(over, np.nextafter(r, np.float32(0)), r)
    return r.astype(np.float64)


def emulate_tc(A, B, splitk=1, kb_per_split=None, tf32=False, drop=None, C0=None) -> np.ndarray:
    """C = A[M,K] B[K,N] (+ C0) as gemm_tf32x3_kernel computes it: operands split hi = rna_tf32, lo = x - hi (lo read
    as TF32 by the MMA); per k-block of 32 the k-steps of 8 run the MMAs lo*hi, hi*lo, hi*hi (TF32: hi*hi) on an
    accumulator that starts from zero and truncates; the block sum goes into a float32 total with round-to-nearest;
    split-K partials are added in split order, then C0. drop: "a_lo_b_hi" or "a_hi_b_lo" leaves that product out."""
    A = np.asarray(A, np.float32)
    B = np.asarray(B, np.float32)
    M, K = A.shape
    N = B.shape[1]
    ah, bh = round_tf32(A), round_tf32(B)
    al, bl = trunc_tf32(A - ah), trunc_tf32(B - bh)
    ah, bh = ah.astype(np.float64), bh.astype(np.float64)
    nkb = (K + BK - 1) // BK
    if kb_per_split is None:
        kb_per_split = (nkb + splitk - 1) // splitk
    prods = [(ah, bh)] if tf32 else [p for n, p in (("a_lo_b_hi", (al, bh)), ("a_hi_b_lo", (ah, bl)),
                                                     ("a_hi_b_hi", (ah, bh))) if n != drop]
    parts = []
    for s0 in range(0, nkb, kb_per_split):
        total = np.zeros((M, N), np.float32)
        for kb in range(s0, min(nkb, s0 + kb_per_split)):
            acc = np.zeros((M, N))
            for k0 in range(kb * BK, min(K, kb * BK + BK), 8):
                k1 = min(K, k0 + 8)
                for x, y in prods:
                    acc = trunc_f32(acc + x[:, k0:k1] @ y[k0:k1, :])
            total = (total + acc.astype(np.float32)).astype(np.float32)
        parts.append(total)
    if len(parts) == 1 and C0 is None:
        return parts[0]
    s = np.zeros((M, N), np.float32)
    for p in parts:
        s = (s + p).astype(np.float32)
    if C0 is not None:
        s = (s + np.asarray(C0, np.float32)).astype(np.float32)
    return s


def sharp_operands(M, K, N, rng, scale_exp=20):
    """positive operands a = h (1 + 2^-12) with h exactly TF32 (so hi = h and lo = 2^-12 h exactly: every correction
    product is positive and a lost one moves each output by 2^-12 S), rows of A and columns of B scaled by 2^e,
    e in [-scale_exp, scale_exp]"""
    def one(shape):
        h = round_tf32(rng.uniform(1.0, 2.0, shape)).astype(np.float64)
        return h * (1.0 + 2.0 ** -12)
    A = one((M, K)) * np.exp2(rng.integers(-scale_exp, scale_exp + 1, (M, 1)))
    B = one((K, N)) * np.exp2(rng.integers(-scale_exp, scale_exp + 1, (1, N)))
    return A.astype(np.float32), B.astype(np.float32)


def max_ratio(C, C64, S, kap) -> float:
    """max over elements of |C - C64| / (kappa u S)"""
    err = np.abs(np.asarray(C, np.float64) - C64)
    return float((err / (kap * U * S)).max())
