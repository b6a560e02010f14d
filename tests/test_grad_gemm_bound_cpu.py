"""The gradient-GEMM rounding bound (oracle/grad_gemm.py) is met by an intact emulation of the tensor-core GEMM and
missed by one that loses a correction product, without a GPU.

oracle.grad_gemm.emulate_tc runs the 3xTF32 arithmetic of gemm_tf32x3_kernel in numpy: TF32 split, lo operands read as
TF32, truncating accumulation inside each k-block of 32, round-to-nearest sums over k-blocks and over K splits. The
shapes are those of tests/test_gpu_grad_gemm_f64.py cut to a few rows and columns (the bound is per element, so M and N
do not enter it), the K values and splits are theirs."""
import numpy as np
import pytest

from oracle.grad_gemm import U, emulate_tc, kappa, max_ratio, sharp_operands

# K, split-K count as tc_splitk_plan chooses it at these K (1 split below 16 k-blocks), k-blocks per split
CASES = [(1, 1), (31, 1), (32, 1), (33, 1), (480, 1), (1100, 4), (1856, 7), (7616, 11), (15360, 1)]


def _plan(K, splitk):
    nkb = (K + 31) // 32
    kbs = (nkb + splitk - 1) // splitk
    return (nkb + kbs - 1) // kbs, kbs


def _ratio(A, B, splitk, kbs, tf32=False, drop=None, C0=None):
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    C64 = A64 @ B64 + (0 if C0 is None else C0.astype(np.float64))
    S = np.abs(A64) @ np.abs(B64) + (0 if C0 is None else np.abs(C0.astype(np.float64)))
    C = emulate_tc(A, B, splitk=splitk, kb_per_split=kbs, tf32=tf32, drop=drop, C0=C0)
    return max_ratio(C, C64, S, kappa("tc", tf32, kbs, splitk))


@pytest.mark.parametrize("K,splitk", CASES)
@pytest.mark.parametrize("data", ["sharp", "random"])
def test_intact_emulation_meets_the_bound(K, splitk, data):
    rng = np.random.default_rng(K)
    M, N = 4, 6
    if data == "sharp":
        A, B = sharp_operands(M, K, N, rng)
    else:
        A = rng.standard_normal((M, K)).astype(np.float32)
        B = rng.standard_normal((K, N)).astype(np.float32)
    splitk, kbs = _plan(K, splitk)
    assert _ratio(A, B, splitk, kbs) <= 0.5
    C0 = rng.standard_normal((M, N)).astype(np.float32) * np.float32(np.sqrt(K))
    assert _ratio(A, B, splitk, kbs, C0=C0) <= 0.5


@pytest.mark.parametrize("K,splitk", CASES)
@pytest.mark.parametrize("drop", ["a_lo_b_hi", "a_hi_b_lo"])
def test_lost_correction_product_fails_on_sharp_operands(K, splitk, drop):
    rng = np.random.default_rng(K + 1)
    A, B = sharp_operands(3, K, 5, rng)
    splitk, kbs = _plan(K, splitk)
    assert _ratio(A, B, splitk, kbs, drop=drop) > 10.0


@pytest.mark.parametrize("K", [1, 31, 32, 33])
def test_lost_correction_product_fails_on_random_operands_at_small_k(K):
    rng = np.random.default_rng(K + 2)
    A = rng.standard_normal((64, K)).astype(np.float32)
    B = rng.standard_normal((K, 64)).astype(np.float32)
    assert _ratio(A, B, 1, (K + 31) // 32, drop="a_lo_b_hi") > 1.0


def test_lost_product_shift_is_2_to_the_minus_12_of_s():
    """the sharp operands' claim itself: hi = h, lo = 2^-12 h exactly, so the lost product is 2^-12 S on every element"""
    rng = np.random.default_rng(0)
    A, B = sharp_operands(3, 64, 4, rng, scale_exp=0)
    S = np.abs(A.astype(np.float64)) @ np.abs(B.astype(np.float64))
    shift = emulate_tc(A, B) - emulate_tc(A, B, drop="a_lo_b_hi")
    assert np.allclose(shift / S, 2.0 ** -12 / (1 + 2.0 ** -12) ** 2, rtol=1e-3)
    assert (shift / (U * S)).min() > 4000


def test_tf32_emulation_on_rounded_operands_is_the_accumulation_only():
    from oracle.tf32 import round_tf32

    rng = np.random.default_rng(5)
    A = rng.standard_normal((4, 1100)).astype(np.float32)
    B = rng.standard_normal((1100, 6)).astype(np.float32)
    Ar, Br = round_tf32(A).astype(np.float64), round_tf32(B).astype(np.float64)
    C = emulate_tc(A, B, splitk=4, kb_per_split=9, tf32=True)
    assert max_ratio(C, Ar @ Br, np.abs(Ar) @ np.abs(Br), kappa("tc", True, 9, 4)) <= 0.5
