"""The fp16-pair input projection's rounding bound (tests/gemm_h16_bound.py) is met by a numpy emulation of its arithmetic
(row scale per k-block of 64, fp16 hi / lo, three products per k16 step, truncating accumulation restarted per k-block,
fma unscale) and missed by one that drops a correction product, without a GPU."""
import numpy as np
import pytest

from gemm_h16_bound import emulate, max_ratio, scale_exp


def _sharp(M, K, N, rng, e=20):
    """positive operands h (1 + 2^-12), h fp16-exact in [1, 2): lo carries 2^-12 of every element, so a lost correction
    product moves each output by ~2^-12 S; rows of A and of W scaled by 2^[-e, e]"""
    def one(shape):
        return rng.uniform(1.0, 2.0, shape).astype(np.float16).astype(np.float64) * (1.0 + 2.0 ** -12)
    A = one((M, K)) * np.exp2(rng.integers(-e, e + 1, (M, 1)))
    W = one((N, K)) * np.exp2(rng.integers(-e, e + 1, (N, 1)))
    return A.astype(np.float32), W.astype(np.float32)


def _operands(kind, M, K, N, rng):
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    if kind == "sharp":
        return _sharp(M, K, N, rng)
    if kind == "scaled":  # rows and columns x 2^[-20, 20]
        A = A * np.exp2(rng.integers(-20, 21, (M, 1))) * np.exp2(rng.integers(-20, 21, (1, K)))
        W = W * np.exp2(rng.integers(-20, 21, (N, 1)))
    elif kind == "zero":
        A[1] = 0.0
        A[2, : K // 2] = 0.0
        W[0] = 0.0
    elif kind == "subnormal":
        A[0, ::3] = np.float32(1e-40)
        A[1] = np.float32(3e-42) * rng.standard_normal(K).astype(np.float32)
        W[1, ::5] = np.float32(2e-39)
    elif kind == "huge":
        A[0, 3] = np.float32(1e30)
        W[2, 7] = np.float32(-1e20)
    return A.astype(np.float32), W.astype(np.float32)


@pytest.mark.parametrize("K", [64, 128, 256, 1024])
@pytest.mark.parametrize("kind", ["random", "sharp", "scaled", "zero", "subnormal", "huge"])
def test_intact_emulation_meets_the_bound(K, kind):
    rng = np.random.default_rng(K)
    A, W = _operands(kind, 5, K, 7, rng)
    b = rng.standard_normal(7).astype(np.float32)
    C = emulate(A, W, b)
    assert np.isfinite(C).all()
    assert max_ratio(C, A, W, b) <= 0.5


@pytest.mark.parametrize("K", [64, 256, 1024])
@pytest.mark.parametrize("drop", ["lo_hi", "hi_lo"])
def test_dropped_correction_product_fails(K, drop):
    rng = np.random.default_rng(K + 1)
    A, W = _sharp(3, K, 4, rng)
    assert max_ratio(emulate(A, W, drop=drop), A, W) > 10.0


def test_scale_exp_rules():
    m = np.array([0.0, np.inf, np.nan, 1.0, 2.0 ** 14, 2.0 ** 15, 1e-38, 1e-45, 3.0e38])
    e = scale_exp(m)
    assert e[0] == 0 and e[1] == 0 and e[2] == 0
    for v, x in zip(m[3:6], e[3:6]):
        assert 2.0 ** 14 <= v * 2.0 ** x < 2.0 ** 15
    assert e[6] == 112 and e[7] == 112 and e[8] < 0  # below 2^-98 the scale is capped


def test_non_finite_rows_stay_in_their_row():
    rng = np.random.default_rng(3)
    A, W = _operands("random", 6, 128, 5, rng)
    A[2, 5] = np.nan
    A[4, 70] = np.inf
    C = emulate(A, W)
    bad = ~np.isfinite(C)
    assert bad[2].all() and bad[4].all()
    assert not bad[[0, 1, 3, 5]].any()
