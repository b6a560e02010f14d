"""oracle/round16.py against numpy's float64 -> float16 conversion (correctly rounded in one step) and torch's
float32 -> bfloat16 conversion on float32 inputs (one rounding), at every part of the range: normal, subnormal,
overflow, ties and the midpoints the distance function reports."""
import numpy as np
import torch

from oracle.round16 import midpoint_distance, round16, ulp16


def _samples(rng, lo, hi, n=20000):
    mag = np.exp2(rng.uniform(lo, hi, n))
    return np.concatenate([mag * rng.choice([-1.0, 1.0], n), [0.0, -0.0, np.inf, -np.inf]])


def test_round16_float16_matches_numpy():
    rng = np.random.default_rng(0)
    v = _samples(rng, -27, 17)
    with np.errstate(over="ignore"):
        assert np.array_equal(round16(v, torch.float16), v.astype(np.float16).astype(np.float64))
    # ties: exact midpoints round to even, the overflow threshold rounds to infinity
    q = ulp16(1.0, torch.float16)
    assert round16(1.0 + q / 2, torch.float16) == 1.0 and round16(1.0 + 1.5 * q, torch.float16) == 1.0 + 2 * q
    assert round16(65519.99, torch.float16) == 65504.0 and np.isinf(round16(65520.0, torch.float16))
    assert round16(2.0 ** -25, torch.float16) == 0.0 and round16(1.5 * 2.0 ** -25, torch.float16) == 2.0 ** -24


def test_round16_bfloat16_matches_torch_on_float32_inputs():
    rng = np.random.default_rng(1)
    v = _samples(rng, -140, 127.9).astype(np.float32).astype(np.float64)
    want = torch.from_numpy(v).float().to(torch.bfloat16).double().numpy()
    assert np.array_equal(round16(v, torch.bfloat16), want)
    assert np.isinf(round16(float.fromhex("0x1.ffp127"), torch.bfloat16))


def test_midpoint_distance_is_where_rounding_changes():
    rng = np.random.default_rng(2)
    for dt in (torch.float16, torch.bfloat16):
        v = _samples(rng, -20, 14, 5000)[:-2]
        d = midpoint_distance(v, dt)
        assert (d >= 0).all()
        # moving v by less than d never changes its rounding; moving it by a bit more than d sometimes does
        for f in (0.999, -0.999):
            assert np.array_equal(round16(v + f * d, dt), round16(v, dt))
        assert not np.array_equal(round16(v + 1.001 * d, dt), round16(v, dt))
    # just above a power of two the nearest midpoint is the last one of the binade below
    q = ulp16(1.0, torch.float16)
    assert np.isclose(midpoint_distance(1.0 + q / 16, torch.float16), q / 16 + q / 4)
