"""ORACLE — test infrastructure only (never imported by the product path).

Correct rounding of float64 values to float16 / bfloat16 (round to nearest, ties to even, gradual underflow, overflow
to +-Inf), and the distance of a value to the nearest rounding midpoint. Computed here from the formats' definitions
(IEEE 754-2008 binary16; bfloat16 = the top 16 bits of binary32) rather than through numpy or torch casts, so that no
intermediate float32 rounding can hide a double rounding in what is being tested.

A 16-bit result y computed from a float32 value within e of the exact v equals round16(v) wherever
midpoint_distance(v) > e: no rounding boundary lies between the two.
"""
from __future__ import annotations

import numpy as np

# dtype name -> (explicit significand bits, least normal exponent, largest finite value)
FORMATS = {
    "float16": (10, -14, 65504.0),
    "bfloat16": (7, -126, float.fromhex("0x1.fep127")),
}


def _fmt(dtype) -> tuple:
    return FORMATS[str(dtype).replace("torch.", "")]


def _quantum(v: np.ndarray, dtype) -> np.ndarray:
    """spacing of the 16-bit grid around each |v| (the subnormal spacing below the least normal)"""
    mant, emin, _ = _fmt(dtype)
    _, E = np.frexp(np.abs(v))
    e = np.where(v == 0, emin, np.maximum(E - 1, emin))
    return np.ldexp(1.0, e - mant)


def ulp16(v, dtype) -> np.ndarray:
    """one unit in the last place of the 16-bit format at |v| (float64)"""
    return _quantum(np.asarray(v, np.float64), dtype)


def round16(v, dtype) -> np.ndarray:
    """v (float64) correctly rounded to the 16-bit format, returned as float64; NaN stays NaN"""
    v = np.asarray(v, np.float64)
    _, _, vmax = _fmt(dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        q = _quantum(v, dtype)
        r = np.round(v / q) * q   # v / q is exact (q a power of two); np.round ties to even
        return np.where(np.isfinite(v), np.where(np.abs(r) > vmax, np.copysign(np.inf, v), r), v)


def midpoint_distance(v, dtype) -> np.ndarray:
    """distance of each |v| to the nearest point where rounding to the 16-bit format changes its result: the
    midpoints between neighbours in v's binade and, just above a power of two, the last midpoint of the binade below
    (the overflow threshold max + ulp/2 is such a midpoint)"""
    v = np.abs(np.asarray(v, np.float64))
    mant, emin, _ = _fmt(dtype)
    q = _quantum(v, dtype)
    k = v / q
    d = np.abs(k - (np.floor(k) + 0.5)) * q
    _, E = np.frexp(v)
    base = np.ldexp(1.0, E - 1)   # the power of two at the binade's bottom
    normal = (v != 0) & (E - 1 > emin)
    return np.where(normal, np.minimum(d, v - base + q / 4), d)
