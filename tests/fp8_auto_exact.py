"""Exact reference of b200va_quantize_fp8_auto and b200va_dequantize_fp8_auto (include/b200va.h), built on the
per-tensor reference in oracle/fp8_exact.py: numpy and Python floats only, no C, no torch.

The contract:
  amax pass   *d_amax = the larger, as unsigned 64-bit patterns, of *d_amax and M, M the largest finite |a_i| widened
              to f64 (+0.0 when there is none): max(acc, M) for acc = +0.0 or a positive finite value; a NaN, +inf or a
              value with the sign bit set in acc stays.
  scale       k = clamp(K(m) - margin, -126, 126) for the m the amax pass left, K(m) the largest integer k with
              m 2^k <= max finite (448 / 57344) and K(0) = +inf; k = 0 when m is not +0.0 or a positive finite value.
  quantize    fp8_exact.quantize with that k.
  dequantize  fp8_exact.dequantize with the k in *d_scale_exp; a k outside [-126, 126] makes every element a NaN.

K(m) is taken here from frexp (floor(log2 m) for every positive finite m, subnormals included) and the exact
significand, not from the bit fields the kernel reads; the CPU tests check it against a search in `Fraction`.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import fp8_exact as F
from oracle.convert_exact import QNAN
from oracle.stream_exact import STORAGE, widen

EMAX = {"e4m3": 8, "e5m2": 15}          # max finite = 1.75 2^emax
MARGIN_RANGE = (0, 126)


def f64_bits(x: float) -> int:
    return int(np.float64(x).view(np.uint64))


def f64_from_bits(b: int) -> float:
    return float(np.uint64(b).view(np.float64))


def finite_amax(a: np.ndarray, src: str, acc: float = 0.0) -> float:
    """The amax pass: acc max-accumulated with the largest finite |a_i| (NaN and +-inf do not take part), the maximum
    taken on the f64 bit patterns as unsigned integers."""
    x = np.abs(widen(a, src))
    x = x[np.isfinite(x)]
    m = float(x.max()) if x.size else 0.0
    return f64_from_bits(max(f64_bits(acc), f64_bits(m)))


def auto_scale_exp(m: float, fmt: str, margin: int) -> int:
    """The scale exponent chosen from the amax m."""
    assert MARGIN_RANGE[0] <= margin <= MARGIN_RANGE[1]
    if f64_bits(m) >= 0x7FF0000000000000:            # NaN, +inf, or the sign bit set
        return 0
    if m == 0:
        return F.K_RANGE[1]                          # K(0) = +inf
    s, e = math.frexp(m)                             # m = s 2^e, s in [0.5, 1): floor(log2 m) = e - 1
    K = EMAX[fmt] - (e - 1) - (2 * s > 1.75)
    return min(max(K - margin, F.K_RANGE[0]), F.K_RANGE[1])


def quantize_auto(a: np.ndarray, src: str, fmt: str, margin: int = 0, acc: float = 0.0):
    """(FP8 bit patterns, k, the amax left in *d_amax) of b200va_quantize_fp8_auto on a with *d_amax = acc."""
    m = finite_amax(a, src, acc)
    k = auto_scale_exp(m, fmt, margin)
    return F.quantize(a, src, fmt, k), k, m


def dequantize_auto(bits: np.ndarray, fmt: str, dst: str, k: int) -> np.ndarray:
    """b200va_dequantize_fp8_auto with k in *d_scale_exp, in dst storage."""
    if F.K_RANGE[0] <= k <= F.K_RANGE[1]:
        return F.dequantize(bits, fmt, dst, k)
    nan = np.nan if dst in ("f32", "f64") else QNAN[dst]
    return np.full(np.asarray(bits).size, nan, STORAGE[dst])
