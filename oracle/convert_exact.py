"""Exact reference of b200va_convert: numpy and `fractions` only, no C.

The contract (include/b200va.h): c = a rounded once to the destination type, IEEE round-to-nearest-even as if
the exponent range were unbounded, then overflow to +-inf; no FTZ on either side; +-0 and +-inf kept; a NaN gives
a NaN (compared as a class).  The same type is a bit copy.

How this module gets each result: every source value widens exactly to f64 (`stream_exact.widen`), and `round_f64`
rounds f64 bit patterns to the destination with integer arithmetic on the significand: one shift, the dropped
bits compared with half a unit in the last place, ties to even, and an encoding in which a carry out of the
significand moves into the exponent, up to the infinity pattern.  The destination's quantum is fixed below its
normal range, which gives its subnormals.  Widening to f64 is exact, so the result is the value rounded once.

f16/bf16 arrays are uint16 bit patterns, as in stream_exact.
"""
from __future__ import annotations

import numpy as np

from oracle.stream_exact import BITS, FORMATS, STORAGE, widen

DTYPES = ("f32", "f64", "f16", "bf16")
SIZE = {"f32": 4, "f64": 8, "f16": 2, "bf16": 2}
PAIRS = [(s, d) for s in DTYPES for d in DTYPES if s != d]
QNAN = {"f16": 0x7E00, "bf16": 0x7FC0, "f32": 0x7FC00000}


def round_f64(x: np.ndarray, dst: str) -> np.ndarray:
    """f64 values rounded once (RNE) to dst in {f32, f16, bf16}, as dst storage (f32 values, uint16 patterns)."""
    prec, emin, emax = FORMATS[dst]
    ut, eb, mb = BITS[dst]
    x = np.ascontiguousarray(x, np.float64)
    u = x.view(np.uint64)
    sign = (u >> np.uint64(63)).astype(np.uint64)
    E = ((u >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64)
    M = u & np.uint64((1 << 52) - 1)
    sig = np.where(E > 0, M | np.uint64(1 << 52), M)
    exp = np.where(E > 0, E - 1075, -1074)                   # x = sig * 2^exp
    with np.errstate(all="ignore"):
        e = np.frexp(x)[1].astype(np.int64) - 1               # floor(log2 |x|) for finite nonzero x
    finite_nz = (E < 0x7FF) & (sig != 0)
    shift = np.maximum(e, emin) - (prec - 1) - exp            # the dropped low bits of sig
    assert (shift[finite_nz] >= 1).all()
    shift = np.clip(shift, 1, 54).astype(np.uint64)           # >= 54: sig < half an ulp, the result is 0
    q = sig >> shift
    rem = sig & ((np.uint64(1) << shift) - np.uint64(1))
    half = np.uint64(1) << (shift - np.uint64(1))
    q = q + ((rem > half) | ((rem == half) & ((q & np.uint64(1)) == 1))).astype(np.uint64)
    mag = (np.maximum(e, emin) - emin).astype(np.uint64) * np.uint64(1 << (prec - 1)) + q
    inf = np.uint64(((1 << eb) - 1) << mb)
    mag = np.minimum(np.where(finite_nz, mag, 0), inf)        # from the overflow threshold on: inf
    mag = np.where(E == 0x7FF, np.where(M == 0, inf, np.uint64(QNAN[dst])), mag)
    out = ((sign << np.uint64(eb + mb)) | mag).astype(ut)
    return out.view(np.float32) if dst == "f32" else out


def convert(a: np.ndarray, src: str, dst: str) -> np.ndarray:
    """The contract's result of converting a (src storage) to dst, in dst storage."""
    a = np.ascontiguousarray(a)
    assert a.dtype == STORAGE[src], (a.dtype, src)
    if src == dst:
        return a.copy()
    x = widen(a, src)
    return x if dst == "f64" else round_f64(x, dst)


# ------------------------------------------------------------------------------------------- inputs
def from_bits(bits: np.ndarray, dtype: str) -> np.ndarray:
    """Bit patterns (any unsigned ints) as dtype storage."""
    ut = BITS[dtype][0]
    b = np.asarray(bits).astype(ut)
    return b if dtype in ("f16", "bf16") else b.view(STORAGE[dtype])


def random_bits(dtype: str, n: int, rng) -> np.ndarray:
    """Uniformly random bit patterns: every class of value, NaNs included."""
    ut = BITS[dtype][0]
    return from_bits(rng.integers(0, np.iinfo(ut).max, n, dtype=np.uint64, endpoint=True), dtype)


def rounding_patterns(src: str, dst: str, highs: np.ndarray | None = None) -> np.ndarray:
    """For an f32 or f64 source narrowed to dst: each high part of the source pattern (the bits dst keeps in its
    normal range, sign and exponent included; all of them unless `highs` is given) joined with the low parts that
    decide the rounding there: 0, 1, half - 1, half, half + 1 and all ones."""
    _, eb, mb = BITS[src]
    drop = mb - FORMATS[dst][0] + 1
    half = 1 << (drop - 1)
    lows = np.array([0, 1, half - 1, half, half + 1, (1 << drop) - 1], np.uint64)
    if highs is None:
        highs = np.arange(1 << (1 + eb + mb - drop), dtype=np.uint64)
    return from_bits(((highs.astype(np.uint64)[:, None] << np.uint64(drop)) | lows[None, :]).ravel(), src)


def double_rounding_traps(dst: str, n: int = 4096, seed: int = 0) -> np.ndarray:
    """f64 values just off a dst midpoint M, by a relative 2^-40 of either sign: f32 rounds them onto M, after which
    the tie goes to even, while one rounding goes toward the side they lie on.  M runs over the normal binades, the
    subnormal range and the overflow midpoint above the largest finite value."""
    prec, emin, emax = FORMATS[dst]
    rng = np.random.default_rng(seed)
    E = rng.integers(emin - prec + 1, emax + 1, n)              # the exponent of M's ulp's binade (subnormal below emin)
    E[:8] = emax
    m = rng.integers(1 << (prec - 1), 1 << prec, n)             # the lower neighbour's significand
    m[:8] = (1 << prec) - 1                                     # the largest finite value: M is the overflow midpoint
    sub = E < emin
    m = np.where(sub, rng.integers(0, 1 << (prec - 1), n), m)   # below the normal range: a subnormal significand
    q = np.exp2((np.maximum(E, emin) - prec + 1).astype(np.float64))
    M = (m + 0.5) * q
    sigma = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    sigma[:8] = -1.0                                            # just below the overflow midpoint: finite, through f32 inf
    x = M * (1 + sigma * 2.0 ** -40)
    return np.where(rng.random(n) < 0.5, -x, x)
