"""Exact reference of b200va_quantize_fp8 and b200va_dequantize_fp8: numpy and `fractions` only, no C.

The contract (include/b200va.h):
  quantize    c = sat(RN(a 2^k)): the exact product rounded once to the FP8 format (ties to even, the format's
              subnormals, no FTZ), saturating at +-max finite (values that round past it and +-inf included); NaN
              gives NaN (compared as a class); +-0 and values that round to zero keep their sign.
  dequantize  c = a 2^-k rounded once to the destination by b200va_convert's rules.
  amax        max |a_i| over the unscaled source values widened to f64, NaN if any is NaN.

How this module gets each result: the source widens exactly to f64 (`stream_exact.widen`) and np.ldexp scales it
(exact, except where f64 itself under- or overflows, which happens only far below half the smallest FP8 subnormal
or far above the largest finite value, where the result is +-0 or saturates either way).  `round_fp8` then rounds
f64 bit patterns in the manner of `convert_exact.round_f64`: one shift of the significand, the dropped bits
compared with half a unit in the last place, ties to even, a carry out of the significand moving into the
exponent; the quantum is fixed below the normal range, which gives the subnormals; the encoding is clamped at the
largest finite pattern.  Dequantize looks the 256 patterns up in a decode table, scales by 2^-k (exact in f64)
and rounds with `convert_exact.round_f64`.

FP8 arrays are uint8 bit patterns; f16/bf16 arrays are uint16 bit patterns, as in stream_exact.
"""
from __future__ import annotations

import bisect
from fractions import Fraction

import numpy as np

from oracle.convert_exact import round_f64
from oracle.stream_exact import STORAGE, widen

FORMATS8 = ("e4m3", "e5m2")
# (significand bits incl. the implicit one, minimum normal exponent, exponent bits, mantissa bits, largest finite
# pattern, the NaN pattern this module writes)
SPEC = {"e4m3": (4, -6, 4, 3, 0x7E, 0x7F), "e5m2": (3, -14, 5, 2, 0x7B, 0x7F)}
MAX_FINITE = {"e4m3": 448.0, "e5m2": 57344.0}
K_RANGE = (-126, 126)


def _decode(fmt: str) -> np.ndarray:
    """The f64 value of each of the 256 patterns, from the format's definition."""
    prec, emin, eb, mb, _, _ = SPEC[fmt]
    bias = 1 - emin
    out = np.empty(256, np.float64)
    for p in range(256):
        s, e, m = p >> 7, (p >> mb) & ((1 << eb) - 1), p & ((1 << mb) - 1)
        if fmt == "e4m3" and e == 15 and m == 7:
            v = float("nan")
        elif fmt == "e5m2" and e == 31:
            v = float("inf") if m == 0 else float("nan")
        elif e == 0:
            v = m * 2.0 ** (emin - mb)
        else:
            v = (1 + m / (1 << mb)) * 2.0 ** (e - bias)
        out[p] = -v if s else v
    return out


DECODE = {f: _decode(f) for f in FORMATS8}


def round_fp8(x: np.ndarray, fmt: str) -> np.ndarray:
    """f64 values rounded once (RNE) to fmt, saturating at +-max finite: uint8 patterns."""
    prec, emin, eb, mb, top, qnan = SPEC[fmt]
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
    # the biased encoding: a large e gives a huge mag, which the clamp saturates (no overflow: e <= 1023)
    mag = (np.maximum(e, emin) - emin).astype(np.uint64) * np.uint64(1 << (prec - 1)) + q
    mag = np.minimum(np.where(finite_nz, mag, 0), np.uint64(top))
    mag = np.where(E == 0x7FF, np.where(M == 0, np.uint64(top), np.uint64(qnan)), mag)
    return ((sign << np.uint64(7)) | mag).astype(np.uint8)


def quantize(a: np.ndarray, src: str, fmt: str, k: int = 0) -> np.ndarray:
    """The contract's result of quantizing a (src storage) to fmt with scale 2^k: uint8 patterns."""
    assert K_RANGE[0] <= k <= K_RANGE[1]
    a = np.ascontiguousarray(a)
    assert a.dtype == STORAGE[src], (a.dtype, src)
    with np.errstate(all="ignore"):
        return round_fp8(np.ldexp(widen(a, src), k), fmt)


def dequantize(bits: np.ndarray, fmt: str, dst: str, k: int = 0) -> np.ndarray:
    """The contract's result of dequantizing uint8 patterns of fmt to dst with scale 2^-k, in dst storage."""
    assert K_RANGE[0] <= k <= K_RANGE[1]
    x = np.ldexp(DECODE[fmt][np.asarray(bits, np.uint8)], -k)    # exact: FP8 values times 2^+-126 are f64 normals
    return x if dst == "f64" else round_f64(x, dst)


def amax(a: np.ndarray, src: str, acc: float = 0.0) -> float:
    """max(acc, max_i |a_i|) over the unscaled values widened to f64; NaN if any of them (or acc) is NaN."""
    x = np.abs(widen(a, src))
    if np.isnan(x).any() or np.isnan(acc):
        return float("nan")
    return max(acc, float(x.max())) if x.size else acc


# ------------------------------------------------------------------------------------------- inputs
def values(fmt: str) -> np.ndarray:
    """The finite non-negative values of fmt in increasing order."""
    v = DECODE[fmt][:128]
    return np.sort(v[np.isfinite(v)])


def midpoints(fmt: str) -> np.ndarray:
    """Every midpoint between neighbouring non-negative finite values, and the saturation threshold
    (max finite + half an ulp)."""
    v = values(fmt)
    ulp_top = v[-1] - v[-2]
    return np.concatenate([(v[:-1] + v[1:]) / 2, [v[-1] + ulp_top / 2]])


def adversarial(fmt: str, rel: float = 2.0 ** -40) -> dict:
    """{name: f64 values of the scaled product a 2^k, both signs}: where a quantize kernel that rounds wrongly,
    rounds twice, saturates wrongly or loses a sign differs from the contract.  `rel`: the relative offset of the
    values on either side of a midpoint (2^-40 for f64 sources, which an RN conversion to f32 puts onto it)."""
    v, m = values(fmt), midpoints(fmt)
    sat = m[-1]
    tiny = v[1] / 2                                           # half the smallest subnormal
    sets = {
        "midpoints": m,
        "midpoints, just above": m * (1 + rel),
        "midpoints, just below": m * (1 - rel),
        "values": v,
        "saturation threshold": np.array([sat, sat * (1 + rel), sat * (1 - rel), v[-1], 2 * v[-1], 1e300]),
        "half the smallest subnormal": np.array([tiny, tiny * (1 + rel), tiny * (1 - rel), tiny / 2, 3 * tiny]),
        "zeros, infinities and NaN": np.array([0.0, np.inf, np.nan]),
    }
    return {k: np.concatenate([x, -x]) for k, x in sets.items()}


def double_rounding_traps(fmt: str) -> np.ndarray:
    """f64 values a relative 2^-40 off every midpoint (the saturation threshold included), both signs: an RN
    conversion to f32 puts each one onto the midpoint, after which RN to FP8 ties to even, while one rounding
    goes toward the side the value lies on."""
    m = midpoints(fmt)
    x = np.concatenate([m * (1 + 2.0 ** -40), m * (1 - 2.0 ** -40)])
    return np.concatenate([x, -x])


def source_values(x: np.ndarray, src: str, k: int) -> np.ndarray:
    """Products x (f64) as source values a = x 2^-k in src storage (rounded to src where it cannot hold them)."""
    with np.errstate(all="ignore"):
        a = np.ldexp(np.asarray(x, np.float64), -k)
        if src == "f64":
            return a
        if src == "f32":
            return a.astype(np.float32)
        return round_f64(a, src)


# ------------------------------------------------------------------------------------------- Fraction cross-check
_TABLE = {f: [Fraction(y) for y in values(f).tolist()] for f in FORMATS8}


def nearest_fraction(x: Fraction, fmt: str) -> float:
    """The finite fmt value nearest to the rational x, searched in the table of finite values: of the two values
    around |x| the nearer, a tie to the even significand (the i-th non-negative value has pattern i, so an even i),
    and the largest finite value beyond it (saturation).  The result carries x's sign."""
    t = _TABLE[fmt]
    mag = abs(x)
    i = bisect.bisect_left(t, mag)
    if i == len(t):
        r = i - 1
    elif t[i] == mag or i == 0:
        r = i
    else:
        lo, hi = mag - t[i - 1], t[i] - mag
        r = i - 1 if lo < hi or (lo == hi and (i - 1) % 2 == 0) else i
    v = float(t[r])
    return -v if x < 0 else v
