"""Exact reference of b200va_convert_sr_f32 and b200va_quantize_fp8_sr_f32: numpy only, no C.

The contract (include/b200va.h):
  random bits  element i has the global index m = first + i (mod 2^64); key = splitmix64(seed), w_j =
               splitmix64(key + j); r_m is the low 32 bits of w_(m>>1) for even m and the high 32 bits for odd m.
  rounding     y = a (f16/bf16) or a 2^k (FP8).  D is the destination's values, subnormals included, unbounded above.
               lo is the element of D nearest y toward zero, hi the next one away from zero, f = (|y| - |lo|) /
               (|hi| - |lo|) and t = floor(f 2^32); the result is hi if t + r >= 2^32, else lo, with y's sign.
               f16/bf16: past max finite +-inf; FP8: past max finite (+-inf included) +-max finite.  +-0 stays +-0,
               NaN gives NaN (compared as a class).

How this module gets each result: the f32 source widens exactly to f64 and np.ldexp scales it (exact: an f32 value
times 2^k, k in [-126, 126], is an f64 normal or zero).  `round_sr` then splits the f64 significand as
`convert_exact.round_f64` does for round-to-nearest: one shift by the destination's quantum at |y| (fixed below its
normal range, which gives its subnormals), the kept bits being lo and the dropped bits its fractional position.  t is
the dropped bits scaled to 32 bits (at least 42 bits are dropped, since an f64 significand has 53 bits and D at most
11, so t is a right shift).  A round-up adds one to the kept bits; in the encoding (exponent above the minimum times
2^(p-1), plus the kept bits) a carry out of the significand moves into the exponent.  The encoding is then clamped at
the infinity pattern (f16/bf16) or the largest finite pattern (FP8).

f16/bf16 results are uint16 bit patterns and FP8 results uint8 bit patterns, as in stream_exact and fp8_exact.
"""
from __future__ import annotations

import numpy as np

from oracle.convert_exact import QNAN
from oracle.fp8_exact import K_RANGE, SPEC
from oracle.stream_exact import BITS, FORMATS

DESTS = ("f16", "bf16", "e4m3", "e5m2")
_M64 = (1 << 64) - 1


def _params(dst: str) -> tuple[int, int, int, int, np.dtype]:
    """(significand bits incl. the implicit one, minimum normal exponent, the pattern past max finite's place (the
    clamp), the sign bit's position, storage) of a destination."""
    if dst in ("f16", "bf16"):
        prec, emin, _ = FORMATS[dst]
        _, eb, mb = BITS[dst]
        return prec, emin, ((1 << eb) - 1) << mb, eb + mb, np.uint16
    prec, emin, _, _, top, _ = SPEC[dst]
    return prec, emin, top, 7, np.uint8


def splitmix64(z) -> np.ndarray:
    """splitmix64 of uint64 values (mod 2^64), vectorised."""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def random_words(seed: int, first: int, n: int) -> np.ndarray:
    """r_m for m = first + i, i in [0, n): uint32."""
    key = splitmix64(np.uint64(seed & _M64))
    with np.errstate(over="ignore"):
        m = np.uint64(first & _M64) + np.arange(n, dtype=np.uint64)
        w = splitmix64(key + (m >> np.uint64(1)))
    return np.where((m & np.uint64(1)) == 1, w >> np.uint64(32), w & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def _split(a: np.ndarray, dst: str, k: int):
    """y = a 2^k (f64, exact) split at dst's quantum: (y's bit fields sign, E, M, floor(log2 |y|) e, finite nonzero,
    the kept bits q (lo's significand on dst's quantum), t)."""
    assert dst in DESTS and (k == 0 or dst in ("e4m3", "e5m2")) and K_RANGE[0] <= k <= K_RANGE[1]
    prec, emin, _, _, _ = _params(dst)
    x = np.ldexp(np.ascontiguousarray(a, np.float32).astype(np.float64), k)
    u = x.view(np.uint64)
    sign = u >> np.uint64(63)
    E = ((u >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64)
    M = u & np.uint64((1 << 52) - 1)
    sig = np.where(E > 0, M | np.uint64(1 << 52), M)
    exp = np.where(E > 0, E - 1075, -1074)                   # y = sig * 2^exp
    with np.errstate(all="ignore"):
        e = np.frexp(x)[1].astype(np.int64) - 1               # floor(log2 |y|) for finite nonzero y
    finite_nz = (E < 0x7FF) & (sig != 0)
    shift = np.maximum(e, emin) - (prec - 1) - exp            # the dropped low bits of sig: at least 53 - 11
    assert (shift[finite_nz] >= 42).all()
    shift = np.clip(shift, 42, 96).astype(np.uint64)
    big = shift >= 64                                         # everything is dropped: lo = 0
    q = np.where(big, np.uint64(0), sig >> np.minimum(shift, np.uint64(63)))
    rem = np.where(big, sig, sig & ((np.uint64(1) << np.minimum(shift, np.uint64(63))) - np.uint64(1)))
    t = np.where(finite_nz, rem >> np.minimum(shift - np.uint64(32), np.uint64(63)), np.uint64(0))
    return sign, E, M, e, finite_nz, q, t


def threshold_t(a: np.ndarray, dst: str, k: int = 0) -> np.ndarray:
    """t = floor(f 2^32) per element, 0 where y is zero or not finite (uint64): r >= 2^32 - t rounds up."""
    return _split(a, dst, k)[6]


def round_sr(a: np.ndarray, dst: str, r: np.ndarray, k: int = 0) -> np.ndarray:
    """f32 values a (times 2^k for FP8) rounded stochastically to dst with the 32-bit words r: dst bit patterns."""
    prec, emin, clamp, sbit, ut = _params(dst)
    sign, E, M, e, finite_nz, q, t = _split(a, dst, k)
    r = np.ascontiguousarray(r, np.uint32).astype(np.uint64)
    assert r.shape == t.shape
    q = q + ((t + r) >= np.uint64(1 << 32)).astype(np.uint64)
    mag = (np.maximum(e, emin) - emin).astype(np.uint64) * np.uint64(1 << (prec - 1)) + q
    mag = np.minimum(np.where(finite_nz, mag, 0), np.uint64(clamp))
    nan = QNAN[dst] if dst in QNAN else SPEC[dst][5]
    mag = np.where(E == 0x7FF, np.where(M == 0, np.uint64(clamp), np.uint64(nan)), mag)
    return ((sign << np.uint64(sbit)) | mag).astype(ut)


def convert_sr(a: np.ndarray, dst: str, seed: int, first: int = 0) -> np.ndarray:
    """The contract's result of b200va_convert_sr_f32 (dst "f16" or "bf16"): uint16 patterns."""
    assert dst in ("f16", "bf16")
    a = np.ascontiguousarray(a, np.float32)
    return round_sr(a, dst, random_words(seed, first, a.size).reshape(a.shape))


def quantize_fp8_sr(a: np.ndarray, fmt: str, seed: int, first: int = 0, k: int = 0) -> np.ndarray:
    """The contract's result of b200va_quantize_fp8_sr_f32 (fmt "e4m3" or "e5m2", scale 2^k): uint8 patterns."""
    assert fmt in ("e4m3", "e5m2")
    a = np.ascontiguousarray(a, np.float32)
    return round_sr(a, fmt, random_words(seed, first, a.size).reshape(a.shape), k)
