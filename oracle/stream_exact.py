"""Exact reference of b200va_stream, independent of vadd_oracle.c: numpy and `fractions` only, no C.

The contract (include/b200va.h, csrc/b200va_stream.cuh):
  COPY c = a (the input bits)   SCALE c = s*a   ADD c = a + b   TRIAD c = fma(s, b, a), one rounding.
  f32, f16, bf16: the operands widen exactly to f32, s is rounded to f32, the op is rounded once to f32 (RNE) and
  the f32 result is rounded to the storage type (RNE).  f16/bf16 TRIAD therefore rounds twice.
  f64: computed natively with the double s as given, RNE.

How this module gets each result without restating that arithmetic:
  f32 family: every operand widens exactly to f64 and p = f32(s)*b is exact in f64 (at most 48 significant bits,
  and the product of two f32 subnormals is still an f64 normal).  hi = a + p and its TwoSum error lo represent the
  exact sum; hi + lo is rounded to f32 once.  Rounding hi alone is right except where hi is exactly an f32 midpoint
  (lo breaks the tie) and where hi is exactly the binary32 overflow threshold FLT_MAX + ulp/2 (lo < 0 keeps FLT_MAX).
  f16 uses numpy's float32 -> float16 cast (RNE); bf16 is rounded with integer RNE here.
  f64: numpy's add and multiply are correctly rounded; TRIAD is Fraction(a) + Fraction(s)*Fraction(b) converted
  with float(), which rounds correctly -- slow, so limited to FRACTION_LIMIT elements per call.

`adversarial` builds the inputs where a plausible kernel bug shows, shared by the CPU and the GPU tests.
f16/bf16 arrays are uint16 bit patterns, as in oracle.stream.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

FRACTION_LIMIT = 200_000
FLT_MAX = float(np.finfo(np.float32).max)
F32_OVERFLOW = float(2 ** 128 - 2 ** 103)          # FLT_MAX + ulp/2: from here on RNE gives inf
F64_OVERFLOW = Fraction(2 ** 1024 - 2 ** 970)      # DBL_MAX + ulp/2
# (significand bits incl. the implicit one, minimum normal exponent, maximum exponent)
FORMATS = {"f16": (11, -14, 15), "bf16": (8, -126, 127), "f32": (24, -126, 127), "f64": (53, -1022, 1023)}
BITS = {"f16": (np.uint16, 5, 10), "bf16": (np.uint16, 8, 7), "f32": (np.uint32, 8, 23), "f64": (np.uint64, 11, 52)}
STORAGE = {"f32": np.float32, "f64": np.float64, "f16": np.uint16, "bf16": np.uint16}


# ------------------------------------------------------------------------------------------- conversions
def widen(x: np.ndarray, dtype: str) -> np.ndarray:
    """Storage values (bit patterns for f16/bf16) as exact f64."""
    x = np.ascontiguousarray(x)
    with np.errstate(all="ignore"):                  # signalling NaNs stay NaNs
        if dtype == "f16":
            return x.view(np.float16).astype(np.float64)
        if dtype == "bf16":
            return (x.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        return x.astype(np.float64)


def narrow(r: np.ndarray, dtype: str) -> np.ndarray:
    """f32 values rounded to nearest-even into the storage type."""
    r = np.ascontiguousarray(r, np.float32)
    if dtype == "f32":
        return r
    if dtype == "f16":
        with np.errstate(all="ignore"):
            return r.astype(np.float16).view(np.uint16)
    u = r.view(np.uint32)
    keep, rest = u >> 16, u & 0xFFFF
    up = (rest > 0x8000) | ((rest == 0x8000) & ((keep & 1) == 1))
    h = keep + up                                    # a carry moves into the exponent, up to inf
    return np.where((u & 0x7FFFFFFF) > 0x7F800000, keep | 0x7FC0, h).astype(np.uint16)


def round_f32(hi: np.ndarray, lo: np.ndarray) -> np.ndarray:
    """hi + lo rounded once to f32 (RNE), for hi = fl64(hi + lo) and lo its exact error."""
    hi, lo = np.asarray(hi, np.float64), np.asarray(lo, np.float64)
    with np.errstate(all="ignore"):
        r = hi.astype(np.float32)
        r64 = r.astype(np.float64)
        fin = np.isfinite(r64)
        d = np.where(fin, hi - r64, 0.0)             # exact: r is within half an f32 ulp of hi
        nb = np.where(d > 0, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf)))
        gap = np.abs(nb.astype(np.float64) - r64)    # inf beyond FLT_MAX: never a tie there
        tie = fin & (d != 0) & (2 * np.abs(d) == gap) & (np.sign(lo) == np.sign(d))
        r = np.where(tie, nb, r)
        # hi exactly on the overflow threshold rounds to inf (FLT_MAX is odd); an exact sum below it is FLT_MAX
        under = np.isfinite(hi) & (np.abs(hi) == F32_OVERFLOW) & (np.sign(lo) == -np.sign(hi))
        return np.where(under, np.copysign(np.float32(FLT_MAX), hi), r).astype(np.float32)


def round_fraction(x: Fraction, dtype: str) -> float:
    """The dtype value nearest to the nonzero rational x (ties to even; inf from the overflow threshold on), as a
    Python float.  Written from the format's definition, for cross-checks."""
    prec, emin, emax = FORMATS[dtype]
    assert x != 0
    sign, x = (-1.0 if x < 0 else 1.0), abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    while Fraction(2) ** e > x:
        e -= 1
    while Fraction(2) ** (e + 1) <= x:
        e += 1
    q = Fraction(2) ** (max(e, emin) - prec + 1)     # the spacing at x (fixed below the normal range)
    m = x / q
    f, rem = divmod(m.numerator, m.denominator)
    if 2 * rem > m.denominator or (2 * rem == m.denominator and f & 1):
        f += 1
    v = f * q
    return sign * float("inf") if v >= Fraction(2) ** (emax + 1) else sign * float(v)


def _fraction_fma64(a: float, b: float, s: float) -> float:
    """fma(s, b, a) for doubles, through the exact rational."""
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(s)):
        if np.isfinite(s) and np.isfinite(b):
            return a                                 # a finite product added to inf or NaN
        return s * b + a                             # the product is inf or NaN already
    x = Fraction(a) + Fraction(s) * Fraction(b)
    if x == 0:
        return (s * b) + a if a == 0 and s * b == 0 else 0.0   # signed zeros follow IEEE; cancellation is +0
    if abs(x) >= F64_OVERFLOW:
        return float("inf") if x > 0 else float("-inf")
    return float(x)


# ------------------------------------------------------------------------------------------- the reference
def stream(op: str, dtype: str, a: np.ndarray, b: np.ndarray | None, s: float = 0.0) -> np.ndarray:
    """The contract's result of op over dtype, in the storage format."""
    a = np.ascontiguousarray(a)
    assert a.dtype == STORAGE[dtype], (a.dtype, dtype)
    if op == "copy":
        return a.copy()
    if op in ("add", "triad"):
        b = np.ascontiguousarray(b)
        assert b.dtype == a.dtype and b.size == a.size
    if dtype == "f64":
        with np.errstate(all="ignore"):
            if op == "scale":
                return np.float64(s) * a
            if op == "add":
                return a + b
        assert a.size <= FRACTION_LIMIT, "f64 triad through Fraction: use a sample"
        return np.array([_fraction_fma64(x, y, float(s)) for x, y in zip(a.tolist(), b.tolist())], np.float64)
    A, S = widen(a, dtype), np.float64(f32_scalar(s))
    with np.errstate(all="ignore"):
        if op == "scale":
            r = (S * A).astype(np.float32)           # the product is exact: one rounding
        else:
            p = widen(b, dtype) if op == "add" else S * widen(b, dtype)
            hi = A + p
            bb = hi - A
            lo = (A - (hi - bb)) + (p - bb)          # TwoSum
            r = round_f32(hi, lo)
    return narrow(r, dtype)


def f32_scalar(s: float) -> float:
    """s rounded to f32 (RNE, inf from the overflow threshold on), as the f32/f16/bf16 ops use it."""
    with np.errstate(all="ignore"):
        return float(np.float32(s))


# ------------------------------------------------------------------------------------------- adversarial inputs
def _bits(dtype, sign, exp, man):
    ut, eb, mb = BITS[dtype]
    return ((sign.astype(np.uint64) << np.uint64(eb + mb)) | (exp.astype(np.uint64) << np.uint64(mb))
            | man.astype(np.uint64)).astype(ut).view(STORAGE[dtype])


def finite(dtype: str, n: int, rng, scale: float = 4.0) -> np.ndarray:
    """Normally distributed values rounded to the storage type."""
    x = rng.standard_normal(n) * scale
    return narrow(x.astype(np.float32), dtype) if dtype in ("f16", "bf16") else x.astype(STORAGE[dtype])


def negate(x: np.ndarray, dtype: str) -> np.ndarray:
    return x ^ np.uint16(0x8000) if dtype in ("f16", "bf16") else -x


def _tiny(dtype, n, rng):
    """The smallest normals (exponent field 1..6): scaled by s < 1 they round into the subnormals."""
    _, eb, mb = BITS[dtype]
    return _bits(dtype, rng.integers(0, 2, n), rng.integers(1, 7, n), rng.integers(0, 1 << mb, n, dtype=np.uint64))


def nan_payloads(dtype: str, n: int, seed: int = 0) -> np.ndarray:
    """Random bit patterns, a third of them NaNs with random payloads: quiet and signalling, both signs."""
    ut, eb, mb = BITS[dtype]
    rng = np.random.default_rng(seed)
    x = rng.integers(0, np.iinfo(ut).max, n, dtype=np.uint64, endpoint=True).astype(ut)
    k = n // 3
    man = rng.integers(1, 1 << mb, k, dtype=np.uint64)
    man[::2] &= np.uint64((1 << (mb - 1)) - 1)       # quiet bit clear: signalling (payload != 0)
    man[man == 0] = 1
    x[:k] = _bits(dtype, rng.integers(0, 2, k), np.full(k, (1 << eb) - 1), man).view(ut)
    return x.view(STORAGE[dtype])


def edge_values(dtype: str, n: int, seed: int = 0) -> np.ndarray:
    """Operands near both ends of the range: zeros, subnormals, the smallest normals, the largest finite values,
    inf and NaN, each sign."""
    _, eb, mb = BITS[dtype]
    rng = np.random.default_rng(seed)
    top = (1 << eb) - 2
    exps = np.array([0, 0, 1, 2, 3, mb // 2, top - 2, top - 1, top, top, top + 1], np.uint64)
    exp = exps[rng.integers(0, exps.size, n)]
    man = rng.integers(0, 1 << mb, n, dtype=np.uint64)
    man[rng.random(n) < 0.08] = 0                    # exact zeros, powers of two and infinities
    man[rng.random(n) < 0.05] = (1 << mb) - 1        # the largest significand of a binade
    return _bits(dtype, rng.integers(0, 2, n), exp, man)


def _signed_zero_pairs(dtype, rng, n):
    """a + b == 0 exactly: (+-0, +-0) in all four combinations and x + (-x)."""
    z = narrow(np.array([0.0, -0.0], np.float32), dtype) if dtype != "f64" else np.array([0.0, -0.0])
    x = finite(dtype, n, rng)
    return np.concatenate([np.repeat(z, 2), x, negate(x, dtype)]), np.concatenate([np.tile(z, 2), negate(x, dtype), x])


def _cancellation(dtype, s, rng, n):
    """a = -fl(f32(s)*b) (f64: -fl(s*b)): a fused TRIAD returns the rounding error of the product, an unfused one
    returns 0 (or, for f16/bf16, where a is the product rounded to the storage type, a different small value)."""
    b = finite(dtype, n, rng)
    if dtype == "f64":
        return -(np.float64(s) * b), b
    p = np.float32(f32_scalar(s)) * widen(b, dtype).astype(np.float32)      # numpy's f32 product: one rounding
    return narrow(-p, dtype), b


def _half_midpoints(dtype, sigma, rng, n):
    """f16/bf16 TRIAD inputs whose exact result is a storage-type midpoint M plus a tiny nonzero t of sign sigma:
    f32 rounds a + s*b to M exactly, the narrowing then ties to even, and a single rounding of a + s*b would go
    toward t.  With s = 1 + sigma 2^-22, b = (2k+1) 2^(E-p) (an odd number of half ulps at exponent E) and a an
    exponent-E value of p bits: a + b = M and t = sigma 2^-22 b, below half an f32 ulp of M.  E runs over the whole
    normal range, including the midpoint above the largest finite value, which rounds to inf."""
    prec, emin, emax = FORMATS[dtype]
    s = 1.0 + sigma * 2.0 ** -22
    E = rng.integers(emin + 1, emax + 1, n)
    E[: min(n, 8)] = emax
    m = rng.integers(1 << (prec - 1), 1 << prec, n)
    m[: min(n, 8)] = (1 << prec) - 1                  # a = the largest finite value: M is the overflow midpoint
    k = rng.integers(0, 1 << (prec - 3), n)
    k = np.minimum(k, (1 << prec) - 1 - m)           # a + b stays in a's binade
    sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    a = sign * m * np.exp2((E - prec + 1).astype(np.float64))
    b = sign * (2 * k + 1) * np.exp2((E - prec).astype(np.float64))
    return s, narrow(a.astype(np.float32), dtype), narrow(b.astype(np.float32), dtype)


def _f32_overflow_ties():
    """f32 TRIAD/ADD at and across the overflow threshold T = FLT_MAX + 2^103, with the f64 sum landing exactly on T
    and the TwoSum error of either sign: (s, a, b) per case, both signs."""
    cases = [
        (1.0 + 2.0 ** -10, FLT_MAX, 1047553.0 * 2.0 ** 83),        # s*b = 2^103 + 2^73: exact T + 2^73 -> inf
        (1.0 + 2.0 ** -15, FLT_MAX, 2.0 ** 103 * (1 - 2.0 ** -15)),  # s*b = 2^103 - 2^73: exact T - 2^73 -> FLT_MAX
        (1.0, FLT_MAX, 2.0 ** 103),                                 # exactly T: the tie goes to inf
        (1.0, FLT_MAX, 2.0 ** 103 * (1 - 2.0 ** -24)),              # just below T: FLT_MAX
        (1.0, FLT_MAX, 2.0 ** 103 * (1 + 2.0 ** -23)),              # just above T: inf
        (2.0, 2.0 ** 127, 2.0 ** 126),                              # far beyond
    ]
    out = []
    for s, a, b in cases:
        out.append((s, np.array([a, -a], np.float32), np.array([b, -b], np.float32)))
    return out


def adversarial(op: str, dtype: str, seed: int = 0, n: int = 4096) -> list[tuple[str, float, np.ndarray, np.ndarray]]:
    """[(name, s, a, b)]: the inputs of `op` over `dtype` where a subtly wrong kernel differs from the contract."""
    rng = np.random.default_rng([seed, list(BITS).index(dtype), ["copy", "scale", "add", "triad"].index(op)])
    if op == "copy":
        return [("nan payloads", 0.0, nan_payloads(dtype, n, seed), nan_payloads(dtype, n, seed + 1))]
    sets = []
    ea, eb = edge_values(dtype, n, seed), edge_values(dtype, n, seed + 1)
    for s in ((0.5, 2.0 ** -10, 3.0, -1.5, 1.0 + 2.0 ** -23) if op != "add" else (0.0,)):
        sets.append((f"edges s={s!r}", s, ea, eb))
    if op in ("add", "triad"):
        za, zb = _signed_zero_pairs(dtype, rng, n // 4)
        sets.append(("signed zeros", 1.0, za, zb))
    if op == "scale":
        sets.append(("signed zeros", -0.0, ea, eb))
    if op in ("scale", "triad"):
        for s in (0.1, -1.0 / 3.0):
            sets.append((f"into subnormals s={s!r}", s, _tiny(dtype, n, rng), _tiny(dtype, n, rng)))
    if op == "triad":
        for s in (0.1, -1.0 / 3.0, 1.0 + 2.0 ** -23 if dtype != "f64" else 1.0 + 2.0 ** -52):
            a, b = _cancellation(dtype, s, rng, n)
            sets.append((f"fma cancellation s={s!r}", s, a, b))
        if dtype in ("f16", "bf16"):
            for sigma in (1, -1):
                s, a, b = _half_midpoints(dtype, sigma, rng, n)
                sets.append((f"storage midpoints s={s!r}", s, a, b))
    if dtype == "f32" and op in ("add", "triad"):
        for i, (s, a, b) in enumerate(_f32_overflow_ties()):
            if op == "triad" or s == 1.0:
                sets.append((f"overflow threshold {i}", s, a, b))
    if dtype == "f64" and op in ("add", "triad"):
        dmax = np.finfo(np.float64).max
        a = np.array([dmax, -dmax, dmax, -dmax], np.float64)
        b = np.array([2.0 ** 970, -2.0 ** 970, 2.0 ** 970 * (1 - 2.0 ** -53), -2.0 ** 970 * (1 - 2.0 ** -53)])
        sets.append(("overflow threshold", 1.0, a, b))
        if op == "triad":
            sets.append(("overflow threshold s=1+2^-52", 1.0 + 2.0 ** -52, a, b))
            sets.append(("overflow threshold s=1-2^-53", 1.0 - 2.0 ** -53, a, b))
    return sets
