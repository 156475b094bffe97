"""Exact reference of b200va_dot: numpy and `fractions` only, sharing no arithmetic with the kernels.

The contract (include/b200va.h), over LANES = 2048 and CHUNK = 65536:
  1. lane chain   the elements i of chunk k with the same i mod LANES form a lane, accumulated in increasing
                  index order: acc = +0.0; acc = fma(a_i, b_i, acc) in binary64 RNE, operands widened exactly
  2. chunk value  the 2048 lane values summed as an aligned dyadic (pairwise) tree
  3. total        the chunk values summed with the same tree; an empty upper half passes the lower half up
How this module replays it:
  f32, f16, bf16: every product of two widened operands is exact in f64, so the fma is one numpy f64 add.  The
  chunks are reshaped to (K, 32, 2048), padded with +0.0 products, and the 32 rows are added in order; then the
  trees.  Padding with +0.0 is exact: no lane value or chunk value is ever -0.0, and x + 0.0 == x otherwise.
  f64: the fma goes through Fraction (stream_exact's fma), limited to FRACTION_LIMIT elements.
  Both stream over blocks of chunks, so n = 2^28 needs a few GiB of host memory.

Also here: `exact_sum` (the exact dot as a Fraction), `error_bound` (the a-priori bound of the contract's
evaluation), `family` (inputs whose products and partial sums are all exact, so every order gives the exact
sum, known in closed form even far beyond the Fraction limit) and `adversarial` (inputs on which plausible wrong
kernels give other bits; shared by the CPU and the GPU tests).  f16/bf16 arrays are uint16 bit patterns.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from .stream_exact import BITS, FRACTION_LIMIT, STORAGE, _fraction_fma64, narrow, widen

LANES, CHUNK = 2048, 65536
ROWS = CHUNK // LANES
BLOCK_CHUNKS = 128                                   # chunks per streamed block: 2^23 elements


def chunks(n: int) -> int:
    return -(-n // CHUNK)


def tree(x: np.ndarray) -> np.ndarray:
    """The aligned dyadic tree along the last axis, padded with +0.0 to a power of two."""
    m = x.shape[-1]
    width = 1 << max(0, (m - 1).bit_length())
    if m == 0:
        return np.zeros(x.shape[:-1])
    if width != m:
        x = np.concatenate([x, np.zeros(x.shape[:-1] + (width - m,))], axis=-1)
    with np.errstate(all="ignore"):
        while x.shape[-1] > 1:
            x = x[..., 0::2] + x[..., 1::2]
    return x[..., 0]


def _lane_values_products(p: np.ndarray) -> np.ndarray:
    """(K, LANES) lane values of whole chunks of exact f64 products p (length a multiple of CHUNK)."""
    rows = p.reshape(-1, ROWS, LANES)
    acc = np.zeros((rows.shape[0], LANES))
    with np.errstate(all="ignore"):
        for r in range(ROWS):
            acc = acc + rows[:, r, :]
    return acc


def _lane_values_f64(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """(K, LANES) lane values of f64 operands, one Fraction fma per element (absent elements are +0.0 lanes)."""
    n = a.size
    out = np.zeros((chunks(n), LANES))
    xa, xb = a.tolist(), b.tolist()
    for k in range(chunks(n)):
        for lane in range(LANES):
            acc = 0.0
            for i in range(k * CHUNK + lane, min(n, (k + 1) * CHUNK), LANES):
                acc = _fraction_fma64(acc, xb[i], xa[i])
            out[k, lane] = acc
    return out


def chunk_values(a: np.ndarray, b: np.ndarray, dtype: str) -> np.ndarray:
    """The ceil(n / CHUNK) chunk values (rules 1 and 2)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == STORAGE[dtype] and b.dtype == a.dtype and a.size == b.size, (a.dtype, b.dtype, dtype)
    n = a.size
    if dtype == "f64":
        assert n <= FRACTION_LIMIT, "f64 lane chains through Fraction: use the exact family beyond FRACTION_LIMIT"
    out = []
    step = BLOCK_CHUNKS * CHUNK
    for lo in range(0, n, step):
        hi = min(n, lo + step)
        pad = chunks(hi - lo) * CHUNK - (hi - lo)
        if dtype == "f64":
            lanes = _lane_values_f64(a[lo:hi], b[lo:hi])
        else:
            with np.errstate(all="ignore"):
                p = widen(a[lo:hi], dtype) * widen(b[lo:hi], dtype)      # exact
            lanes = _lane_values_products(np.concatenate([p, np.zeros(pad)]))
        out.append(tree(lanes))
    return np.concatenate(out) if out else np.zeros(0)


def dot(a: np.ndarray, b: np.ndarray, dtype: str) -> float:
    """The contract's result (a Python float, never -0.0)."""
    return float(tree(chunk_values(a, b, dtype)))


# ------------------------------------------------------------------------------------------- exact values
def exact_sum(a: np.ndarray, b: np.ndarray, dtype: str) -> Fraction | None:
    """sum a_i b_i exactly, or None if an operand is not finite.  Integer arithmetic on the binary expansions."""
    x, y = widen(a, dtype), widen(b, dtype)
    if not (np.isfinite(x).all() and np.isfinite(y).all()):
        return None
    shift = 2 * 1074 + 2
    total = 0
    for u, v in zip(x.tolist(), y.tolist()):
        nu, du = u.as_integer_ratio()
        nv, dv = v.as_integer_ratio()
        total += (nu * nv) << (shift - (du.bit_length() - 1) - (dv.bit_length() - 1))
    return Fraction(total, 1 << shift)


def depth(n: int) -> int:
    """Roundings any one product passes through: the lane chain, the lane tree and the chunk tree."""
    return ROWS + (LANES.bit_length() - 1) + max(0, (chunks(n) - 1).bit_length())


def error_bound(a: np.ndarray, b: np.ndarray, dtype: str) -> Fraction:
    """A-priori bound on |result - exact_sum| (no overflow): gamma_d sum |a_i b_i|, d = depth(n), u = 2^-53.
    Every product enters the result through at most d additions, each with a relative error of at most u
    (f32/f16/bf16 products are exact; the f64 fma rounds the product and the sum once); a result in the
    subnormal range of an addition is exact."""
    d = depth(a.size)
    u = Fraction(1, 1 << 53)
    gamma = d * u / (1 - d * u)
    x, y = widen(a, dtype), widen(b, dtype)
    return gamma * exact_sum(np.abs(x), np.abs(y), "f64")


def family(dtype: str, n: int, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """a_i = m_i / 8, b_i = k_i / 4 with integers |m|, |k| <= 7: every product is (m k) / 32, every partial sum is
    an integer over 32 of magnitude at most 49 n / 32 < 2^53 for n <= 2^40, so any order of addition is exact."""
    rng = np.random.default_rng([seed, list(BITS).index(dtype)])
    m, k = rng.integers(-7, 8, n), rng.integers(-7, 8, n)
    return _store(m / 8.0, dtype), _store(k / 4.0, dtype)


def family_sum(a: np.ndarray, b: np.ndarray, dtype: str, n: int | None = None) -> float:
    """The exact (= the contract's) dot of the family arrays a, b repeated to n elements (default: their length)."""
    ma = np.rint(widen(a, dtype) * 8).astype(np.int64)
    kb = np.rint(widen(b, dtype) * 4).astype(np.int64)
    p = ma * kb
    n = a.size if n is None else n
    if n == 0:
        return 0.0
    q, r = divmod(n, a.size)
    total = q * int(p.sum()) + int(p[:r].sum())
    assert abs(total) < 1 << 53
    return float(Fraction(total, 32)) + 0.0          # + 0.0: never -0.0


def _store(x: np.ndarray, dtype: str) -> np.ndarray:
    """Exactly representable f64 values in the storage type."""
    if dtype in ("f16", "bf16"):
        return narrow(x.astype(np.float32), dtype)
    return x.astype(STORAGE[dtype])


# ------------------------------------------------------------------------------------------- adversarial inputs
# Operand exponents per type: small operands in [lo, top), the lane pair, the edge and chunk pairs, the head.
# A sum holding a large product rounds the small ones to a few bits.  f16 products are multiples of 2^-48, so
# its large products must reach 2^16 and more before f64 rounds anything; its small operands reach into the
# f16 subnormals.
_SMALL = {"f16": (-24, -16, 8, 10, 7), "bf16": (-20, -10, 14, 8, 5), "f32": (-20, -10, 14, 8, 5),
          "f64": (-20, -10, 14, 8, 5)}


def _random_mantissa(dtype, rng, e):
    """Values 2^e (1 + f) with random f, rounded to the storage type, random signs."""
    x = np.exp2(e.astype(np.float64)) * (1.0 + rng.random(e.size))
    x *= np.where(rng.random(e.size) < 0.5, -1.0, 1.0)
    return _store(x, dtype)


def cancellation(dtype: str, n: int = 3 * CHUNK + 5, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """Small products of random mantissas, and large products +-L that cancel in pairs: within one lane (rows 2
    and 29 of lane 5), across the edge of chunks 0 and 1 (the last element of one, the first of the next), across
    lanes of chunk 1 and across chunks 1 and 2.  A sum that holds an unmatched L loses the small products added to
    it, so which small products survive depends on exactly how the sums are grouped: every other lane count,
    chunk size or chunk edge, a sequential sum or a peeled first element (a middling product) gives other bits."""
    return _cancellation(dtype, n, seed, ("lane", "edge", "chunk", "head"))


def _cancellation(dtype, n, seed, features):
    """Small products of random mantissas plus the chosen features:
    lane   +-L1 in rows 2 and 29 of lane 5 of chunk 0, L1 = 2^(2 top + 48): what lane 5 adds in between keeps a
           few bits only
    edge   +-L2 as the last element of chunk 0 and the first of chunk 1, L2 = 2^(2 top + 36)
    chunk  +-L2 in lane 9 of chunk 1 and lane 11 of chunk 2
    head   a middling first element, 2^(2 top + 30)"""
    lo, top, lane_e, edge_e, head_e = _SMALL[dtype]
    rng = np.random.default_rng([seed, list(BITS).index(dtype), 1])
    e = rng.integers(lo, top, n)
    a, b = _random_mantissa(dtype, rng, e), _random_mantissa(dtype, rng, e)
    pairs = []
    if "lane" in features:
        pairs.append((2 * LANES + 5, 29 * LANES + 5, lane_e))
    if "edge" in features:
        pairs.append((CHUNK - 1, CHUNK, edge_e))
    if "chunk" in features:
        pairs.append((CHUNK + 2 * LANES + 9, 2 * CHUNK + 11, edge_e))
    for i, j, h in pairs:
        if j < n:
            big, nbig = _store(np.array([2.0 ** h, -2.0 ** h]), dtype)
            a[i], b[i], a[j], b[j] = big, big, big, nbig
    if "head" in features and n:
        a[0], b[0] = _store(np.array([2.0 ** head_e, 2.0 ** head_e]), dtype)
    return a, b


def specials(dtype: str, n: int = 2 * CHUNK + 77, seed: int = 0) -> list[tuple[str, np.ndarray, np.ndarray]]:
    """NaN, +-inf, inf * 0 and inf - inf (the last in different lanes and in different chunks), among finite values."""
    rng = np.random.default_rng([seed, list(BITS).index(dtype), 2])
    sets = []
    inf, ninf, nan, zero = (_store(np.array([v]), dtype)[0] for v in (np.inf, -np.inf, np.nan, 0.0))

    def base():
        return _random_mantissa(dtype, rng, rng.integers(-4, 4, n)), _random_mantissa(dtype, rng, rng.integers(-4, 4, n))

    a, b = base(); a[n // 2] = inf; b[n // 2] = np.abs(b[n // 2]) if dtype not in ("f16", "bf16") else b[n // 2] & 0x7FFF
    sets.append(("+inf", a, b))
    a, b = base(); a[7] = ninf; b[7] = _store(np.array([2.0]), dtype)[0]
    sets.append(("-inf", a, b))
    a, b = base(); a[CHUNK + 3] = inf; b[CHUNK + 3] = zero
    sets.append(("inf * 0", a, b))
    a, b = base(); a[5] = inf; b[5] = _store(np.array([1.0]), dtype)[0]; a[6] = ninf; b[6] = b[5]
    sets.append(("inf - inf across lanes", a, b))
    a, b = base(); a[5] = inf; b[5] = _store(np.array([1.0]), dtype)[0]; a[CHUNK + 9] = ninf; b[CHUNK + 9] = b[5]
    sets.append(("inf - inf across chunks", a, b))
    a, b = base(); a[n - 1] = nan
    sets.append(("NaN", a, b))
    return sets


def subnormals(dtype: str, n: int = CHUNK + 301, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """Operands in the subnormal range of the storage type (f64: products in f64's subnormal range) times
    ordinary values: a kernel that flushes subnormal operands or results to zero gets another sum (often 0)."""
    rng = np.random.default_rng([seed, list(BITS).index(dtype), 3])
    _, eb, mb = BITS[dtype]
    ut = BITS[dtype][0]
    man = rng.integers(1, 1 << mb, n, dtype=np.uint64)
    sign = rng.integers(0, 2, n).astype(np.uint64)
    a = ((sign << np.uint64(eb + mb)) | man).astype(ut).view(STORAGE[dtype])       # exponent field 0
    if dtype == "f64":
        b = _store(np.exp2(rng.integers(-60, -40, n).astype(np.float64)) * (1 + rng.random(n)), dtype)
    else:
        b = _store(np.exp2(rng.integers(-3, 3, n).astype(np.float64)) * (1 + rng.random(n)), dtype)
    return a, b


def adversarial(dtype: str, seed: int = 0) -> list[tuple[str, np.ndarray, np.ndarray]]:
    """[(name, a, b)]: the input sets where a plausible wrong kernel gives bits other than the contract's."""
    n = 3 * CHUNK + 5
    sets = [("cancellation", *cancellation(dtype, n, seed))]
    sets += [(f"cancellation: {f}", *_cancellation(dtype, n, seed + 1, (f,))) for f in ("lane", "edge", "chunk", "head")]
    sets.append(("subnormals", *subnormals(dtype, seed=seed)))
    return sets + specials(dtype, seed=seed)
