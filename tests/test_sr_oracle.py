"""CPU checks of oracle/sr_exact.py, the reference of b200va_convert_sr_f32 and b200va_quantize_fp8_sr_f32, and of the
stochastic-rounding kernel's SASS.

- round_sr against a restatement of the rule in `Fraction` (lo and hi from the quantum at |y|, f, t, the threshold,
  then overflow or saturation), on named sets for all four destinations: values already in D at many r; r = 2^32 - t
  and 2^32 - t - 1, which land on hi and on lo; subnormal targets and f32 subnormal sources; deep underflow (t = 0);
  the f16 / bf16 overflow band; FP8 saturation; +-0, +-inf and NaN; the FP8 scale at k = -126, 0 and 126.
- Unbiasedness, exactly: over a full residue system of r's high 20 bits, values whose t is a multiple of 2^12 round
  up exactly t / 2^12 times.  Over 2^20 hashed words for fixed seeds, the round-up count lies within six binomial
  standard deviations of f 2^20.
- The random bits: shard invariance, the numpy splitmix64 against the C oracle's counter generator, and for
  f32 -> bf16 the torch-eager "add the high 16 bits of r, clear the low 16 bits" idiom on the same bits.
- Mutants of the rule and of the bits (> for >=, the words' halves swapped, pairing by i instead of first + i, 16
  random bits instead of 32 for FP8, inf instead of saturation) give other bytes on the named sets.
- Without a GPU both entry points return an error and write nothing.
- The SASS: one sr_cast_vec in each library, with the four narrowing conversions and no local memory.
"""
import math
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle
from conftest import has_gpu
from oracle import fp8_exact as F
from oracle import sr_exact as S
from oracle import stream_exact as X

import k8s_gpu_hpa_b200 as pkg  # noqa: F401  (the session fixture has built the library)
import sass
from k8s_gpu_hpa_b200 import capi

TWO32 = 1 << 32
FP8 = ("e4m3", "e5m2")


def _fmt(dst):
    """(significand bits, minimum normal exponent, largest finite value) from the format tables."""
    if dst in FP8:
        prec, emin = F.SPEC[dst][:2]
        return prec, emin, Fraction(F.MAX_FINITE[dst])
    prec, emin, emax = X.FORMATS[dst]
    return prec, emin, (2 - Fraction(2) ** (1 - prec)) * Fraction(2) ** emax


PATTERN8 = {f: {float(v): p for p, v in enumerate(F.DECODE[f].tolist()) if not math.isnan(v)} for f in FP8}


def _encode(v: float, dst: str) -> int:
    """The pattern of a value of dst (+-inf for f16/bf16 included)."""
    if dst in FP8:
        return PATTERN8[dst][v] if v != 0 else (0x80 if math.copysign(1, v) < 0 else 0)
    if dst == "bf16":
        return int(np.array([v], np.float32).view(np.uint32)[0] >> 16)      # exact: v is a bf16 value
    return int(np.array([v], np.float16).view(np.uint16)[0])                # exact: v is an f16 value


def fraction_parts(v: float, dst: str, k: int):
    """(lo, hi, t) of the finite nonzero y = v 2^k by the rule, in Fraction."""
    prec, emin, _ = _fmt(dst)
    mag = abs(Fraction(v) * Fraction(2) ** k)
    e = mag.numerator.bit_length() - mag.denominator.bit_length()
    while Fraction(2) ** e > mag:
        e -= 1
    while Fraction(2) ** (e + 1) <= mag:
        e += 1
    q = Fraction(2) ** (max(e, emin) - prec + 1)            # D's spacing at |y|: fixed below the normal range
    lo = (mag // q) * q
    hi = lo + q
    t = math.floor((mag - lo) / (hi - lo) * TWO32)
    return lo, hi, t


def fraction_sr(a: np.ndarray, dst: str, r: np.ndarray, k: int = 0) -> np.ndarray:
    _, _, top = _fmt(dst)
    out = []
    for v, rr in zip(a.astype(np.float64).tolist(), r.tolist()):
        if math.isnan(v):
            out.append(None)
            continue
        if math.isinf(v):
            res = math.inf if dst not in FP8 else float(top)
        elif v == 0:
            res = 0.0
        else:
            lo, hi, t = fraction_parts(v, dst, k)
            if dst in FP8 and lo <= top:
                assert float(lo) in PATTERN8[dst] and (hi > top or float(hi) in PATTERN8[dst])   # D is the table
            res = hi if t + rr >= TWO32 else lo
            if res > top:
                res = math.inf if dst not in FP8 else top
            res = float(res)
        out.append(_encode(math.copysign(res, v), dst))
    return out


def is_nan(p, dst):
    p = np.asarray(p).astype(np.int64)
    if dst == "e4m3":
        return (p & 0x7F) == 0x7F
    if dst == "e5m2":
        return (p & 0x7F) > 0x7C
    if dst == "f16":
        return (p & 0x7FFF) > 0x7C00
    return (p & 0x7FFF) > 0x7F80


def assert_same(got, want, dst, what):
    got = np.asarray(got).astype(np.int64)
    nan_w = np.array([w is None for w in want])
    w = np.array([0 if x is None else x for x in want], np.int64)
    bad = np.where(nan_w, ~is_nan(got, dst), got != w)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} differ, first at {i}: got {got[i]:#x} want {want[i]}")


def f32(x):
    with np.errstate(all="ignore"):
        return np.asarray(x, np.float64).astype(np.float32)


def d_values(dst: str) -> np.ndarray:
    """Finite nonzero values of D (as f64), both signs: every one for FP8, a spread for f16 and bf16."""
    if dst in FP8:
        v = F.values(dst)[1:]
    else:
        bits = np.arange(1, 0x7C00 if dst == "f16" else 0x7F80, 7, dtype=np.uint16)
        v = X.widen(bits, dst)
    return np.concatenate([v, -v])


def threshold_pairs(a: np.ndarray, dst: str, k: int):
    """For each element with t > 0 (by the Fraction rule): (a, r) with r = 2^32 - t and r = 2^32 - t - 1, and the
    two expected results hi and lo."""
    xs, rs = [], []
    for v in a.astype(np.float64).tolist():
        if not math.isfinite(v) or v == 0:
            continue
        _, _, t = fraction_parts(v, dst, k)
        if t == 0:
            continue
        xs += [v, v]
        rs += [TWO32 - t, TWO32 - t - 1]
    return f32(xs), np.array(rs, np.uint64).astype(np.uint32)


def named_sets(dst: str, k: int = 0, seed: int = 0) -> dict:
    """{name: (a, r)}: f32 sources (y = a 2^k) and their random words."""
    rng = np.random.default_rng([seed, S.DESTS.index(dst), k + 200])
    prec, emin, top = _fmt(dst)
    scale = 2.0 ** -k
    sets = {}
    # values already in D, each at several r
    v = d_values(dst) * scale
    v = v[np.isfinite(f32(v)) & (f32(v) != 0)]
    v = v[f32(v).astype(np.float64) == v]                         # exactly representable as f32 sources
    rr = np.array([0, 1, 1 << 31, TWO32 - 1, 12345], np.uint64)
    sets["values in D"] = (f32(np.repeat(v, rr.size)), np.tile(rr, v.size).astype(np.uint32))
    # around the threshold: random values in the normal range, the subnormal range and the overflow band
    lo_n, hi_n = emin, (15 if dst in FP8 else X.FORMATS[dst][2])
    normal = np.ldexp(1 + rng.random(300), rng.integers(lo_n, hi_n + 1, 300)) * scale
    sub = rng.random(200) * 2.0 ** emin * scale
    sets["threshold, normal"] = threshold_pairs(f32(np.concatenate([normal, -normal])), dst, k)
    sets["threshold, subnormal targets"] = threshold_pairs(f32(np.concatenate([sub, -sub])), dst, k)
    # f32 subnormal sources (and their neighbours among the smallest normals)
    bits = np.concatenate([rng.integers(1, 1 << 23, 200), rng.integers(1 << 23, 1 << 24, 50)]).astype(np.uint32)
    fs = np.concatenate([bits, bits | np.uint32(1 << 31)]).view(np.float32)
    sets["f32 subnormal sources"] = (fs, rng.integers(0, TWO32, fs.size, dtype=np.uint64).astype(np.uint32))
    sets["f32 subnormal sources, threshold"] = threshold_pairs(fs, dst, k)
    # deep underflow: t = 0, so every r gives +-0
    # (|y| < 2^(emin-prec+1-32), and a = y 2^-k at least f32's smallest subnormal: none for bf16, or FP8 at k = 126)
    if -149 + k < emin - prec - 32:
        deep = np.ldexp(1 + rng.random(100), rng.integers(-149 + k, emin - prec - 32, 100)) * scale
        deep = f32(np.concatenate([deep, -deep]))
        sets["deep underflow"] = (deep, np.full(deep.size, TWO32 - 1, np.uint64).astype(np.uint32))
    # the top: f16/bf16 between max finite and the next binade (inf past it), FP8 saturation
    t = float(top)
    band = np.concatenate([t + rng.random(100) * (2 ** math.floor(math.log2(t)) * 2 - t), [t, np.nextafter(t, 0)]])
    if dst in FP8:
        band = np.concatenate([band, [t * 1.01, t * 2, t * 1000, 3e38 * scale]])
    band = f32(band * scale)
    band = band[np.isfinite(band)]
    band = np.concatenate([band, -band])
    sets["overflow or saturation band"] = (band, rng.integers(0, TWO32, band.size, dtype=np.uint64).astype(np.uint32))
    sets["overflow or saturation band, threshold"] = threshold_pairs(band, dst, k)
    special = f32([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 3.4e38, -3.4e38])
    special = np.tile(special, 4)
    sets["zeros, infinities, NaN"] = (special, np.repeat(np.array([0, 1, 1 << 31, TWO32 - 1], np.uint64),
                                                         8).astype(np.uint32))
    return {name: v for name, v in sets.items() if v[0].size}    # no f32 subnormal has t > 0 for f16 and FP8


def _cases():
    return [(d, 0) for d in S.DESTS] + [(f, k) for f in FP8 for k in (-126, 126)]


@pytest.mark.parametrize("dst,k", _cases())
def test_oracle_equals_the_rule_in_fractions_on_the_named_sets(dst, k):
    for name, (a, r) in named_sets(dst, k).items():
        assert a.size, name
        assert_same(S.round_sr(a, dst, r, k), fraction_sr(a, dst, r, k), dst, f"{dst} k={k} {name}")


@pytest.mark.parametrize("dst,k", _cases())
def test_threshold_lands_on_hi_and_on_lo(dst, k):
    """r = 2^32 - t gives hi, r = 2^32 - t - 1 gives lo: the two results are one step of D apart (the one above
    the top of the finite range excepted, where hi overflows or saturates)."""
    sets = named_sets(dst, k)
    for name in ("threshold, normal", "threshold, subnormal targets", "f32 subnormal sources, threshold"):
        if name not in sets:
            continue
        a, r = sets[name]
        got = S.round_sr(a, dst, r, k).astype(np.int64)
        hi, lo = got[0::2], got[1::2]
        assert hi.size
        mask = 0x7F if dst in FP8 else 0x7FFF
        below = (lo & mask) < (F.SPEC[dst][4] if dst in FP8 else 0x7FFF)      # FP8 saturates from the top on
        assert below.any() and ((hi & mask) == (lo & mask) + 1)[below].all(), (dst, k, name)
        assert (hi[~below] == lo[~below]).all(), (dst, k, name)
        assert (S.threshold_t(a[0::2], dst, k) == (TWO32 - r[0::2].astype(np.uint64))).all()


def test_values_in_d_never_move():
    for dst in S.DESTS:
        a, r = named_sets(dst)["values in D"]
        assert (S.threshold_t(a, dst) == 0).all()
        want = X.narrow(a, dst) if dst not in FP8 else F.quantize(a, "f32", dst)
        assert (S.round_sr(a, dst, r) == want).all(), dst


def test_unbiased_over_a_full_residue_system_of_the_high_bits():
    """Values whose t is a multiple of 2^12 (every f32 pattern in the normal range for bf16, f16 and E4M3; those with
    the last bit clear for E5M2): with r = 2^12 j + c over all j < 2^20 and a fixed c, exactly t / 2^12 round up."""
    rng = np.random.default_rng(3)
    j = np.arange(1 << 20, dtype=np.uint64)
    for dst in S.DESTS:
        prec, emin, _ = _fmt(dst)
        hi_e = 15 if dst in FP8 else X.FORMATS[dst][2]
        for v in np.ldexp(1 + rng.random(6), rng.integers(emin, hi_e, 6)):
            a = f32([v])
            a = (a.view(np.uint32) & np.uint32(~1 & 0xFFFFFFFF)).view(np.float32)
            t = int(S.threshold_t(a, dst)[0])
            assert t % (1 << 12) == 0
            lo = S.round_sr(a, dst, np.zeros(1, np.uint32))[0]
            c = int(rng.integers(0, 1 << 12))
            got = S.round_sr(np.repeat(a, j.size), dst, ((j << np.uint64(12)) + np.uint64(c)).astype(np.uint32))
            assert int((got != lo).sum()) == t >> 12, (dst, v, t)


def test_unbiased_within_a_binomial_bound_over_hashed_words():
    """2^20 words from random_words for fixed seeds: the round-up count of a fixed value lies within 6 standard
    deviations of f 2^20 (deterministic: the seeds are fixed)."""
    n = 1 << 20
    rng = np.random.default_rng(4)
    for seed in (1, 0xDEADBEEF, 1 << 63):
        r = S.random_words(seed, seed >> 3, n)
        for dst in S.DESTS:
            prec, emin, _ = _fmt(dst)
            for v in (1 + rng.random() * 2.0 ** -(prec - 1), 2.0 ** (emin - 1) * rng.random()):
                a = np.full(n, np.float32(v))
                lo, hi, t = fraction_parts(float(np.float32(v)), dst, 0)
                f = float((abs(Fraction(float(np.float32(v)))) - lo) / (hi - lo))
                ups = int((S.round_sr(a, dst, r) != S.round_sr(a[:1], dst, np.zeros(1, np.uint32))[0]).sum())
                assert abs(ups - f * n) <= 6 * math.sqrt(n * f * (1 - f)) + 1, (seed, dst, v, ups, f * n)


def test_shard_invariance():
    rng = np.random.default_rng(5)
    a = f32(rng.standard_normal(10_007) * 100)
    for first in (0, 1, (1 << 32) + 3, (1 << 64) - 5):
        whole = S.convert_sr(a, "bf16", 7, first)
        q = S.quantize_fp8_sr(a, "e4m3", 7, first, 2)
        for i0, i1 in ((0, 1), (1, 4), (3, 8), (999, 5000), (5001, 10_007)):
            assert (S.convert_sr(a[i0:i1], "bf16", 7, first + i0) == whole[i0:i1]).all()
            assert (S.quantize_fp8_sr(a[i0:i1], "e4m3", 7, first + i0, 2) == q[i0:i1]).all()


def test_random_words_layout_and_the_c_counter_generator():
    """splitmix64 here equals the C oracle's counter generator (x = (splitmix64(seed PHI + first + i) >> 40) 2^-24);
    r_m takes the low half of w_(m>>1) for even m and the high half for odd m, with w_j = splitmix64(key + j)."""
    for n, seed, first in ((1000, 0x0A, 0), (4097, 0x0B, 1 << 33), (77, 3, (1 << 64) - 40)):
        with np.errstate(over="ignore"):
            base = np.uint64((seed * 0x9E3779B97F4A7C15 + first) & ((1 << 64) - 1))
            z = S.splitmix64(base + np.arange(n, dtype=np.uint64))
        mine = (z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
        assert np.array_equal(mine, oracle.fill_ctr(n, seed, first))
    key = int(S.splitmix64(np.uint64(9)))
    r = S.random_words(9, 5, 4)                              # m = 5, 6, 7, 8
    w = [int(S.splitmix64(np.uint64((key + j) & ((1 << 64) - 1)))) for j in (2, 3, 4)]
    assert r.tolist() == [w[0] >> 32, w[1] & 0xFFFFFFFF, w[1] >> 32, w[2] & 0xFFFFFFFF]


def test_bf16_equals_the_torch_eager_idiom():
    """(pattern + (r >> 16)) with the low 16 bits cleared, on the same r: equal for every finite source."""
    rng = np.random.default_rng(6)
    bits = rng.integers(0, TWO32, 1 << 18, dtype=np.uint64).astype(np.uint32)
    a = bits.view(np.float32)
    a = a[np.isfinite(a)]
    r = S.random_words(11, 3, a.size)
    x = torch.from_numpy(a.copy()).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    y = ((x + (torch.from_numpy(r.astype(np.int64)) >> 16)) & 0xFFFF0000).to(torch.int32)   # a carry past 2^32 only
    want = y.view(torch.float32).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)  # from -max: none here
    assert np.array_equal(S.round_sr(a, "bf16", r), want)


# ------------------------------------------------------------------------------------------- mutants
def _mutant_round(a, dst, r, k=0, *, gt=False, bits16=False, inf_not_sat=False):
    """round_sr with one mistake."""
    prec, emin, clamp, sbit, ut = S._params(dst)
    sign, E, M, e, finite_nz, q, t = S._split(a, dst, k)
    r = r.astype(np.uint64)
    if gt:
        up = (t + r) > np.uint64(TWO32)
    elif bits16:
        up = ((t >> np.uint64(16)) + (r >> np.uint64(16))) >= np.uint64(1 << 16)
    else:
        up = (t + r) >= np.uint64(TWO32)
    if inf_not_sat:
        clamp = 0x7C if dst == "e5m2" else 0x7F
    mag = (np.maximum(e, emin) - emin).astype(np.uint64) * np.uint64(1 << (prec - 1)) + q + up.astype(np.uint64)
    mag = np.minimum(np.where(finite_nz, mag, 0), np.uint64(clamp))
    mag = np.where(E == 0x7FF, np.where(M == 0, np.uint64(clamp), np.uint64(0x7F)), mag)
    return ((sign << np.uint64(sbit)) | mag).astype(ut)


def _mutant_words(seed, first, n, *, swapped=False, by_i=False):
    key = S.splitmix64(np.uint64(seed))
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        m = np.uint64(first) + i
        j = (np.uint64(first) >> np.uint64(1)) + (i >> np.uint64(1)) if by_i else m >> np.uint64(1)
        w = S.splitmix64(key + j)
    odd = ((i if by_i else m) & np.uint64(1)) == 1
    if swapped:
        odd = ~odd
    return np.where(odd, w >> np.uint64(32), w & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def _all_named(dst, k=0):
    sets = named_sets(dst, k)
    return np.concatenate([a for a, _ in sets.values()]), np.concatenate([r for _, r in sets.values()])


@pytest.mark.parametrize("dst", S.DESTS)
def test_mutants_of_the_rule_are_caught(dst):
    for k in ((0,) if dst not in FP8 else (-126, 0, 126)):
        a, r = _all_named(dst, k)
        want = S.round_sr(a, dst, r, k)
        assert (_mutant_round(a, dst, r, k, gt=True) != want).any(), (dst, k, "> for >=")
        if dst in FP8:
            assert (_mutant_round(a, dst, r, k, bits16=True) != want).any(), (dst, k, "16 random bits")
            assert (_mutant_round(a, dst, r, k, inf_not_sat=True) != want).any(), (dst, k, "inf, not saturation")


@pytest.mark.parametrize("dst", S.DESTS)
def test_mutants_of_the_bits_are_caught(dst):
    """On the named sets with random_words for an odd first: the halves swapped, and pairing by i."""
    a, _ = _all_named(dst)
    a = a[np.isfinite(a)]
    k = 0
    for first in (1, (1 << 40) + 7):
        want = S.round_sr(a, dst, S.random_words(5, first, a.size), k)
        for kw in ({"swapped": True}, {"by_i": True}):
            got = S.round_sr(a, dst, _mutant_words(5, first, a.size, **kw), k)
            assert (got != want).any(), (dst, first, kw)


# ------------------------------------------------------------------------------------------- no GPU, SASS
@pytest.mark.skipif(has_gpu(), reason="checks the no-GPU failure mode")
def test_entry_points_fail_without_a_gpu_and_write_nothing():
    a = np.ones(64, np.float32)
    c = np.full(64, 0x5A, np.uint8)
    m = np.full(1, -7.0)
    assert capi.lib.b200va_convert_sr_f32(a.ctypes.data, 3, c.ctypes.data, 16, 1, 0, None) != capi.OK
    assert capi.lib.b200va_quantize_fp8_sr_f32(a.ctypes.data, 0, c.ctypes.data, 64, 0, 1, 0, m.ctypes.data, None) != capi.OK
    assert (c == 0x5A).all() and m[0] == -7.0


def _sr_functions(path: str) -> dict[str, str]:
    return {fn: body for fn, body in sass.functions(path).items() if "sr_cast_vec" in fn}


@pytest.mark.parametrize("path", ["production", "tune"])
def test_one_sr_kernel_with_all_four_narrowings_and_no_local_memory(path):
    fns = _sr_functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH)
    assert len(fns) == 1, sorted(fns)
    body = next(iter(fns.values()))
    for op in ("F2FP.SATFINITE.E4M3.F32", "F2FP.SATFINITE.E5M2.F32", "F2FP.BF16.F32.PACK_AB", "F2FP.F16.F32.PACK_AB"):
        assert op in body, op
    assert "LDG.E.128" in body and "STG.E.NA.128" in body
    assert not re.search(r"\b(LDL|STL)\b", body)
