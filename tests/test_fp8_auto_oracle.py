"""CPU checks of tests/fp8_auto_exact.py, the reference of b200va_quantize_fp8_auto and b200va_dequantize_fp8_auto,
and of the SASS of the kernels that carry them.

- auto_scale_exp against a search in `Fraction` for the largest k with m 2^k <= max finite, for both formats and
  margins 0, 1 and 4: m at, just below and just above every binade edge of f64, the significands 1.75 and 1.75 +- 1
  ulp in every binade, the subnormals of f32, f16 and bf16 widened, the f64 subnormals, 0 and DBL_MAX (-126).
- A NaN, +inf or a value with the sign bit set left in *d_amax gives k = 0.
- The no-saturation property: with margin >= 0 and k not clamped, every finite element times 2^k lies within max
  finite; with margin 0 the next k would not.  Only +-inf gives +-max finite.
- finite_amax skips NaN and +-inf and keeps what the unsigned maximum keeps.
- The SASS of both libraries: each fp8_quant_vec holds one atomic for both of its bodies, and writes the 32-bit k;
  no FP8 kernel spills; the production library still has 199 functions.
"""
import math
import re
import sys
from fractions import Fraction

import numpy as np
import pytest

from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X

import fp8_auto_exact as A
import k8s_gpu_hpa_b200 as pkg  # noqa: F401  (builds nothing; the session fixture has built the library)
import sass
from k8s_gpu_hpa_b200 import capi

MARGINS = (0, 1, 4)
DBL_MAX = sys.float_info.max


def fraction_scale_exp(m: float, fmt: str, margin: int) -> int:
    """The largest integer k with m 2^k <= max finite, by bisection in `Fraction`, less margin, clamped."""
    if m == 0:
        return 126
    top, x = Fraction(F.MAX_FINITE[fmt]), Fraction(m)
    lo, hi = -1200, 1200                     # m 2^lo <= top < m 2^hi for every positive finite f64
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if x * Fraction(2) ** mid <= top:
            lo = mid
        else:
            hi = mid
    return min(max(lo - margin, -126), 126)


def binade_edges() -> list[float]:
    """2^e for every f64 binade (and the subnormal steps below it), with the neighbouring doubles, and 1.75 2^e with
    its neighbours."""
    out = []
    for e in range(-1074, 1024):
        p = math.ldexp(1.0, e)
        out += [p, math.nextafter(p, 0.0), math.nextafter(p, math.inf)]
        if e >= -1022:
            s = math.ldexp(1.75, e)
            out += [s, math.nextafter(s, 0.0), math.nextafter(s, math.inf)]
    return [v for v in out if 0 < v <= DBL_MAX]


def narrow_subnormals() -> list[float]:
    vals = []
    for dt, mb in (("f16", 10), ("bf16", 7)):
        bits = np.array([1, 2, 3, (1 << mb) - 1, 1 << mb], np.uint16)
        vals += X.widen(bits, dt).tolist()
    f32 = np.array([1, 2, 0x7FFFFF, 0x800000], np.uint32).view(np.float32)
    return vals + X.widen(f32, "f32").tolist()


@pytest.mark.parametrize("margin", MARGINS)
@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_scale_exp_equals_the_largest_k_in_fractions(fmt, margin):
    ms = binade_edges() + narrow_subnormals() + [0.0, DBL_MAX, 448.0, 57344.0, 5e-324]
    bad = [(m, A.auto_scale_exp(m, fmt, margin), fraction_scale_exp(m, fmt, margin)) for m in ms
           if A.auto_scale_exp(m, fmt, margin) != fraction_scale_exp(m, fmt, margin)]
    assert not bad, (len(bad), bad[:5])
    assert A.auto_scale_exp(0.0, fmt, margin) == 126 and A.auto_scale_exp(DBL_MAX, fmt, margin) == -126
    assert A.auto_scale_exp(F.MAX_FINITE[fmt], fmt, margin) == -margin
    # 1.75 2^e is max finite at k = emax - e; one ulp above it takes one more step down
    e = 3
    assert A.auto_scale_exp(math.ldexp(1.75, e), fmt, 0) == A.EMAX[fmt] - e
    assert A.auto_scale_exp(math.nextafter(math.ldexp(1.75, e), math.inf), fmt, 0) == A.EMAX[fmt] - e - 1


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_an_amax_the_caller_left_invalid_gives_k_0(fmt):
    for m in (math.nan, -math.nan, math.inf, -math.inf, -1.0, -0.0, -5e-324, -DBL_MAX):
        for margin in MARGINS:
            assert A.auto_scale_exp(m, fmt, margin) == 0, (m, margin)


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", V.DTYPES)
def test_no_finite_element_saturates(src, fmt):
    rng = np.random.default_rng([V.DTYPES.index(src), F.FORMATS8.index(fmt)])
    top = F.SPEC[fmt][4]
    for scale in (1e-3, 1.0, 300.0) + ((2.0 ** -30, 2.0 ** 20) if src != "f16" else ()):
        a = X.finite(src, 4099, rng, scale)
        for margin in (0, 1, 3):
            q, k, m = A.quantize_auto(a, src, fmt, margin)
            assert -126 < k < 126, (scale, k)
            x = np.abs(X.widen(a, src))
            assert (np.ldexp(x, k) <= F.MAX_FINITE[fmt]).all()
            if margin == 0:
                assert m * 2.0 ** (k + 1) > F.MAX_FINITE[fmt]       # k is the largest that fits
            # the rounded results stay within max finite: a result at max finite comes from a value that rounds to it
            at_top = (q & 0x7F) == top
            assert (np.ldexp(x[at_top], k) > F.values(fmt)[-2]).all()
    # +-inf saturates and NaN stays NaN, neither taking part in the amax
    x = np.array([1.5, -np.inf, np.inf, np.nan, -3.0])
    a = x.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(x, src)
    q, k, m = A.quantize_auto(a, src, fmt, 0)
    assert m == 3.0 and k == A.auto_scale_exp(3.0, fmt, 0)
    assert q[1] == 0x80 | top and q[2] == top and (q[3] & 0x7F) == 0x7F
    assert (q[[0, 4]] & 0x7F != top).all()


def test_finite_amax_skips_nan_and_infinities():
    a = np.array([1.0, np.nan, -np.inf, np.inf, -2.5, 0.5], np.float32)
    assert A.finite_amax(a, "f32") == 2.5
    assert A.finite_amax(np.array([np.nan, np.inf]), "f64") == 0.0
    assert A.finite_amax(np.array([np.nan]), "f64", 7.0) == 7.0
    assert A.finite_amax(V.round_f64(np.array([-65504.0, np.inf]), "f16"), "f16") == 65504.0
    assert A.finite_amax(np.array([1e300, -1e308]), "f64", 5.0) == 1e308
    # what the unsigned maximum of the patterns keeps: a NaN, +inf, or a value with the sign bit set
    assert math.isnan(A.finite_amax(a, "f32", math.nan)) and A.finite_amax(a, "f32", math.inf) == math.inf
    assert A.finite_amax(a, "f32", -1.0) == -1.0
    assert A.f64_bits(A.finite_amax(a, "f32", -0.0)) == 1 << 63
    # the quantize reference takes the amax it leaves
    q, k, m = A.quantize_auto(a, "f32", "e4m3", 0, 100.0)
    assert m == 100.0 and k == A.auto_scale_exp(100.0, "e4m3", 0) == 2


def test_dequantize_auto_out_of_range_is_nan():
    bits = np.arange(256, dtype=np.uint8)
    for dst in V.DTYPES:
        for k in (127, -127, -(1 << 31)):
            assert np.isnan(X.widen(A.dequantize_auto(bits, "e5m2", dst, k), dst)).all()
        got, want = A.dequantize_auto(bits, "e4m3", dst, -126), F.dequantize(bits, "e4m3", dst, -126)
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


# ------------------------------------------------------------------------------------------- SASS
def _fp8_functions(path: str) -> dict[str, str]:
    return {fn: body for fn, body in sass.functions(path).items() if re.match(r"_ZN6b200va\d+fp8_", fn)}


@pytest.mark.parametrize("path", ["production", "tune"])
def test_quant_kernels_share_one_atomic_and_write_k_after_the_wait(path):
    """The amax-only body and the quantize body reach one cta_amax, so one atomic; the 32-bit store of k (the only
    32-bit global store of a quantize kernel) comes after the wait."""
    fns = _fp8_functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH)
    quant = {fn: b for fn, b in fns.items() if "fp8_quant_vec" in fn}
    assert len(quant) == 4 and len(fns) == 8, sorted(fns)
    for fn, body in quant.items():
        ops = sass.opcodes(body)
        assert sum(o.startswith(("ATOMG", "RED")) for o in ops) == 1, fn
        stores = [i for i, o in enumerate(ops) if o == "STG.E"]
        assert stores and min(stores) > ops.index("ACQBULK"), (fn, stores)


def test_fp8_kernels_do_not_spill_and_the_production_library_keeps_199_functions():
    for path in (capi.LIB_PATH, capi.TUNE_LIB_PATH):
        for fn, body in _fp8_functions(path).items():
            assert not re.search(r"\b(LDL|STL)\b", body), fn
    assert len(sass.functions(capi.LIB_PATH)) == 199
