"""CPU checks of oracle/mxfp8_exact.py, the reference of b200va_quantize_mxfp8 and b200va_dequantize_mxfp8, and of the
block-scaled kernels' SASS.

- quantize against a restatement of the contract in `Fraction`, written independently: the block maximum as a
  rational, e found by comparing with powers of two (for "nosat": the smallest e under which the maximum fits, which
  is how the header words it), `fp8_exact.nearest_fraction` for the rounding; every source, both formats, all three
  blocks, both rules, on random bit patterns with n ragged around the block edges and on the named sets of
  `mxfp8_exact.named_blocks`.
- What the named sets pin: the two rules differ exactly where the maximum exceeds 1.75 2^j, and there OCP saturates;
  blocks of zeros, -0, subnormals, inf and NaN; both clamps from f64; an outlier changes its own block's scale only.
- The sets have teeth: blocks counted from another origin, a maximum that includes inf, ceil instead of floor, and
  subnormals flushed to zero each give other bytes.
- dequantize against `Fraction` rounded once for all 256 patterns and the scale bytes 0, 1, 126, 127, 128, 254, 255;
  the round trip is exact whenever a block's values are FP8 values times one power of two.
- The SASS of both libraries: 3 + 3 mx_ kernels, each with the bodies of both formats, the block maximum by
  SHFL.BFLY, 16-byte loads and stores, no RN F2F.F32.F64, no local memory, no atomics.
"""
import math
import re
from fractions import Fraction

import numpy as np
import pytest

from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import mxfp8_exact as MX
from oracle import stream_exact as X

import k8s_gpu_hpa_b200 as pkg  # noqa: F401  (builds nothing; the session fixture has built the library)
import sass
from k8s_gpu_hpa_b200 import capi

DTYPES = V.DTYPES
SCALE_BYTES = (0, 1, 126, 127, 128, 254, 255)
PATTERN = {f: {float(v): p for p, v in enumerate(F.DECODE[f].tolist()) if not math.isnan(v)} for f in F.FORMATS8}


def is_nan8(p, fmt):
    m = np.asarray(p, np.uint8) & 0x7F
    return m == 0x7F if fmt == "e4m3" else m > 0x7C


def assert_same8(got, want, fmt, what=""):
    g, w = np.asarray(got, np.uint8), np.asarray(want, np.uint8)
    bad = (g != w) & ~(is_nan8(g, fmt) & is_nan8(w, fmt))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} mismatches, first at {i}: got {g[i]:#04x} want {w[i]:#04x}")


def _floor_log2(m: Fraction) -> int:
    e = m.numerator.bit_length() - m.denominator.bit_length()
    while Fraction(2) ** e > m:
        e -= 1
    while Fraction(2) ** (e + 1) <= m:
        e += 1
    return e


def fraction_exponent(m: Fraction, fmt: str, rule: str) -> int:
    """The contract's e for a block maximum m, by comparison with powers of two."""
    if m == 0:
        return -127
    top = Fraction(F.MAX_FINITE[fmt])
    if rule == "ocp":
        e = _floor_log2(m) - MX.EMAX[fmt]
    else:                                               # the smallest e with m 2^-e <= max finite
        e = _floor_log2(m) - MX.EMAX[fmt] - 2
        while m / Fraction(2) ** e > top:
            e += 1
        assert m / Fraction(2) ** (e - 1) > top
    return max(-127, min(127, e))


def fraction_quantize(a, src, fmt, block, rule):
    """The contract block by block and element by element in `Fraction`: (FP8 patterns, scale bytes)."""
    vals = X.widen(a, src).tolist()
    out, scales = [], []
    for lo in range(0, len(vals), block):
        blk = vals[lo:lo + block]
        m = max((abs(Fraction(v)) for v in blk if math.isfinite(v)), default=Fraction(0))
        e = fraction_exponent(m, fmt, rule)
        scales.append(e + 127)
        for v in blk:
            if math.isnan(v):
                out.append(0x7F)
                continue
            if math.isinf(v):
                r = math.copysign(F.MAX_FINITE[fmt], v)
            elif v == 0:
                r = v
            else:
                r = F.nearest_fraction(Fraction(v) / Fraction(2) ** e, fmt)
                if r == 0:
                    r = math.copysign(0.0, v)
            out.append(PATTERN[fmt][r] if r != 0 else (0x80 if math.copysign(1, r) < 0 else 0))
    return np.array(out, np.uint8), np.array(scales, np.uint8)


def check_against_fractions(a, src, fmt, block, rule, what):
    q, s = MX.quantize(a, src, fmt, block, rule)
    wq, ws = fraction_quantize(a, src, fmt, block, rule)
    assert s.dtype == np.uint8 and s.size == MX.scale_count(a.size, block) and (s != 0xFF).all(), what
    assert (s == ws).all(), (what, "scales", np.flatnonzero(s != ws)[:5], s[s != ws][:5], ws[s != ws][:5])
    assert_same8(q, wq, fmt, what)


# ------------------------------------------------------------------------------------------- quantize
@pytest.mark.parametrize("rule", MX.RULES)
@pytest.mark.parametrize("block", MX.BLOCKS)
@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_equals_the_contract_in_fractions(src, fmt, block, rule):
    rng = np.random.default_rng([DTYPES.index(src), F.FORMATS8.index(fmt), block, MX.RULES.index(rule)])
    for n in (1, block - 1, block, block + 1, 3 * block + 17):
        check_against_fractions(V.random_bits(src, n, rng), src, fmt, block, rule, f"{src}->{fmt} random bits n={n}")
        check_against_fractions(X.finite(src, n, rng, 3.0), src, fmt, block, rule, f"{src}->{fmt} finite n={n}")
    for name, a in MX.named_blocks(src, fmt, block).items():
        check_against_fractions(a, src, fmt, block, rule, f"{src}->{fmt} block {block} {rule}: {name}")
    assert MX.quantize(np.zeros(0, X.STORAGE[src]), src, fmt, block, rule)[1].size == 0


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_the_rules_differ_exactly_above_one_point_seven_five(src, fmt):
    """e(nosat) = e(ocp) + 1 where the maximum's significand exceeds 1.75 and equal elsewhere; under OCP the maximum
    saturates there (it lies in (max finite, 2^(emax+1)) 2^e) and under NOSAT no finite value is clamped."""
    sets = MX.named_blocks(src, fmt, 32)
    top = F.SPEC[fmt][4]
    for name in ("m = 2^j", "m = 1.75 2^j", "m one ulp below 1.75 2^j"):
        assert (MX.block_exponents(sets[name], src, fmt, 32, "ocp") == MX.block_exponents(sets[name], src, fmt, 32, "nosat")).all()
    a = sets["m one ulp above 1.75 2^j"]
    eo, en = MX.block_exponents(a, src, fmt, 32, "ocp"), MX.block_exponents(a, src, fmt, 32, "nosat")
    free = (eo > -127) & (eo < 127)                              # not clamped
    assert free.sum() >= 5 and (en[free] == eo[free] + 1).all()
    x = np.abs(X.widen(a, src)).reshape(-1, 32)
    at_max = x == x.max(axis=1, keepdims=True)
    qo = (MX.quantize(a, src, fmt, 32, "ocp")[0] & 0x7F).reshape(-1, 32)
    assert (qo[at_max & free[:, None]] == top).all()
    # under NOSAT the scaled maximum is at most max finite: nothing finite lies beyond it
    scaled = np.ldexp(x, -np.repeat(en, 32).reshape(-1, 32))
    assert (scaled[en < 127] <= F.MAX_FINITE[fmt]).all()
    # and a maximum of exactly 1.75 2^j maps onto max finite under both rules
    a = sets["m = 1.75 2^j"]
    x = np.abs(X.widen(a, src)).reshape(-1, 32)
    free = np.abs(MX.block_exponents(a, src, fmt, 32, "ocp")) < 127
    q = (MX.quantize(a, src, fmt, 32, "ocp")[0] & 0x7F).reshape(-1, 32)
    assert (q[(x == x.max(axis=1, keepdims=True)) & free[:, None]] == top).all()


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_value_classes(src, fmt):
    sets = MX.named_blocks(src, fmt, 64)
    top = F.SPEC[fmt][4]
    q, s = MX.quantize(sets["zeros"], src, fmt, 64)
    assert (q == 0).all() and s.tolist() == [0]
    q, s = MX.quantize(sets["-0"], src, fmt, 64)
    assert (q == 0x80).all() and s.tolist() == [0]
    q, s = MX.quantize(sets["all NaN"], src, fmt, 64)
    assert is_nan8(q, fmt).all() and s.tolist() == [0]
    q, s = MX.quantize(sets["inf, -inf and NaN only"], src, fmt, 64)
    assert s.tolist() == [0] and q[:4].tolist()[:2] == [top, 0x80 | top] and is_nan8(q[2:4], fmt).all()
    # inf and NaN leave the scale alone and follow the FP8 rules themselves
    plain = MX.named_blocks(src, fmt, 64)["an inf beside finite values"].copy()
    with_inf = plain.copy()
    plain[1] = plain[2]
    (qp, sp), (qi, si) = MX.quantize(plain, src, fmt, 64), MX.quantize(with_inf, src, fmt, 64)
    assert (sp == si).all() and qi[1] == top and (np.delete(qp, 1) == np.delete(qi, 1)).all()
    q, s = MX.quantize(sets["a -inf and a NaN beside finite values"], src, fmt, 64)
    assert (s == si).all() and q[1] == 0x80 | top and is_nan8(q[2], fmt)
    # subnormal-only blocks clamp at -127 and still quantize to nonzero values where 2^127 lifts them into range
    q, s = MX.quantize(sets["subnormals only"], src, fmt, 64)
    if src != "f16":                                            # f16 subnormals are above 2^-24: not clamped
        assert (s == 0).all()
    if src in ("f32", "bf16", "f16"):
        assert ((q & 0x7F) != 0).any()
    # an outlier changes its own block only
    (q0, s0), (q1, s1) = MX.quantize(sets["no outlier"], src, fmt, 64), MX.quantize(sets["an outlier in the middle block"], src, fmt, 64)
    assert s0[0] == s1[0] and s0[2] == s1[2] and s1[1] > s0[1]
    assert (q0[:64] == q1[:64]).all() and (q0[128:] == q1[128:]).all() and (q0[64:128] != q1[64:128]).any()


def test_both_clamps_from_f64():
    for fmt in F.FORMATS8:
        emax = MX.EMAX[fmt]
        m = np.array([2.0 ** (127 + emax), 2.0 ** (128 + emax), 2.0 ** 1023, 2.0 ** (emax - 127), 2.0 ** (emax - 128), 5e-324])
        a = MX.blocks_with_maximum(m, "f64", 32)
        for rule in MX.RULES:
            assert MX.block_exponents(a, "f64", fmt, 32, rule).tolist() == [127, 127, 127, -127, -127, -127]
        q, s = MX.quantize(a, "f64", fmt, 32)
        assert s.tolist() == [254, 254, 254, 0, 0, 0]
        x = np.abs(a).reshape(-1, 32)
        at_max = x == x.max(axis=1, keepdims=True)
        qm = (q & 0x7F).reshape(-1, 32)[at_max]
        assert qm[0] == PATTERN[fmt][2.0 ** emax] and qm[1] == qm[2] == F.SPEC[fmt][4]     # clamped at 127: saturates
        assert qm[3] == PATTERN[fmt][2.0 ** emax] and qm[4] == PATTERN[fmt][2.0 ** (emax - 1)] and qm[5] == 0
    # e = 127 is out of reach of the f32 family: its largest value gives 127 - emax (+ 1)
    big = np.full(32, np.finfo(np.float32).max, np.float32)
    assert MX.block_exponents(big, "f32", "e4m3", 32, "nosat").tolist() == [127 - 8 + 1]


# ------------------------------------------------------------------------------------------- teeth
def _requantize(a, src, fmt, block, e):
    """a quantized with the given per-block exponents (what a wrong scale rule would store and use)."""
    e = np.clip(e, -127, 127)
    with np.errstate(all="ignore"):
        return F.round_fp8(np.ldexp(X.widen(a, src), -np.repeat(e, block)[:a.size]), fmt), (e + 127).astype(np.uint8)


def _differs(got, want, fmt):
    (gq, gs), (wq, ws) = got, want
    return bool(((gq != wq) & ~(is_nan8(gq, fmt) & is_nan8(wq, fmt))).any() or (gs != ws).any())


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_the_named_sets_have_teeth(src, fmt):
    block = 32
    sets = MX.named_blocks(src, fmt, block)
    # blocks counted from an address boundary instead of element 0: the array 8 elements further on
    a = np.concatenate([sets["no outlier"], sets["an outlier in the middle block"], sets["m = 2^j"]])
    shifted = MX.quantize(a[8:], src, fmt, block)
    whole = MX.quantize(a, src, fmt, block)
    assert (shifted[0] != whole[0][8:]).any()
    # a maximum that includes inf
    a = sets["an inf beside finite values"]
    assert _differs(_requantize(a, src, fmt, block, np.array([127])), MX.quantize(a, src, fmt, block), fmt)
    # ceil(log2 m) for the OCP rule
    a = sets["m = 1.75 2^j"]
    m = MX.block_maxima(a, src, block)
    ceil_e = np.ceil(np.log2(m)).astype(np.int64) - MX.EMAX[fmt]
    assert _differs(_requantize(a, src, fmt, block, ceil_e), MX.quantize(a, src, fmt, block), fmt)
    # subnormal sources flushed to zero
    a = sets["subnormals only"]
    if src != "f64":                                    # f64 subnormals times 2^127 are far below every FP8 value
        x = X.widen(a, src)
        tiny = 2.0 ** X.FORMATS[src][1]
        flushed = MX._storage(np.where(np.abs(x) < tiny, np.copysign(0.0, x), x), src)
        assert _differs(MX.quantize(flushed, src, fmt, block), MX.quantize(a, src, fmt, block), fmt)


# ------------------------------------------------------------------------------------------- dequantize
@pytest.mark.parametrize("block", MX.BLOCKS)
@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("dst", DTYPES)
def test_dequantize_equals_fraction_rounded_once(dst, fmt, block):
    bits = np.tile(np.arange(256, dtype=np.uint8), -(-len(SCALE_BYTES) * block // 256))[:len(SCALE_BYTES) * block]
    bits = np.concatenate([bits, bits[:5]])                     # a short last block
    scales = np.array(SCALE_BYTES + (130,), np.uint8)
    got = X.widen(MX.dequantize(bits, scales, fmt, dst, block), dst)
    want = []
    for i, p in enumerate(bits.tolist()):
        v, s = float(F.DECODE[fmt][p]), int(scales[i // block])
        if s == 0xFF or math.isnan(v):
            want.append(math.nan)
        elif math.isinf(v) or v == 0:
            want.append(v)
        else:
            want.append(X.round_fraction(Fraction(v) * Fraction(2) ** (s - 127), dst))
    w = np.array(want, np.float64)
    same = (got.view(np.uint64) == w.view(np.uint64)) | (np.isnan(got) & np.isnan(w))
    assert same.all(), (dst, fmt, block, np.flatnonzero(~same)[:5])
    assert np.isnan(got[6 * block:7 * block]).all()             # 0xFF: the zeros and the infinities too


@pytest.mark.parametrize("rule", MX.RULES)
@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_round_trip_is_exact_for_fp8_values_times_one_power_of_two(fmt, rule):
    """Under NOSAT for every such block; under OCP unless the block maximum's significand is 1.875 (E4M3 has such
    values below its top binade), which the OCP rule saturates."""
    rng = np.random.default_rng(F.FORMATS8.index(fmt))
    finite = np.flatnonzero(np.isfinite(F.DECODE[fmt])).astype(np.uint8)
    if (fmt, rule) == ("e4m3", "ocp"):
        finite = finite[(finite & 7) != 7]
    for block in MX.BLOCKS:
        nb = 40
        p = rng.choice(finite, nb * block)
        j = rng.integers(-90, 90, nb)
        a = np.ldexp(F.DECODE[fmt][p], np.repeat(j, block))
        for src in ("f64", "f32"):
            q, s = MX.quantize(a.astype(X.STORAGE[src]), src, fmt, block, rule)
            back = MX.dequantize(q, s, fmt, "f64", block)
            assert (back == a).all() and (np.signbit(back) == np.signbit(a)).all(), (fmt, rule, block, src)


# ------------------------------------------------------------------------------------------- SASS
def _functions(path: str) -> dict[str, str]:
    return {fn: body for fn, body in sass.functions(path).items() if re.match(r"_ZN6b200va\d+mx_", fn)}


@pytest.mark.parametrize("path", ["production", "tune"])
def test_mx_kernels_in_the_sass(path):
    """One kernel per element size of the non-FP8 side and direction (3 + 3: f16 and bf16 share one), each carrying
    the bodies of both formats."""
    fns = _functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH)
    quant = {fn: b for fn, b in fns.items() if "mx_quant_vec" in fn}
    deq = {fn: b for fn, b in fns.items() if "mx_dequant_vec" in fn}
    assert len(quant) == 3 and len(deq) == 3 and len(fns) == 6, sorted(fns)
    assert {int(re.search(r"ILi(\d)EE", fn).group(1)) for fn in quant} == {2, 4, 8} == {int(re.search(r"ILi(\d)EE", fn).group(1)) for fn in deq}
    for fn, body in fns.items():
        assert not re.search(r"\b(LDL|STL)\b", body), fn                     # no spills
        assert not re.search(r"\b(ATOM|ATOMG|RED|REDG)\b", body), fn
        assert not re.search(r"F2F\.F32\.F64(?!\.RZ)", body), fn             # never RN from f64 to f32
        assert "STG.E.NA.128" in body, fn
    for fn, body in quant.items():
        es = int(re.search(r"ILi(\d)EE", fn).group(1))
        for f8 in ("E4M3", "E5M2"):
            assert f"F2FP.SATFINITE.{f8}.F32" in body, (fn, f8)
        assert "SHFL.BFLY" in body and "LDG.E.128" in body and "STG.E.U8" in body, fn
        if es == 8:
            assert "F2F.F32.F64.RZ" in body, fn
    for fn, body in deq.items():
        es = int(re.search(r"ILi(\d)EE", fn).group(1))
        for f8 in ("E4M3", "E5M2"):
            assert f"F2FP.F16.{f8}.UNPACK_B" in body, (fn, f8)
        assert "LDG.E.U8" in body and "SHFL" not in body, fn                 # the scale byte; no exchange between lanes
        if es == 2:
            assert "F2FP.F16.F32.PACK_AB" in body and "F2FP.BF16.F32.PACK_AB" in body, fn


def test_scale_bytes():
    L = capi.lib
    for block in MX.BLOCKS:
        for n in (0, 1, block - 1, block, block + 1, 10 * block, (1 << 40)):
            assert L.b200va_mxfp8_scale_bytes(n, block) == MX.scale_count(n, block)
    for block in (0, 16, 33, 256, -32):
        assert L.b200va_mxfp8_scale_bytes(1000, block) == 0
