"""CPU checks of oracle/convert_exact.py, the reference of b200va_convert, and of the convert kernels' SASS.

- For all 12 pairs of distinct types, the reference equals `Fraction` rounded once by `stream_exact.round_fraction`
  (code written from the format definitions) on random bit patterns and on the adversarial sets; zeros, infinities
  and NaNs by class and sign.  numpy's casts that round once (f64 -> f32, f32 -> f16, f64 -> f16) and
  stream_exact's f32 -> bf16 give the same bits.
- Double-rounding traps: f64 values just off an f16 or bf16 midpoint that f32 rounds onto it.  Going through f32
  gives other bits on the set, so the set catches a kernel that does.
- The overflow thresholds and the exact ties on them, the smallest subnormal, half of it and the values around
  that tie, signed zeros and NaNs.
- The SASS of libb200va.so: 12 convert kernels; the f64 -> f16/bf16 ones round in one F2F from f64; 16-byte loads
  and stores; nothing but the trigger and the L2 prefetch ahead of griddepcontrol.wait.
"""
import math
import re
from fractions import Fraction

import numpy as np
import pytest

from oracle import convert_exact as V
from oracle import stream_exact as X

import k8s_gpu_hpa_b200 as pkg  # noqa: F401  (builds nothing; the session fixture has built the library)
import sass
from k8s_gpu_hpa_b200 import capi

PAIRS = V.PAIRS


def bits_of(x: np.ndarray, dtype: str) -> np.ndarray:
    return np.ascontiguousarray(x).view(X.BITS[dtype][0])


def fraction_reference(a: np.ndarray, src: str, dst: str) -> np.ndarray:
    """Element by element: the exact rational of each finite nonzero input rounded once by round_fraction;
    zeros and infinities keep their sign; NaN gives the reference's quiet NaN."""
    x = X.widen(a, src)
    ut, eb, mb = X.BITS[dst]
    out = []
    for v in x.tolist():
        if math.isnan(v):
            r = float("nan")
        elif v == 0 or math.isinf(v):
            r = v
        else:
            r = X.round_fraction(Fraction(v), dst)
        out.append(r)
    r = np.array(out, np.float64)
    if dst == "f64":
        return r
    if dst == "f32":
        return r.astype(np.float32)
    if dst == "f16":
        return r.astype(np.float16).view(np.uint16)                     # exact: every r is an f16 value
    return (r.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)   # exact: every r is a bf16 value


def assert_same(got, want, dtype, what=""):
    g, w = bits_of(got, dtype), bits_of(want, dtype)
    ng = np.isnan(X.widen(got, dtype))
    nw = np.isnan(X.widen(want, dtype))
    bad = (g != w) & ~(ng & nw)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} mismatches, first at {i}: got {g[i]:#x} want {w[i]:#x}")


def adversarial(src: str, n: int, seed: int) -> dict:
    rng = np.random.default_rng(seed)
    sets = {"random bits": V.random_bits(src, n, rng), "edges": X.edge_values(src, n, seed),
            "finite": X.finite(src, n, rng), "nan payloads": X.nan_payloads(src, n, seed)}
    if src == "f64":
        for dst in ("f16", "bf16"):
            sets[f"double rounding traps {dst}"] = V.double_rounding_traps(dst, n, seed)
    return sets


@pytest.mark.parametrize("src,dst", PAIRS)
def test_reference_equals_fraction_rounded_once(src, dst):
    for name, a in adversarial(src, 3000, 7).items():
        assert_same(V.convert(a, src, dst), fraction_reference(a, src, dst), dst, f"{src}->{dst} {name}")


@pytest.mark.parametrize("src,dst", [("f64", "f32"), ("f32", "f16"), ("f64", "f16"), ("f32", "bf16")])
def test_second_opinions_that_round_once(src, dst):
    """numpy's casts round once for these pairs; stream_exact.narrow is the integer RNE of f32 -> bf16."""
    rng = np.random.default_rng(3)
    a = np.concatenate([V.random_bits(src, 200_000, rng), X.edge_values(src, 20_000, 4)])
    if src == "f32":
        highs = np.arange(0, 1 << (8 + X.FORMATS[dst][0]), 5, dtype=np.uint64)     # sign, exponent, kept bits
        a = np.concatenate([a, V.rounding_patterns(src, dst, highs)])
    with np.errstate(all="ignore"):
        if dst == "bf16":
            second = X.narrow(a, dst)
        else:
            second = a.astype(np.float16).view(np.uint16) if dst == "f16" else a.astype(np.float32)
    assert_same(V.convert(a, src, dst), second, dst, f"{src}->{dst}")


@pytest.mark.parametrize("dst", ["f16", "bf16"])
def test_double_rounding_traps_catch_a_conversion_through_f32(dst):
    x = V.double_rounding_traps(dst, 4096, 11)
    want = V.convert(x, "f64", dst)
    assert_same(want, fraction_reference(x, "f64", dst), dst, "traps")
    with np.errstate(all="ignore"):
        via_f32 = V.convert(x.astype(np.float32), "f32", dst)
    differ = bits_of(via_f32, dst) != bits_of(want, dst)
    assert differ.mean() > 0.3, differ.mean()          # about half: where the tie goes to even against the offset
    assert differ[:8].all()                            # just below the overflow midpoint: f32 rounds onto it, then to inf


def one(x: float, src: str, dst: str) -> int:
    a = np.array([x], np.float64).astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(np.array([x]), src)
    return int(bits_of(V.convert(a, src, dst), dst)[0])


def test_overflow_thresholds_and_their_ties():
    # f16: 65504 is the largest finite value, 65520 the midpoint above it (RNE: to inf, as 65504 is odd)
    for src in ("f32", "f64"):
        assert one(65504.0, src, "f16") == 0x7BFF
        assert one(65520.0, src, "f16") == 0x7C00
        assert one(-65520.0, src, "f16") == 0xFC00
    assert one(65520.0 - 2.0 ** -8, "f32", "f16") == 0x7BFF            # the f32 just below the tie
    assert one(float(np.nextafter(65520.0, 0)), "f64", "f16") == 0x7BFF
    # bf16 from f64 and f32: the largest finite (2 - 2^-7) 2^127, the threshold (2 - 2^-8) 2^127
    T = (2 - 2.0 ** -8) * 2.0 ** 127
    for src in ("f32", "f64"):
        assert one((2 - 2.0 ** -7) * 2.0 ** 127, src, "bf16") == 0x7F7F
        assert one(T, src, "bf16") == 0x7F80
        assert one(-T, src, "bf16") == 0xFF80
    assert one(float(np.nextafter(np.float32(T), np.float32(0))), "f32", "bf16") == 0x7F7F
    assert one(float(np.nextafter(T, 0)), "f64", "bf16") == 0x7F7F
    # f32 from f64: FLT_MAX + ulp/2
    T32 = X.F32_OVERFLOW
    assert one(T32, "f64", "f32") == 0x7F800000
    assert one(float(np.nextafter(T32, 0)), "f64", "f32") == 0x7F7FFFFF
    assert one(-T32, "f64", "f32") == 0xFF800000
    assert one(1e300, "f64", "f16") == 0x7C00 and one(1e300, "f64", "bf16") == 0x7F80


@pytest.mark.parametrize("src,dst", [("f64", "f32"), ("f64", "f16"), ("f64", "bf16"), ("f32", "f16"), ("f32", "bf16")])
def test_smallest_subnormal_half_of_it_and_the_tie_above(src, dst):
    prec, emin, _ = X.FORMATS[dst]
    s = 2.0 ** (emin - prec + 1)                          # the smallest subnormal of dst
    if src == "f32" and s / 2 < 2.0 ** -149:
        pytest.skip("half of it is no f32")
    just_above = s / 2 * (1 + 2.0 ** -12)                  # exact in f32 (quantum 2^-149) and f64
    cases = [(s, 1), (s / 2, 0), (just_above, 1), (s / 2 * (1 - 2.0 ** -12), 0), (1.5 * s, 2), (2.5 * s, 2),
             (3.5 * s, 4)]
    for x, k in cases:
        assert one(x, src, dst) == k, (x, k)
        sign = 1 << (X.BITS[dst][1] + X.BITS[dst][2])
        assert one(-x, src, dst) == sign | k, (-x, k)


@pytest.mark.parametrize("src,dst", PAIRS)
def test_signed_zeros_infinities_and_nans(src, dst):
    a = X.narrow(np.array([0.0, -0.0, np.inf, -np.inf, np.nan], np.float32), src) if src in ("f16", "bf16") else \
        np.array([0.0, -0.0, np.inf, -np.inf, np.nan]).astype(X.STORAGE[src])
    r = X.widen(V.convert(a, src, dst), dst)
    assert r[0] == 0 and math.copysign(1, r[0]) > 0 and r[1] == 0 and math.copysign(1, r[1]) < 0
    assert r[2] == np.inf and r[3] == -np.inf and np.isnan(r[4])
    nans = X.nan_payloads(src, 3000, 2)
    widened = X.widen(nans, src)
    assert (np.isnan(X.widen(V.convert(nans, src, dst), dst)) == np.isnan(widened)).all()


def test_same_type_is_a_bit_copy():
    for dt in V.DTYPES:
        a = X.nan_payloads(dt, 1000, 1)
        assert (bits_of(V.convert(a, dt, dt), dt) == bits_of(a, dt)).all()


def test_rounding_patterns_are_the_decisive_low_parts():
    p = bits_of(V.rounding_patterns("f32", "f16", np.array([0x12345], np.uint64)), "f32")
    assert p.tolist() == [(0x12345 << 13) | lo for lo in (0, 1, 0xFFF, 0x1000, 0x1001, 0x1FFF)]
    assert V.rounding_patterns("f32", "bf16").size == 6 << 16


# ------------------------------------------------------------------------------------------- SASS
def test_convert_kernels_in_the_sass_wait_before_they_release_the_next_launch():
    fns = sass.functions(capi.LIB_PATH)
    names = sorted(fn for fn in fns if re.match(r"_ZN6b200va\d+convert_\w+", fn))
    assert len(names) == 12, names
    code = {"f32": 0, "f64": 1, "f16": 2, "bf16": 3}
    for fn in names:
        body = fns[fn]
        src, dst = (k for c in re.search(r"ILi(\d)ELi(\d)E", fn).groups() for k, v in code.items() if v == int(c))
        ops = re.findall(r"\b(LDG\.E\S*|STG\.E\S*|ACQBULK|UBLKPF\.L2|PREEXIT)\b", body)
        assert ops[:2] == ["UBLKPF.L2", "ACQBULK"] and "PREEXIT" in ops[2:], (fn, ops[:4])   # the trigger after the wait
        assert "LDG.E.128" in ops and any(re.fullmatch(r"STG\.E\S*\.128", o) for o in ops), fn
        if src == "f64" and dst in ("f16", "bf16"):
            want = "F2F.F16.F64" if dst == "f16" else "F2F.BF16.F64"
            assert want in body and "F2F.F32.F64" not in body, fn
