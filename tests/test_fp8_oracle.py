"""CPU checks of oracle/fp8_exact.py, the reference of b200va_quantize_fp8 and b200va_dequantize_fp8, and of the FP8
kernels' SASS.

- The decode tables against the format definitions in `Fraction`, and against torch's float8 -> float32 for all 256
  patterns of each format.
- quantize against a search of the table of finite values in `Fraction` (nearest value, ties to the even
  significand, the largest finite value beyond it) for every source, both formats and several k, on random bit
  patterns, finite values and the adversarial sets; zeros, infinities and NaNs by class and sign.
- quantize against torch's cast from f32 below each format's overflow midpoint (464 for E4M3, 61440 for E5M2).  From
  the midpoint on, torch's CPU cast gives NaN (E4M3) or inf (E5M2) where the contract saturates.
- The f64 double-rounding traps have teeth: RN to f32 and then RN to FP8 gives other bits on them, while round-to-odd
  to f32 and then RN (the kernels' path, written here in numpy) gives the reference's bits.
- dequantize against `Fraction` rounded once by `stream_exact.round_fraction`.
- The SASS of both libraries: 4 + 4 FP8 kernels, each with the bodies of both formats; the quantize kernels round
  with F2FP.SATFINITE.{E4M3,E5M2}; the f64-source ones reach f32 with F2F.F32.F64.RZ and never with an RN
  F2F.F32.F64; dequantize unpacks with F2FP.F16.{E4M3,E5M2} and stores 16-byte vectors.
"""
import math
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X

import k8s_gpu_hpa_b200 as pkg  # noqa: F401  (builds nothing; the session fixture has built the library)
import sass
from k8s_gpu_hpa_b200 import capi

DTYPES = V.DTYPES
KS = (-126, -8, 0, 5, 126)
TORCH8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
OVERFLOW_MIDPOINT = {"e4m3": 464.0, "e5m2": 61440.0}


def is_nan8(p: np.ndarray, fmt: str) -> np.ndarray:
    m = np.asarray(p, np.uint8) & 0x7F
    return m == 0x7F if fmt == "e4m3" else m > 0x7C


def assert_same8(got, want, fmt, what=""):
    g, w = np.asarray(got, np.uint8), np.asarray(want, np.uint8)
    bad = (g != w) & ~(is_nan8(g, fmt) & is_nan8(w, fmt))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} mismatches, first at {i}: got {g[i]:#04x} want {w[i]:#04x}")


PATTERN = {f: {float(v): p for p, v in enumerate(F.DECODE[f].tolist()) if not math.isnan(v)} for f in F.FORMATS8}


def fraction_quantize(a: np.ndarray, src: str, fmt: str, k: int) -> np.ndarray:
    """Element by element: NaN gives NaN, +-inf gives +-max finite, +-0 keeps its sign, everything else is the
    exact rational a 2^k searched in the table (nearest_fraction), with a zero result taking a's sign."""
    out = []
    for v in X.widen(a, src).tolist():
        if math.isnan(v):
            out.append(0x7F)
            continue
        if math.isinf(v):
            r = math.copysign(F.MAX_FINITE[fmt], v)
        elif v == 0:
            r = v
        else:
            r = F.nearest_fraction(Fraction(v) * Fraction(2) ** k, fmt)
            if r == 0:
                r = math.copysign(0.0, v)
        out.append(PATTERN[fmt][r] if r != 0 else (0x80 if math.copysign(1, r) < 0 else 0))
    return np.array(out, np.uint8)


def quantize_inputs(src: str, fmt: str, k: int, n: int, seed: int) -> dict:
    rng = np.random.default_rng([seed, DTYPES.index(src), F.FORMATS8.index(fmt), k + 200])
    sets = {"random bits": V.random_bits(src, n, rng),
            "finite": X.finite(src, n, rng, min(F.MAX_FINITE[fmt] * 2.0 ** -k / 8, 2.0 ** 100))}
    rel = 2.0 ** -40 if src == "f64" else 2.0 ** -16
    for name, x in F.adversarial(fmt, rel).items():
        sets[name] = F.source_values(x, src, k)
    return sets


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_decode_table_against_the_format_definition_and_torch(fmt):
    prec, emin, eb, mb, top, _ = F.SPEC[fmt]
    d = F.DECODE[fmt]
    for p in range(256):
        s, e, m = p >> 7, (p >> mb) & ((1 << eb) - 1), p & ((1 << mb) - 1)
        nan = (e == (1 << eb) - 1) and (m == (1 << mb) - 1 if fmt == "e4m3" else m != 0)
        if nan:
            assert math.isnan(d[p]), p
            continue
        if fmt == "e5m2" and e == 31:
            assert d[p] == (-math.inf if s else math.inf), p
            continue
        v = Fraction(m, 1 << mb) * Fraction(2) ** emin if e == 0 else (1 + Fraction(m, 1 << mb)) * Fraction(2) ** (e - (1 - emin))
        assert Fraction(d[p]) == (-v if s else v) and math.copysign(1, d[p]) == (-1 if s else 1), p
    assert d[top] == F.MAX_FINITE[fmt] and F.values(fmt)[-1] == F.MAX_FINITE[fmt]
    t = torch.arange(256, dtype=torch.uint8).view(TORCH8[fmt]).float().numpy().astype(np.float64)
    same = (t.view(np.uint64) == d.view(np.uint64)) | (np.isnan(t) & np.isnan(d))
    assert same.all(), np.flatnonzero(~same)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_equals_the_nearest_finite_value_in_fractions(src, fmt, k):
    for name, a in quantize_inputs(src, fmt, k, 600, 1).items():
        assert_same8(F.quantize(a, src, fmt, k), fraction_quantize(a, src, fmt, k), fmt, f"{src}->{fmt} k={k} {name}")


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", DTYPES)
def test_zeros_infinities_and_nans(src, fmt):
    x = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e-30, -1e-30])
    a = x.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(x, src)
    top = F.SPEC[fmt][4]
    for k in KS:
        got = F.quantize(a, src, fmt, k)
        assert got[:4].tolist() == [0x00, 0x80, top, 0x80 | top], (k, got)
        assert is_nan8(got[4:6], fmt).all()
        if k <= 0:
            assert got[6:].tolist() == [0x00, 0x80]
    nans = X.nan_payloads(src, 3000, 2)
    assert (is_nan8(F.quantize(nans, src, fmt, 0), fmt) == np.isnan(X.widen(nans, src))).all()


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_quantize_equals_torch_below_the_overflow_midpoint(fmt):
    """torch's CPU cast from f32 rounds once to nearest-even, but from the overflow midpoint on it gives NaN (E4M3)
    or inf (E5M2) where the contract saturates: the comparison stops just below that midpoint."""
    rng = np.random.default_rng(5)
    a = np.concatenate([V.random_bits("f32", 200_000, rng), F.adversarial(fmt, 2.0 ** -16)["midpoints"].astype(np.float32),
                        np.arange(1 << 16, dtype=np.uint32).astype(np.float32) * np.float32(2.0 ** -20)])
    a = a[~(np.abs(a) >= OVERFLOW_MIDPOINT[fmt])]                   # keeps NaNs
    want = torch.from_numpy(a).to(TORCH8[fmt]).view(torch.uint8).numpy()
    assert_same8(F.quantize(a, "f32", fmt, 0), want, fmt, f"f32->{fmt} vs torch")
    at = np.array([OVERFLOW_MIDPOINT[fmt]], np.float32)
    assert F.quantize(at, "f32", fmt, 0)[0] == F.SPEC[fmt][4]       # where torch stops agreeing: saturation


def round_to_odd_f32(x: np.ndarray) -> np.ndarray:
    """f64 -> f32 with round-to-odd: toward zero, then the last bit set when that was inexact (as the kernels do
    with cvt.rz.f32.f64)."""
    with np.errstate(all="ignore"):
        r = x.astype(np.float32)                                     # RN
        over = np.abs(r.astype(np.float64)) > np.abs(x)
        r = np.where(over, np.nextafter(r, np.float32(0)), r)         # toward zero
        r = np.where(np.isinf(r) & np.isfinite(x), np.copysign(np.float32(np.finfo(np.float32).max), x), r)
        u = r.astype(np.float32).view(np.uint32)
        inexact = (r.astype(np.float64) != x) & ~np.isnan(x)
        return (u | inexact.astype(np.uint32)).view(np.float32)


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_double_rounding_traps_have_teeth(fmt):
    x = F.double_rounding_traps(fmt)
    want = F.quantize(x, "f64", fmt, 0)
    assert_same8(want, fraction_quantize(x, "f64", fmt, 0), fmt, "traps")
    with np.errstate(all="ignore"):
        via_rn = F.quantize(x.astype(np.float32), "f32", fmt, 0)
    differ = via_rn != want
    assert differ.mean() > 0.3, differ.mean()          # where the tie to even goes against the offset
    assert_same8(F.quantize(round_to_odd_f32(x), "f32", fmt, 0), want, fmt, "round-to-odd, then RN")
    for k in (-126, 5, 126):                            # the same with a scale: a = x 2^-k, f64 holds it exactly
        a = F.source_values(x, "f64", k)
        assert_same8(F.quantize(a, "f64", fmt, k), want, fmt, f"k={k}")
        prod = np.ldexp(a, k)
        assert_same8(F.quantize(round_to_odd_f32(prod), "f32", fmt, 0), want, fmt, f"round-to-odd k={k}")


def test_amax():
    a = np.array([1.0, -3.5, 2.0], np.float32)
    assert F.amax(a, "f32") == 3.5 and F.amax(a, "f32", 7.0) == 7.0
    assert math.isnan(F.amax(np.array([1.0, np.nan], np.float32), "f32"))
    assert F.amax(np.array([-0.0]), "f64") == 0.0 and math.isinf(F.amax(np.array([-np.inf]), "f64"))
    assert F.amax(V.round_f64(np.array([-65504.0, 1.0]), "f16"), "f16") == 65504.0


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("dst", DTYPES)
def test_dequantize_equals_fraction_rounded_once(fmt, dst):
    bits = np.arange(256, dtype=np.uint8)
    for k in (-126, -1, 0, 1, 126):
        got = F.dequantize(bits, fmt, dst, k)
        want = []
        for v in F.DECODE[fmt].tolist():
            if math.isnan(v) or math.isinf(v) or v == 0:
                want.append(v)
            else:
                want.append(X.round_fraction(Fraction(v) * Fraction(2) ** -k, dst))
        w = np.array(want, np.float64)
        g = X.widen(got, dst)
        same = (g.view(np.uint64) == w.view(np.uint64)) | (np.isnan(g) & np.isnan(w))
        assert same.all(), (fmt, dst, k, np.flatnonzero(~same)[:5])


def test_quantize_then_dequantize_gives_the_fp8_values_scaled_back():
    rng = np.random.default_rng(9)
    for fmt in F.FORMATS8:
        for k in (-8, 0, 5):
            a = X.finite("f64", 5000, rng, F.MAX_FINITE[fmt] * 2.0 ** -k / 4)
            q = F.quantize(a, "f64", fmt, k)
            assert (F.dequantize(q, fmt, "f64", k) == np.ldexp(F.DECODE[fmt][q], -k)).all()


# ------------------------------------------------------------------------------------------- SASS
def _functions(path: str) -> dict[str, str]:
    return {fn: body for fn, body in sass.functions(path).items() if re.match(r"_ZN6b200va\d+fp8_", fn)}


@pytest.mark.parametrize("path", ["production", "tune"])
def test_fp8_kernels_in_the_sass(path):
    """One kernel per non-FP8 type and direction (4 + 4), each carrying the bodies of both formats."""
    fns = _functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH)
    quant = {fn: b for fn, b in fns.items() if "fp8_quant_vec" in fn}
    deq = {fn: b for fn, b in fns.items() if "fp8_dequant_vec" in fn}
    assert len(quant) == 4 and len(deq) == 4 and len(fns) == 8, sorted(fns)
    for fn, body in quant.items():
        src = int(re.search(r"ILi(\d)EE", fn).group(1))
        for f8 in ("E4M3", "E5M2"):
            assert f"F2FP.SATFINITE.{f8}.F32" in body, (fn, f8)
        assert "LDG.E.128" in body and "STG.E.NA.128" in body, fn
        if src == 1:
            assert "F2F.F32.F64.RZ" in body, fn
            assert not re.search(r"F2F\.F32\.F64(?!\.RZ)", body), fn
        ops = re.findall(r"\b(ACQBULK|ATOMG\S*|RED\S*)\b", body)
        assert ops[0] == "ACQBULK" and sum(o.startswith(("ATOMG", "RED")) for o in ops) == 1, (fn, ops)
    for fn, body in deq.items():
        dst = int(re.search(r"ILi(\d)EE", fn).group(1))
        for f8 in ("E4M3", "E5M2"):
            assert f"F2FP.F16.{f8}.UNPACK_B" in body, (fn, f8)
        stores = re.findall(r"\b(STG\.E\S*)", body)
        assert "STG.E.NA.128" in stores, (fn, stores)
        assert set(stores) - {"STG.E.NA.128"} == {{0: "STG.E", 1: "STG.E.64", 2: "STG.E.U16", 3: "STG.E.U16"}[dst]}, (fn, stores)


def test_fp8_kernels_do_not_spill():
    """ptxas -v would say so; the SASS says it too: no local-memory access in any FP8 kernel."""
    for path in (capi.LIB_PATH, capi.TUNE_LIB_PATH):
        for fn, body in _functions(path).items():
            assert not re.search(r"\b(LDL|STL)\b", body), fn
