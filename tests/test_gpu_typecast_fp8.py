"""b200va_quantize_fp8 and b200va_dequantize_fp8 on the GPU, element by element against oracle/fp8_exact.py (NaN
matches NaN as a class).  Outputs are poisoned beforehand and guard elements on both sides must keep the poison.

- All 16 pairs at ragged sizes around the group of 16 and the 16-byte edges, at every element offset of A and C
  within 16 bytes: the vector body with every head, and the mixed-phase scalar path.
- All 65536 patterns of f16 and bf16 into both formats at k in {-126, -8, 0, 5, 126}; all 256 patterns of each
  format into every destination at k in {-126, -1, 0, 1, 126} (f16 overflow and subnormal rounding included).
- The adversarial sets (midpoints and their neighbours, the saturation threshold, half the smallest subnormal,
  signed zeros, inf, NaN) from f32 and f64, and the f64 double-rounding traps; NaN payloads and +-inf from every
  source.
- Both sides of the HBM class edge per pair, and a ragged, misaligned n in it; f16 -> E4M3 -> f16 at n = 2^32 + 4099.
- amax: random values and each value class, a NaN, -0, two half-calls against one call, NULL.
- Every rejected argument writes nothing, *d_amax included.
- A stream op -> quantize -> dequantize -> stream op chain on one stream without a host sync; a captured graph
  replayed twice with the amax reset inside it; a quantize tail reading the end of X behind the 2^28 K2d writer of
  test_gpu_pdl_chains.py.
- A profiler trace of the planned kernels, grids and blocks.
This module's name sorts after test_gpu_typecast.py: a module with profiler traces that runs before the parity and
stream modules makes their traces lose kernels (DESIGN.md section 3).
"""
import json
import math

import numpy as np
import pytest

from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va
    from test_gpu_parity import _profiled_kernel_name
    from test_gpu_pdl_chains import LO, M, _chains, _run, env  # noqa: F401  (env: the module-scoped fixture)
    from test_gpu_stream import GUARD, POISON, assert_guards, assert_matches, poisoned, tiled, to_dev
    from test_gpu_typecast import expected_cast_launch

    TORCH = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}
    TORCH8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}

DTYPES = V.DTYPES
FMTS = F.FORMATS8
ES = V.SIZE
DT_CODE = {"f32": 0, "f64": 1, "f16": 2, "bf16": 3}
F8_CODE = {"e4m3": 0, "e5m2": 1}
PAIRS = [("q", t, f) for t in DTYPES for f in FMTS] + [("d", t, f) for t in DTYPES for f in FMTS]
PERIOD = 199_999


# ------------------------------------------------------------------------------------------- helpers
def to_dev8(bits, fmt):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint8)).cuda().view(TORCH8[fmt])


def tiled8(bits, n, fmt):
    t = torch.from_numpy(np.ascontiguousarray(bits, np.uint8)).cuda()
    t = t.repeat(-(-n // t.numel()))[:n] if n > t.numel() else t[:n].contiguous()
    return t.view(TORCH8[fmt])


def poisoned8(n, fmt, off=0):
    buf = torch.empty(GUARD + off + n + GUARD, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    return buf, buf[GUARD + off:GUARD + off + n].view(TORCH8[fmt])


def _nan8(u8, fmt):
    m = u8 & 0x7F
    return m == 0x7F if fmt == "e4m3" else m > 0x7C


def assert_matches8(got, want, fmt, what="", chunk=1 << 30):
    """FP8 bit patterns equal element by element on the device, NaN matching NaN as a class."""
    assert got.numel() == want.numel()
    for lo in range(0, got.numel(), chunk):
        g, w = got[lo:lo + chunk].view(torch.uint8), want[lo:lo + chunk].view(torch.uint8)
        bad = (g != w) & ~(_nan8(g, fmt) & _nan8(w, fmt))
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            raise AssertionError(f"{what}: {int(bad.sum())} mismatches, first at {lo + i} of {got.numel()}: "
                                 f"got {int(g[i]):#04x} want {int(w[i]):#04x}")


def random_fp8(n, rng):
    return rng.integers(0, 256, n, dtype=np.uint16).astype(np.uint8)


def quantize(a, fmt, out, k=0, **kw):
    return va.quantize_fp8(a, TORCH8[fmt], scale_exp=k, out=out, **kw)


def dequantize(a, dst, out, k=0, **kw):
    return va.dequantize_fp8(a, TORCH[dst], scale_exp=k, out=out, **kw)


def check_quant(src, fmt, a_host, a_dev, k=0, off_c=0, what=""):
    n = a_host.size
    buf, out = poisoned8(n, fmt, off_c)
    quantize(a_dev, fmt, out, k)
    torch.cuda.synchronize()
    assert_matches8(out, to_dev8(F.quantize(a_host, src, fmt, k), fmt), fmt, what)
    assert_guards(buf, GUARD + off_c, n, what)


def check_dequant(fmt, dst, bits, a_dev, k=0, off_c=0, what=""):
    n = bits.size
    buf, out = poisoned(n, dst, off_c)
    dequantize(a_dev, dst, out, k)
    torch.cuda.synchronize()
    assert_matches(out, to_dev(F.dequantize(bits, fmt, dst, k), dst), dst, what)
    assert_guards(buf, GUARD + off_c, n, what)


def hbm_n(t):
    """The smallest n in the HBM class of a pair with wide type t: the wide operand holds 2^25 four-byte words."""
    return (1 << 25) * 4 // ES[t]


def _amax_tensor(v=0.0):
    return torch.full((1,), v, dtype=torch.float64, device="cuda")


def _same_f64(got: float, want: float) -> bool:
    return (math.isnan(got) and math.isnan(want)) or np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64)


# ------------------------------------------------------------------------------------------- element offsets
@pytest.mark.parametrize("kind,t,fmt", PAIRS)
def test_sizes_around_the_group_at_every_offset(kind, t, fmt):
    sizes = sorted({0, 1, 2, 3, 7, 15, 16, 17, 31, 33, 47, 4099, 70_001})
    rng = np.random.default_rng([DT_CODE[t], F8_CODE[fmt], kind == "q"])
    total = max(sizes) + 16
    k = 3 if kind == "q" else -3
    if kind == "q":
        host = V.random_bits(t, total, rng)
        want_all = F.quantize(host, t, fmt, k)
        offs_a, offs_c = range(16 // ES[t]), range(16)
    else:
        host = random_fp8(total, rng)
        want_all = F.dequantize(host, fmt, t, k)
        offs_a, offs_c = range(16), range(16 // ES[t])
    for oa in offs_a:
        if kind == "q":
            abuf, _ = poisoned(total, t)
            abuf[GUARD:GUARD + total].copy_(to_dev(host, t))
        else:
            abuf, _ = poisoned8(total, fmt)
            abuf[GUARD:GUARD + total].copy_(torch.from_numpy(host).cuda())
            abuf = abuf.view(TORCH8[fmt])
        for oc in offs_c:
            for n in sizes:
                a, what = abuf[GUARD + oa:GUARD + oa + n], f"{kind} {t} {fmt} n={n} offsets A {oa} C {oc}"
                if kind == "q":
                    buf, out = poisoned8(n, fmt, oc)
                    quantize(a, fmt, out, k)
                    torch.cuda.synchronize()
                    assert_matches8(out, to_dev8(want_all[oa:oa + n], fmt), fmt, what)
                else:
                    buf, out = poisoned(n, t, oc)
                    dequantize(a, t, out, k)
                    torch.cuda.synchronize()
                    assert_matches(out, to_dev(want_all[oa:oa + n], t), t, what)
                assert_guards(buf, GUARD + oc, n, what)


# ------------------------------------------------------------------------------------------- exhaustive and adversarial
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", ["f16", "bf16"])
def test_every_16_bit_pattern(src, fmt):
    x = np.arange(1 << 16, dtype=np.uint16)
    a = to_dev(x, src)
    for k in (-126, -8, 0, 5, 126):
        for off_c in (0, 1):
            check_quant(src, fmt, x, a, k, off_c, f"{src}->{fmt} all patterns, k={k}, C offset {off_c}")


@pytest.mark.parametrize("dst", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_every_fp8_pattern(fmt, dst):
    bits = np.tile(np.arange(256, dtype=np.uint8), 5)      # several groups, so the vector body sees every pattern
    a = to_dev8(bits, fmt)
    for k in (-126, -1, 0, 1, 126):
        for off_c in (0, 1):
            check_dequant(fmt, dst, bits, a, k, off_c, f"{fmt}->{dst} all patterns, k={k}, C offset {off_c}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", ["f32", "f64"])
def test_adversarial_sets_and_double_rounding_traps(src, fmt):
    rel = 2.0 ** -40 if src == "f64" else 2.0 ** -16
    for k in (-126, -8, 0, 5, 126):
        sets = dict(F.adversarial(fmt, rel))
        if src == "f64":
            sets["double rounding traps"] = F.double_rounding_traps(fmt)
        for name, x in sets.items():
            a = F.source_values(x, src, k)
            check_quant(src, fmt, a, to_dev(a, src), k, 0, f"{src}->{fmt} k={k} {name}")
            check_quant(src, fmt, a, to_dev(a, src), k, 3, f"{src}->{fmt} k={k} {name}, C offset 3")


@pytest.mark.parametrize("src", DTYPES)
def test_infinities_and_nans_from_every_source(src):
    x = X.nan_payloads(src, 30_001, 4)
    inf = np.array([np.inf, -np.inf, 0.0, -0.0])
    inf = inf.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(inf, src)
    x = np.concatenate([x, np.tile(inf, 100)])
    for fmt in FMTS:
        for k in (-126, 0, 126):
            check_quant(src, fmt, x, to_dev(x, src), k, 0, f"{src}->{fmt} NaNs and infinities k={k}")


# ------------------------------------------------------------------------------------------- size classes
@pytest.mark.parametrize("kind,t,fmt", PAIRS)
def test_both_sides_of_the_hbm_edge(kind, t, fmt):
    """n = h - 1 and h at aligned pointers, then h + 37 with A and C one element past a 16-byte boundary."""
    h = hbm_n(t)
    big = h + 37
    rng = np.random.default_rng([9, DT_CODE[t], F8_CODE[fmt], kind == "q"])
    k = -2 if kind == "q" else 2
    if kind == "q":
        block = V.random_bits(t, PERIOD, rng)
        a, want = tiled(block, big + 1, t), tiled8(F.quantize(block, t, fmt, k), big + 1, fmt)
    else:
        block = random_fp8(PERIOD, rng)
        a, want = tiled8(block, big + 1, fmt), tiled(F.dequantize(block, fmt, t, k), big + 1, t)
    for n, off in ((h - 1, 0), (h, 0), (big, 1)):
        what = f"{kind} {t} {fmt} n={n} offset {off}"
        if kind == "q":
            buf, out = poisoned8(n, fmt, off)
            quantize(a[off:off + n], fmt, out, k)
            torch.cuda.synchronize()
            assert_matches8(out, want[off:off + n], fmt, what)
        else:
            buf, out = poisoned(n, t, off)
            dequantize(a[off:off + n], t, out, k)
            torch.cuda.synchronize()
            assert_matches(out, want[off:off + n], t, what)
        assert_guards(buf, GUARD + off, n, what)
        del buf, out


def test_f16_e4m3_f16_beyond_32_bit_offsets():
    """n = 2^32 + 4099: element 2^31 is byte 2^32 of the f16 arrays and element 2^32 needs a 64-bit index.  The input
    repeats a random block of odd length, so a wrapped index or byte offset gives another element."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * 2 * n + 2 * n + (4 << 30):
        pytest.skip("needs ~28 GiB of free device memory")
    block = V.random_bits("f16", PERIOD, np.random.default_rng(31))
    q_block = F.quantize(block, "f16", "e4m3", 4)
    a = tiled(block, n, "f16")
    q = torch.empty(n, dtype=torch.uint8, device="cuda")
    q.fill_(POISON)
    quantize(a, "e4m3", q.view(torch.float8_e4m3fn), 4)
    del a
    want = tiled8(q_block, n, "e4m3")
    assert_matches8(q.view(torch.float8_e4m3fn), want, "e4m3", "quantize, n = 2^32 + 4099")
    del want
    c = torch.empty(n, dtype=torch.float16, device="cuda")
    c.view(torch.uint8).fill_(POISON)
    dequantize(q.view(torch.float8_e4m3fn), "f16", c, 4)
    want = tiled(F.dequantize(q_block, "e4m3", "f16", 4), n, "f16")
    for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - 8192):
        assert_matches(c[lo:lo + 8192], want[lo:lo + 8192], "f16", f"window at {lo}")
    assert_matches(c, want, "f16", "dequantize, n = 2^32 + 4099")


# ------------------------------------------------------------------------------------------- amax
@pytest.mark.parametrize("src", DTYPES)
def test_amax(src):
    rng = np.random.default_rng(DT_CODE[src])
    out = torch.empty(300_007, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    out5 = torch.empty(300_007, dtype=torch.uint8, device="cuda").view(torch.float8_e5m2)
    finite = X.finite(src, 300_007, rng, 50.0)
    edges = X.edge_values(src, 300_007, 3)
    edges = edges[~np.isnan(X.widen(edges, src))]
    z = np.array([-0.0, -0.0, -0.0])
    neg_zero = z.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(z, src)
    with_nan = finite.copy()
    nan =np.array([np.nan]).astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(np.array([np.nan]), src)
    with_nan[123_457] = nan[0]
    big = (np.array([3.0, -1e300, 7.0]) if src == "f64" else
           np.array([3.0, -6e4, 7.0]).astype(np.float32) if src == "f32" else V.round_f64(np.array([3.0, -6e4, 7.0]), src))
    for name, x in (("finite", finite), ("value classes without NaN", edges), ("-0", neg_zero), ("one NaN", with_nan),
                    ("a negative maximum", big)):
        a = to_dev(x, src)
        m = _amax_tensor()
        quantize(a, "e4m3", out[:x.size], 0, amax=m)
        got, want = float(m.item()), F.amax(x, src)
        assert _same_f64(got, want), (src, name, got, want)
        if name == "-0":
            assert np.float64(got).view(np.uint64) == 0, "amax of -0 is +0"
        # two half-calls max-accumulate into the bits of one call
        h = x.size // 2
        m2 = _amax_tensor()
        quantize(a[:h], "e5m2", out5[:h], 5, amax=m2)
        quantize(a[h:], "e5m2", out5[h:x.size], -5, amax=m2)
        assert _same_f64(float(m2.item()), want), (src, name, "halves")
    # NULL: the quantize is the same, and nothing is written to any amax
    a = to_dev(finite, src)
    m = _amax_tensor(-7.0)
    quantize(a, "e4m3", out, 0)
    torch.cuda.synchronize()
    assert float(m.item()) == -7.0
    assert_matches8(out, to_dev8(F.quantize(finite, src, "e4m3", 0), "e4m3"), "e4m3", "amax NULL")


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A, n = buf.data_ptr() + 4096, 1000
    C_, M_ = A + 16384, A + 32768                       # an output and an amax slot away from A
    F32, F64, F16, BF16 = 0, 1, 2, 3
    E4, E5 = capi.F8_E4M3, capi.F8_E5M2
    q = [
        ((4, A, E4, C_, n, 0, M_), capi.ERR_VARIANT), ((-1, A, E4, C_, n, 0, M_), capi.ERR_VARIANT),
        ((F32, A, 2, C_, n, 0, M_), capi.ERR_VARIANT), ((F32, A, -1, C_, n, 0, M_), capi.ERR_VARIANT),
        ((F32, A, E4, C_, n, 127, M_), capi.ERR_INVALID), ((F32, A, E4, C_, n, -127, M_), capi.ERR_INVALID),
        ((F32, None, E4, C_, n, 0, M_), capi.ERR_INVALID), ((F32, A, E5, None, n, 0, M_), capi.ERR_INVALID),
        ((F32, A, E4, C_, (1 << 40) + 1, 0, M_), capi.ERR_INVALID),
        ((F32, A + 2, E4, C_, n, 0, M_), capi.ERR_ALIGN), ((F64, A + 4, E4, C_, n, 0, M_), capi.ERR_ALIGN),
        ((F16, A + 1, E5, C_, n, 0, M_), capi.ERR_ALIGN), ((F32, A, E4, C_, n, 0, M_ + 4), capi.ERR_ALIGN),
        ((F32, A, E4, A, n, 0, M_), capi.ERR_OVERLAP), ((F32, A, E4, A + 4 * n - 1, n, 0, M_), capi.ERR_OVERLAP),
        ((BF16, A + 8, E4, A, n, 0, M_), capi.ERR_OVERLAP),
        ((F32, A, E4, C_, n, 0, A + 8), capi.ERR_OVERLAP), ((F32, A, E4, C_, n, 0, C_ + n - 8), capi.ERR_OVERLAP),
        ((F64, A, E4, C_, n, 0, A + 8 * n - 8), capi.ERR_OVERLAP),
    ]
    d = [
        ((E4, A, 4, C_, n, 0), capi.ERR_VARIANT), ((2, A, F32, C_, n, 0), capi.ERR_VARIANT),
        ((E5, A, F16, C_, n, 127), capi.ERR_INVALID), ((E5, A, F16, C_, n, -127), capi.ERR_INVALID),
        ((E4, None, F32, C_, n, 0), capi.ERR_INVALID), ((E4, A, F32, None, n, 0), capi.ERR_INVALID),
        ((E4, A, F32, C_, (1 << 40) + 1, 0), capi.ERR_INVALID),
        ((E4, A, F32, C_ + 2, n, 0), capi.ERR_ALIGN), ((E5, A, F64, C_ + 4, n, 0), capi.ERR_ALIGN),
        ((E4, A, BF16, C_ + 1, n, 0), capi.ERR_ALIGN),
        ((E4, A, F32, A, n, 0), capi.ERR_OVERLAP), ((E4, A, F16, A - 2 * n + 2, n, 0), capi.ERR_OVERLAP),
        ((E5, A + 8192, F64, A + 200, n, 0), capi.ERR_OVERLAP),
    ]
    for args, code in q:
        assert L.b200va_quantize_fp8(*args, None) == code, (args, code)
    for args, code in d:
        assert L.b200va_dequantize_fp8(*args, None) == code, (args, code)
    assert L.b200va_quantize_fp8(F32, None, E4, None, 0, 0, None, None) == capi.OK      # n = 0: nothing to do
    assert L.b200va_quantize_fp8(F32, A, E4, C_, 0, 0, M_, None) == capi.OK
    assert L.b200va_dequantize_fp8(E5, None, F64, None, 0, 0, None) == capi.OK
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == POISON).all(), "a rejected or empty call wrote to device memory"
    # right behind each other: no overlap, and the call runs
    assert L.b200va_quantize_fp8(F32, A, E4, A + 4 * n, n, 0, A + 5 * n + 8 - (A + 5 * n) % 8, None) == capi.OK
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- stream order
def test_stream_op_quantize_dequantize_stream_op_on_one_stream():
    """Ten rounds on one stream without a host sync: b = s a (b200va_stream), q = quantize(b, k) with amax,
    c = dequantize(q, k), d_r = c / 2 (b200va_stream); a different s per round, at an L2-resident size and in the
    HBM class of the pair."""
    st = torch.cuda.Stream()
    for src, fmt, dst, k in (("f32", "e4m3", "f32", 4), ("bf16", "e5m2", "f16", -3), ("f64", "e4m3", "bf16", 0)):
        period = 49_999
        a0 = X.finite(src, period, np.random.default_rng(DT_CODE[src]), 8.0)
        scalars = [1.0 + r / 8 for r in range(10)]
        wants, amaxes = [], []
        for s in scalars:
            b = X.stream("scale", src, a0, None, s)
            c = F.dequantize(F.quantize(b, src, fmt, k), fmt, dst, k)
            wants.append(X.stream("scale", dst, c, None, 0.5))
            amaxes.append(F.amax(b, src))
        for n in ((1 << 20) + 5, hbm_n(src) + 5):
            a = tiled(a0, n, src)
            b = torch.empty_like(a)
            q = torch.empty(n, dtype=TORCH8[fmt], device="cuda")
            c = torch.empty(n, dtype=TORCH[dst], device="cuda")
            ds = [torch.empty_like(c) for _ in scalars]
            ms = torch.zeros(len(scalars), dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            for r, (s, d) in enumerate(zip(scalars, ds)):
                va.stream("scale", a, None, b, scalar=s, stream=st)
                quantize(b, fmt, q, k, amax=ms[r:r + 1], stream=st)
                dequantize(q, dst, c, k, stream=st)
                va.stream("scale", c, None, d, scalar=0.5, stream=st)
            st.synchronize()
            for r, (d, w) in enumerate(zip(ds, wants)):
                assert_matches(d, tiled(w, n, dst), dst, f"{src}->{fmt}->{dst} n={n} round {r}")
                assert _same_f64(float(ms[r].item()), amaxes[r]), (src, n, r)
            del a, b, q, c, ds


def test_captured_graph_replays_with_the_amax_reset_inside():
    cases = []
    for src, fmt, dst in (("f32", "e5m2", "f64"), ("f64", "e4m3", "f16"), ("bf16", "e4m3", "f32")):
        x = V.random_bits(src, 100_003, np.random.default_rng(DT_CODE[src] + 40))
        bq, q = poisoned8(x.size, fmt, 1)
        bc, c = poisoned(x.size, dst, 3)
        cases.append((src, fmt, dst, x, to_dev(x, src), bq, q, bc, c, _amax_tensor(5.0)))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for src, fmt, dst, _, a, _, q, _, c, m in cases:
                m.zero_()
                quantize(a, fmt, q, -4, amax=m)
                dequantize(q, dst, c, -4)
    torch.cuda.synchronize()
    for r in range(2):
        for case in cases:
            case[5].fill_(POISON)
            case[7].view(torch.uint8).fill_(POISON)
            case[9].fill_(1e300)
        g.replay()
        torch.cuda.synchronize()
        for src, fmt, dst, x, _, bq, q, bc, c, m in cases:
            what = f"{src}->{fmt}->{dst} replay {r}"
            qb = F.quantize(x, src, fmt, -4)
            assert_matches8(q, to_dev8(qb, fmt), fmt, what)
            assert_matches(c, to_dev(F.dequantize(qb, fmt, dst, -4), dst), dst, what)
            assert_guards(bq, GUARD + 1, x.size, what)
            assert_guards(bc, GUARD + 3, x.size, what)
            assert _same_f64(float(m.item()), F.amax(x, src)), what


def test_quantize_tail_reads_what_the_writer_wrote(env):
    """test_gpu_pdl_chains.py's chains (the 2^28 K2d writer of X, then 0-3 middle launches) with a quantize of the
    end of X, with amax, as the tail: its bytes and its amax against the exact window."""
    middles, chains = _chains(env)
    q = torch.empty(M + 1, dtype=torch.float8_e4m3fn, device="cuda")[1:]
    m = _amax_tensor()
    want = F.quantize(env["ref_window"], "f32", "e4m3", 2)
    want_amax = F.amax(env["ref_window"], "f32")

    def tail(w):
        m.zero_()
        quantize(w, "e4m3", q, 2, amax=m)

    failures = []
    for names in chains:
        q.view(torch.uint8).fill_(POISON)
        _run(env, middles, names, tail)
        got = q.view(torch.uint8).cpu().numpy()
        bad = np.flatnonzero(got != want)
        amax = float(m.item())
        if bad.size or not _same_f64(amax, want_amax):
            failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> quantize: {bad.size} bytes differ, "
                            f"amax {amax!r} want {want_amax!r}")
    assert not failures, "\n".join(failures)
    assert LO + M < env["X"].numel()


# ------------------------------------------------------------------------------------------- trace
def test_trace_shows_the_planned_kernels(tmp_path):
    """Per pair: n = 1000, the HBM class, n = 1001 in mixed phase and an odd n with a head.  Under the profiler the
    kernels after the marker are exactly the planned ones with their grid and block."""
    nmax = max(hbm_n(t) for t in DTYPES) + 64
    wide = {t: torch.zeros(nmax, dtype=TORCH[t], device="cuda") for t in DTYPES}
    narrow = {f: torch.zeros(nmax, dtype=torch.uint8, device="cuda").view(TORCH8[f]) for f in FMTS}
    narrow_out = {f: torch.zeros(nmax, dtype=torch.uint8, device="cuda").view(TORCH8[f]) for f in FMTS}
    wide_out = {t: torch.zeros(nmax, dtype=TORCH[t], device="cuda") for t in DTYPES}
    plan, want = [], []
    for kind, t, fmt in PAIRS:
        for n, oa, oc in ((1000, 0, 0), (hbm_n(t), 0, 0), (1001, 0, 1), (4099, 1, 1)):
            if kind == "q":
                a, c = wide[t][oa:oa + n], narrow_out[fmt][oc:oc + n]
                launch = (f"fp8_quant_vec<{DT_CODE[t]}>", ES[t], 1, n, a.data_ptr(), c.data_ptr())
            else:
                a, c = narrow[fmt][oa:oa + n], wide_out[t][oc:oc + n]
                launch = (f"fp8_dequant_vec<{DT_CODE[t]}>", 1, ES[t], n, a.data_ptr(), c.data_ptr(), ES[t])
            plan.append((kind, t, fmt, a, c))
            want.append(expected_cast_launch(*launch))
    marker = torch.zeros(1, device="cuda")
    amax = _amax_tensor()
    torch.cuda.synchronize()

    def run_plan():
        for kind, t, fmt, a, c in plan:
            if kind == "q":
                quantize(a, fmt, c, 0, amax=amax)
            else:
                dequantize(a, t, c, 0)
        torch.cuda.synchronize()

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_plan()
        marker.fill_(1.0)
        torch.cuda.synchronize()
        run_plan()
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    events = sorted((e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset")),
                    key=lambda e: e["ts"])
    mk = max(i for i, e in enumerate(events) if "fp8_" not in e["name"])
    assert events[mk].get("cat") == "kernel" and "ill" in events[mk]["name"], events[mk]["name"]
    got = [(_profiled_kernel_name(e["name"]), e["args"]["grid"][0], e["args"]["block"][0]) for e in events[mk + 1:]]
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w, p in zip(got, want, plan):
        assert g == w, (p[:3], g, w)
