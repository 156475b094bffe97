"""b200va_quantize_fp8_auto and b200va_dequantize_fp8_auto on the GPU, bit for bit against tests/fp8_auto_exact.py:
the FP8 bytes (NaN matches NaN as a class), *d_scale_exp and the bits of *d_amax.  Outputs are poisoned beforehand
and guard elements on both sides must keep the poison.

- Every source type and format at margins 0, 1 and 3: sizes 0, 1, 15, 16, 17 and 2^20 + 3, random bit patterns
  (NaN and +-inf among them), a ragged size in the HBM class at an offset, and f16 -> E4M3 -> f16 at n = 2^32 + 4099.
- Every element offset of A and C within 16 bytes, which covers the amax pass's own head.
- Value classes: all zeros (k = 126), +-inf and NaN mixed in, f64 beyond the f32 range, a running *d_amax larger
  than the tensor's, and *d_amax seeded with NaN, +inf, -1.0 or -0.0 (k = 0).
- The round trip equals the FP8 values scaled back, byte for byte what b200va_dequantize_fp8 gives with the host k;
  a *d_scale_exp of 127, -127 or INT32_MIN gives all NaN.
- Every rejected argument writes nothing: C, *d_amax and *d_scale_exp keep their poison.
- One captured graph with the amax reset, the quantize and the dequantize, replayed with inputs whose magnitudes
  move by 2^20 between replays: each replay's k, amax and bytes follow its input with no host read between passes.
- A stream op -> quantize -> dequantize -> stream op chain on one stream, with k changing every round.
- A profiler trace: the amax pass and the quantize pass of fp8_quant_vec and one fp8_dequant_vec per call, with
  their planned grids and blocks, and nothing else.
This module's name sorts after test_gpu_typecast.py, as test_gpu_typecast_fp8.py's does (DESIGN.md section 3).
"""
import numpy as np
import pytest

import fp8_auto_exact as A
from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import (DT_CODE, ES, F8_CODE, GUARD, POISON, TORCH, assert_guards, assert_matches,
                             expected_cast_launch, hbm_n, kernels_after_marker, poisoned, tiled, to_dev)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = V.DTYPES
FMTS = F.FORMATS8
PERIOD = 199_999
K_POISON = -999                 # what *d_scale_exp holds before a call


# ------------------------------------------------------------------------------------------- helpers
def storage(x, src):
    """f64 values as src storage."""
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        return x.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(x, src)


def amax_tensor(v=0.0):
    return torch.full((1,), v, dtype=torch.float64, device="cuda")


def k_tensor(v=K_POISON):
    return torch.full((1,), v, dtype=torch.int32, device="cuda")


def amax_bits(m) -> int:
    return int(m.view(torch.int64).item()) & ((1 << 64) - 1)


def check_auto(src, fmt, host, a, margin=0, acc=0.0, off_c=0, what=""):
    """quantize_fp8_auto of the device copy a of host into a poisoned C with *d_amax = acc: bytes, k and amax
    against the reference, guards kept.  Returns (reference bytes, k)."""
    n = host.size
    what = f"{src}->{fmt} margin {margin} n={n} {what}"
    buf, out = poisoned(n, fmt, off_c)
    m, s = amax_tensor(acc), k_tensor()
    q, s2 = va.quantize_fp8_auto(a, TORCH[fmt], margin=margin, amax=m, scale_exp=s, out=out)
    assert q is out and s2 is s
    torch.cuda.synchronize()
    want, k, wm = A.quantize_auto(host, src, fmt, margin, acc)
    assert_matches(out, to_dev(want, fmt), fmt, what)
    assert_guards(buf, GUARD + off_c, n, what)
    if n == 0:                                  # nothing launched: nothing written
        k, wm = K_POISON, acc
    assert int(s.item()) == k, (what, int(s.item()), k)
    assert amax_bits(m) == A.f64_bits(wm), (what, float(m.item()), wm)
    return want, k


# ------------------------------------------------------------------------------------------- types, sizes, margins
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_sizes_and_margins(src, fmt):
    rng = np.random.default_rng([DT_CODE[src], F8_CODE[fmt]])
    top = 4.0 if src == "f16" else 2.0 ** 12
    for margin in (0, 1, 3):
        for i, n in enumerate((0, 1, 15, 16, 17, (1 << 20) + 3)):
            scale = top ** ((i % 3) - 1)        # magnitudes that move k both ways
            host = X.finite(src, n, rng, scale)
            check_auto(src, fmt, host, to_dev(host, src), margin, what=f"finite, scale {scale}")
        host = V.random_bits(src, 4099, rng)
        check_auto(src, fmt, host, to_dev(host, src), margin, what="random bit patterns")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_a_ragged_size_in_the_hbm_class(src, fmt):
    """n = hbm_n + 37 with A and C one element past a 16-byte boundary; the input repeats a block of odd length, so
    the tensor's amax is the block's."""
    n = hbm_n(ES[src]) + 37
    block = X.finite(src, PERIOD, np.random.default_rng([7, DT_CODE[src], F8_CODE[fmt]]), 3.0)
    a = tiled(block, n + 1, src)[1:]
    for margin in (0, 1, 3):
        buf, out = poisoned(n, fmt, 1)
        m, s = amax_tensor(), k_tensor()
        va.quantize_fp8_auto(a, fmt, margin=margin, amax=m, scale_exp=s, out=out)
        torch.cuda.synchronize()
        want, k, wm = A.quantize_auto(block, src, fmt, margin)
        what = f"{src}->{fmt} margin {margin} n={n}"
        assert int(s.item()) == k and amax_bits(m) == A.f64_bits(wm), what
        shifted = np.roll(want, -1)             # a starts at element 1 of the tiled block
        assert_matches(out, tiled(shifted, n, fmt), fmt, what)
        assert_guards(buf, GUARD + 1, n, what)
        del buf, out


def test_f16_e4m3_f16_beyond_32_bit_offsets():
    """n = 2^32 + 4099: element 2^31 is byte 2^32 of the f16 arrays and element 2^32 needs a 64-bit index.  The
    largest magnitude sits in the last element, so an amax pass that stops short gives another k."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * 2 * n + 2 * n + (4 << 30):
        pytest.skip("needs ~28 GiB of free device memory")
    block = X.finite("f16", PERIOD, np.random.default_rng(31), 0.5)
    a = tiled(block, n, "f16")
    big = storage([-100.0], "f16")
    a[n - 1:].view(torch.int16).fill_(int(big.view(np.int16)[0]))
    q = torch.empty(n, dtype=torch.uint8, device="cuda")
    q.fill_(POISON)
    m, s = amax_tensor(), k_tensor()
    va.quantize_fp8_auto(a, "e4m3", amax=m, scale_exp=s, out=q.view(torch.float8_e4m3fn))
    del a
    k = A.auto_scale_exp(100.0, "e4m3", 0)
    assert float(m.item()) == 100.0 and int(s.item()) == k == 2
    want = tiled(F.quantize(block, "f16", "e4m3", k), n, "e4m3")
    want[n - 1:].view(torch.uint8).fill_(int(F.quantize(big, "f16", "e4m3", k)[0]))
    assert_matches(q.view(torch.float8_e4m3fn), want, "e4m3", "quantize, n = 2^32 + 4099")
    del want
    c = torch.empty(n, dtype=torch.float16, device="cuda")
    c.view(torch.uint8).fill_(POISON)
    va.dequantize_fp8_auto(q.view(torch.float8_e4m3fn), s, "f16", out=c)
    want = tiled(F.dequantize(F.quantize(block, "f16", "e4m3", k), "e4m3", "f16", k), n, "f16")
    last = F.dequantize(F.quantize(big, "f16", "e4m3", k), "e4m3", "f16", k)
    want[n - 1:].view(torch.int16).fill_(int(last.view(np.int16)[0]))
    for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - 8192):
        assert_matches(c[lo:lo + 8192], want[lo:lo + 8192], "f16", f"window at {lo}")
    assert_matches(c, want, "f16", "dequantize, n = 2^32 + 4099")


# ------------------------------------------------------------------------------------------- element offsets
@pytest.mark.parametrize("src", DTYPES)
def test_every_offset_of_a_and_c(src):
    rng = np.random.default_rng([11, DT_CODE[src]])
    total = 4099 + 16
    host = X.finite(src, total, rng, 2.0)
    host[rng.integers(0, total, 40)] = storage(rng.standard_normal(40) * 64, src)      # scattered larger magnitudes
    abuf, _ = poisoned(total, src)
    abuf[GUARD:GUARD + total].copy_(to_dev(host, src))
    for oa in range(16 // ES[src]):
        for oc in range(16):
            for n in (33, 4099):
                fmt = FMTS[(oa + oc) % 2]
                check_auto(src, fmt, host[oa:oa + n], abuf[GUARD + oa:GUARD + oa + n], 1, off_c=oc,
                           what=f"offsets A {oa} C {oc}")


# ------------------------------------------------------------------------------------------- value classes
@pytest.mark.parametrize("src", DTYPES)
def test_value_classes(src):
    rng = np.random.default_rng([13, DT_CODE[src]])
    zeros = storage(np.where(rng.integers(0, 2, 1000) == 1, 0.0, -0.0), src)
    for fmt in FMTS:
        for margin in (0, 3):
            _, k = check_auto(src, fmt, zeros, to_dev(zeros, src), margin, what="all zeros")
            assert k == 126
    mixed = X.finite(src, 5003, rng, 10.0)
    mixed[::97] = storage([np.inf], src)[0]
    mixed[5::101] = storage([-np.inf], src)[0]
    mixed[7::89] = storage([np.nan], src)[0]
    for fmt in FMTS:
        want, k = check_auto(src, fmt, mixed, to_dev(mixed, src), 0, what="inf and NaN mixed in")
        assert k == A.auto_scale_exp(float(np.abs(X.widen(mixed, src)[np.isfinite(X.widen(mixed, src))]).max()), fmt, 0)
        top = F.SPEC[fmt][4]
        x = X.widen(mixed, src)
        assert ((want[np.isinf(x)] & 0x7F) == top).all() and ((want[np.isnan(x)] & 0x7F) == 0x7F).all()
        # a running *d_amax larger than the tensor's sets the scale
        run = 4.0 * float(np.abs(x[np.isfinite(x)]).max())
        check_auto(src, fmt, mixed, to_dev(mixed, src), 1, acc=run, what="running amax")
        # a *d_amax the caller left invalid: k = 0, *d_amax keeps it
        for seed in (np.nan, np.inf, -1.0, -0.0):
            _, k = check_auto(src, fmt, mixed, to_dev(mixed, src), 1, acc=seed, what=f"*d_amax seeded {seed}")
            assert k == 0
    if src == "f64":
        for scale in (2.0 ** 130, 2.0 ** -140, 1e300, 2.0 ** 1000):     # beyond the f32 range, both ways
            host = X.finite("f64", 3001, rng, scale)
            for fmt in FMTS:
                check_auto("f64", fmt, host, to_dev(host, "f64"), 0, what=f"f64 scale {scale}")


# ------------------------------------------------------------------------------------------- dequantize
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_round_trip_equals_the_host_k_dequantize(src, fmt):
    rng = np.random.default_rng([17, DT_CODE[src], F8_CODE[fmt]])
    for n, scale in ((4099, 2.0 ** -6), ((1 << 20) + 3, 3.0)):
        host = X.finite(src, n, rng, scale)
        q, s = va.quantize_fp8_auto(to_dev(host, src), fmt, margin=1)
        k = int(s.item())
        want_q, want_k, _ = A.quantize_auto(host, src, fmt, 1)
        assert k == want_k
        for dst in DTYPES:
            what = f"{src}->{fmt}->{dst} n={n}"
            buf, c = poisoned(n, dst, 1)
            assert va.dequantize_fp8_auto(q, s, TORCH[dst], out=c) is c
            torch.cuda.synchronize()
            want = A.dequantize_auto(want_q, fmt, dst, k)
            assert_matches(c, to_dev(want, dst), dst, what)
            assert_matches(c, va.dequantize_fp8(q, TORCH[dst], scale_exp=k), dst, what + " vs host k", nan_class=False)
            assert_guards(buf, GUARD + 1, n, what)
            if dst == "f64":                    # the FP8 values scaled back, exactly
                assert np.array_equal(want, np.ldexp(F.DECODE[fmt][want_q], -k))


def test_an_out_of_range_k_makes_every_element_nan():
    bits = np.tile(np.arange(256, dtype=np.uint8), 17)
    for fmt in FMTS:
        q = to_dev(bits, fmt)
        for dst in DTYPES:
            for k in (127, -127, -(1 << 31), (1 << 31) - 1):
                buf, c = poisoned(bits.size, dst, 3)
                va.dequantize_fp8_auto(q, k_tensor(k), dst, out=c)
                torch.cuda.synchronize()
                assert bool(torch.isnan(c.double()).all()), (fmt, dst, k)
                assert_guards(buf, GUARD + 3, bits.size, f"{fmt}->{dst} k={k}")
            for k in (-126, 126):
                c = va.dequantize_fp8_auto(q, k_tensor(k), dst)
                assert_matches(c, to_dev(F.dequantize(bits, fmt, dst, k), dst), dst, f"{fmt}->{dst} k={k}")


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A_, n = buf.data_ptr() + 4096, 1000
    C_, M_, S_ = A_ + 16384, A_ + 32768, A_ + 40960      # an output, an amax and a scale slot away from A
    F32, F64, F16, BF16 = 0, 1, 2, 3
    E4, E5 = capi.F8_E4M3, capi.F8_E5M2
    q = [
        ((4, A_, E4, C_, n, 0, M_, S_), capi.ERR_VARIANT), ((F32, A_, 2, C_, n, 0, M_, S_), capi.ERR_VARIANT),
        ((F32, A_, E4, C_, n, -1, M_, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, n, 127, M_, S_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, n, 0, None, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, n, 0, M_, None), capi.ERR_INVALID),
        ((F32, A_, E4, C_, 0, 0, None, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, 0, 0, M_, None), capi.ERR_INVALID),
        ((F32, None, E4, C_, n, 0, M_, S_), capi.ERR_INVALID), ((F32, A_, E5, None, n, 0, M_, S_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, (1 << 40) + 1, 0, M_, S_), capi.ERR_INVALID),
        ((F32, A_ + 2, E4, C_, n, 0, M_, S_), capi.ERR_ALIGN), ((F64, A_ + 4, E4, C_, n, 0, M_, S_), capi.ERR_ALIGN),
        ((F16, A_ + 1, E5, C_, n, 0, M_, S_), capi.ERR_ALIGN),
        ((F32, A_, E4, C_, n, 0, M_ + 4, S_), capi.ERR_ALIGN), ((F32, A_, E4, C_, n, 0, M_, S_ + 2), capi.ERR_ALIGN),
        ((F32, A_, E4, A_, n, 0, M_, S_), capi.ERR_OVERLAP), ((BF16, A_ + 8, E4, A_, n, 0, M_, S_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, n, 0, A_ + 8, S_), capi.ERR_OVERLAP), ((F32, A_, E4, C_, n, 0, C_ + n - 8, S_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, n, 0, M_, A_ + 4 * n - 4), capi.ERR_OVERLAP), ((F32, A_, E4, C_, n, 0, M_, C_ + 100), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, n, 0, M_, M_), capi.ERR_OVERLAP), ((F32, A_, E4, C_, n, 0, M_, M_ + 4), capi.ERR_OVERLAP),
    ]
    d = [
        ((E4, A_, 4, C_, n, S_), capi.ERR_VARIANT), ((2, A_, F32, C_, n, S_), capi.ERR_VARIANT),
        ((E4, A_, F32, C_, n, None), capi.ERR_INVALID), ((E4, A_, F32, C_, 0, None), capi.ERR_INVALID),
        ((E4, None, F32, C_, n, S_), capi.ERR_INVALID), ((E4, A_, F32, None, n, S_), capi.ERR_INVALID),
        ((E4, A_, F32, C_, (1 << 40) + 1, S_), capi.ERR_INVALID),
        ((E4, A_, F32, C_ + 2, n, S_), capi.ERR_ALIGN), ((E5, A_, F64, C_ + 4, n, S_), capi.ERR_ALIGN),
        ((E4, A_, F32, C_, n, S_ + 1), capi.ERR_ALIGN),
        ((E4, A_, F32, A_, n, S_), capi.ERR_OVERLAP), ((E4, A_, F16, C_, n, A_ + 4), capi.ERR_OVERLAP),
        ((E5, A_, F64, C_, n, C_ + 8 * n - 4), capi.ERR_OVERLAP),
    ]
    for args, code in q:
        assert L.b200va_quantize_fp8_auto(*args, None) == code, (args, code)
    for args, code in d:
        assert L.b200va_dequantize_fp8_auto(*args, None) == code, (args, code)
    # n = 0: nothing to do, nothing written, nothing launched
    assert L.b200va_quantize_fp8_auto(F32, None, E4, None, 0, 0, M_, S_, None) == capi.OK
    assert L.b200va_quantize_fp8_auto(F32, A_, E4, C_, 0, 0, M_, S_, None) == capi.OK
    assert L.b200va_dequantize_fp8_auto(E5, None, F64, None, 0, S_, None) == capi.OK
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == POISON).all(), "a rejected or empty call wrote to device memory"
    # right behind each other: no overlap, and the calls run
    M2 = A_ + 5 * n + 8 - (A_ + 5 * n) % 8
    assert L.b200va_quantize_fp8_auto(F32, A_, E4, A_ + 4 * n, n, 0, M2, M2 + 8, None) == capi.OK
    assert L.b200va_dequantize_fp8_auto(E4, A_ + 4 * n, F16, C_, n, M2 + 8, None) == capi.OK
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- graphs and stream order
def test_captured_graph_follows_the_scale_across_replays():
    """One graph: reset *d_amax, quantize, dequantize.  Between replays only the input changes, by a factor of 2^20
    either way, so each replay's k must come from its own amax on the device."""
    n = 100_003
    cases = []
    for src, fmt, dst in (("f32", "e4m3", "f32"), ("bf16", "e5m2", "f16"), ("f64", "e4m3", "bf16"), ("f16", "e5m2", "f64")):
        a = torch.empty(n, dtype=TORCH[src], device="cuda")
        bq, q = poisoned(n, fmt, 1)
        bc, c = poisoned(n, dst, 3)
        cases.append((src, fmt, dst, a, bq, q, bc, c, amax_tensor(), k_tensor()))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for src, fmt, dst, a, _, q, _, c, m, s in cases:
                m.zero_()
                va.quantize_fp8_auto(a, fmt, margin=1, amax=m, scale_exp=s, out=q)
                va.dequantize_fp8_auto(q, s, dst, out=c)
    torch.cuda.synchronize()
    rng = np.random.default_rng(19)
    ks = {case[:3]: [] for case in cases}
    for r, e in enumerate((0, 20, 0, -20, 0)):
        hosts = []
        for src, fmt, dst, a, bq, q, bc, c, m, s in cases:
            ee = e // 2 if src == "f16" else e                      # f16 holds 2^+-10 around 1, not 2^+-20
            host = X.finite(src, n, rng, 2.0 ** ee)
            a.copy_(to_dev(host, src))
            hosts.append(host)
            bq.view(torch.uint8).fill_(POISON)
            bc.view(torch.uint8).fill_(POISON)
            m.fill_(1e300)
            s.fill_(K_POISON)
        g.replay()
        torch.cuda.synchronize()
        for host, (src, fmt, dst, a, bq, q, bc, c, m, s) in zip(hosts, cases):
            what = f"{src}->{fmt}->{dst} replay {r}"
            want, k, wm = A.quantize_auto(host, src, fmt, 1)
            assert int(s.item()) == k and amax_bits(m) == A.f64_bits(wm), (what, int(s.item()), k)
            assert_matches(q, to_dev(want, fmt), fmt, what)
            assert_matches(c, to_dev(A.dequantize_auto(want, fmt, dst, k), dst), dst, what)
            assert_guards(bq, GUARD + 1, n, what)
            assert_guards(bc, GUARD + 3, n, what)
            ks[(src, fmt, dst)].append(k)
    for key, seq in ks.items():
        assert len(set(seq)) == 3, (key, seq)                       # the scale followed the input


def test_stream_op_quantize_dequantize_stream_op_on_one_stream():
    """Six rounds on one stream without a host sync: b = s a (b200va_stream), q, k = quantize_fp8_auto(b),
    c = dequantize_fp8_auto(q, k), d_r = c / 2 (b200va_stream); s moves k every round.  At an L2-resident size and in
    the HBM class of the source."""
    st = torch.cuda.Stream()
    for src, fmt, dst in (("f32", "e4m3", "f32"), ("bf16", "e5m2", "f16"), ("f64", "e4m3", "bf16")):
        a0 = X.finite(src, 49_999, np.random.default_rng(DT_CODE[src]), 8.0)
        scalars = [2.0 ** (3 * r - 6) * (1 + r / 8) for r in range(6)]
        wants = []
        for s in scalars:
            b = X.stream("scale", src, a0, None, s)
            q, k, m = A.quantize_auto(b, src, fmt, 0)
            wants.append((X.stream("scale", dst, A.dequantize_auto(q, fmt, dst, k), None, 0.5), k, m))
        assert len({k for _, k, _ in wants}) == len(scalars)
        for n in ((1 << 20) + 5, hbm_n(ES[src]) + 5):
            a = tiled(a0, n, src)
            b = torch.empty_like(a)
            q = torch.empty(n, dtype=TORCH[fmt], device="cuda")
            c = torch.empty(n, dtype=TORCH[dst], device="cuda")
            ds = [torch.empty_like(c) for _ in scalars]
            ms = torch.zeros(len(scalars), dtype=torch.float64, device="cuda")
            ks = torch.full((len(scalars),), K_POISON, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            for r, (s, d) in enumerate(zip(scalars, ds)):
                va.stream("scale", a, None, b, scalar=s, stream=st)
                va.quantize_fp8_auto(b, fmt, amax=ms[r:r + 1], scale_exp=ks[r:r + 1], out=q, stream=st)
                va.dequantize_fp8_auto(q, ks[r:r + 1], dst, out=c, stream=st)
                va.stream("scale", c, None, d, scalar=0.5, stream=st)
            st.synchronize()
            for r, (d, (w, k, m)) in enumerate(zip(ds, wants)):
                what = f"{src}->{fmt}->{dst} n={n} round {r}"
                assert int(ks[r].item()) == k and amax_bits(ms[r:r + 1]) == A.f64_bits(m), what
                assert_matches(d, tiled(w, n, dst), dst, what)
            del a, b, q, c, ds


# ------------------------------------------------------------------------------------------- trace
def expected_amax_launch(kernel, es, n, a_ptr):
    """(kernel, grid, block) of the amax pass (plan_fp8_amax, b200va_typed.cu): A alone, its vector body from the head
    that puts A on a 16-byte boundary, a group of 16 per unit, every other element an edge item."""
    head = min(((16 - a_ptr % 16) % 16) // es, n)
    ngroups = (n - head) // 16
    edges = n - 16 * ngroups
    threads, unroll = (512, 2) if n >= hbm_n(es) else (256, 1)
    blocks = max(-(-ngroups // (threads * unroll)), -(-edges // threads))
    return kernel, max(1, min(blocks, 2 ** 31 - 1)), threads


def test_trace_shows_two_quantize_launches_and_one_dequantize(tmp_path):
    """Per source type: n = 1000, the HBM class, and odd n at offsets that give the amax pass a head of its own.
    After the marker: the amax pass, the quantize pass and the dequantize per call, with their grids and blocks,
    and nothing else."""
    plan, want = [], []
    keep = []
    for i, src in enumerate(DTYPES):
        fmt = FMTS[i % 2]
        nmax = hbm_n(ES[src]) + 64
        wide, wide_out = torch.zeros(nmax, dtype=TORCH[src], device="cuda"), torch.zeros(nmax, dtype=TORCH[src], device="cuda")
        narrow = torch.zeros(nmax, dtype=torch.uint8, device="cuda").view(TORCH[fmt])
        keep += [wide, wide_out, narrow]
        for n, oa, oq, oc in ((1000, 0, 0, 0), (hbm_n(ES[src]), 0, 0, 0), (1001, 1, 0, 1), (4099, 1, 3, 0)):
            a, q, c = wide[oa:oa + n], narrow[oq:oq + n], wide_out[oc:oc + n]
            dt = DT_CODE[src]
            want.append(expected_amax_launch(f"fp8_quant_vec<{dt}>", ES[src], n, a.data_ptr()))
            want.append(expected_cast_launch(f"fp8_quant_vec<{dt}>", ES[src], 1, n, a.data_ptr(), q.data_ptr()))
            want.append(expected_cast_launch(f"fp8_dequant_vec<{dt}>", 1, ES[src], n, q.data_ptr(), c.data_ptr(), ES[src]))
            plan.append((src, fmt, a, q, c, amax_tensor(), k_tensor()))

    def run_plan():
        for src, fmt, a, q, c, m, s in plan:
            va.quantize_fp8_auto(a, fmt, amax=m, scale_exp=s, out=q)
            va.dequantize_fp8_auto(q, s, src, out=c)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("fp8_",))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for j, (g, w) in enumerate(zip(got, want)):
        assert g == w, (plan[j // 3][:2], j % 3, g, w)
