"""b200va_quantize_fp8_blockwise and b200va_dequantize_fp8_blockwise on the GPU, bit for bit against
tests/fp8_block_exact.py.

- Every source type, format and block kind, row-wise only, column-wise only and both, on random bit patterns (every
  value class) with +-0, subnormals, +-inf, NaN payloads and values past the FP8 range planted.
- Tiled shapes, partial bottom tiles (rows % 128 = 16 and 112), ragged shapes (cols % 128 != 0, rows % 16 != 0,
  1 x n, n x 1, 1 x 1) and operands off a 16-byte boundary.  C, Ct, S and St sit between 64 KiB poisoned guards and
  the 128x128 scale padding must keep its poison.
- A planted block maximum at every row and every column position of a tile, blocks that are zero, NaN/inf-only or
  subnormal, maxima at 1.75 2^e +- 1 ulp, and f64 blocks whose k clamps at -126.
- Cross-checks: the column-wise side equals the row-wise side of A.t().contiguous(); 128x128 Ct == C.t(); the 1x128
  row-wise bytes equal quantize_mxfp8(block=128, "nosat") where cols % 128 == 0 and no block clamps.
- Dequantize: the round trip, and random non-power-of-two, NaN, +-inf and 0 scales.
- Every rejected argument alone and in pairs returns the earlier code and writes nothing.
- A captured graph replayed with new inputs, a stream-order chain, a profiler trace of one launch per call, and a
  shape whose Ct byte index passes 2^32.
"""
import numpy as np
import pytest

import fp8_block_exact as BE
from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import DT_CODE, F8_CODE, TORCH, assert_matches, kernels_after_marker, to_dev
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = V.DTYPES
FMTS = F.FORMATS8
KINDS = BE.KINDS
KIND = {"1x128": 0, "128x128": 1}
SIDES = ("row", "col", "both")
PAD = 1 << 16                          # guard bytes on each side of every buffer
POISON = 0xA5
SHAPES = ((256, 256), (144, 384), (240, 128), (16, 128), (100, 200), (33, 130), (1, 300), (300, 1), (1, 1),
          (130, 257))


# ------------------------------------------------------------------------------------------- helpers
def storage(x, src):
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        return x.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(x, src)


def values(src, n, rng):
    host = V.random_bits(src, n, rng)
    tiny = {"f32": 2.0 ** -149, "f64": 5e-324, "f16": 2.0 ** -24, "bf16": 2.0 ** -133}[src]
    planted = storage([0.0, -0.0, np.inf, -np.inf, 1e5, -6e4, tiny, -tiny, 2.0 ** -20, 1.0, -1.5], src)
    for i, v in enumerate(planted):
        host[(i * 37) % n::97] = v
    return host


class Buf:
    """nbytes at byte offset off inside a POISON-filled buffer with PAD bytes either side."""

    def __init__(self, nbytes, off=0):
        self.raw = torch.full((PAD + off + nbytes + PAD,), POISON, dtype=torch.uint8, device="cuda")
        self.lo, self.n = PAD + off, nbytes

    def view(self, dtype):
        return self.raw[self.lo:self.lo + self.n].view(dtype)

    def ptr(self):
        return self.raw.data_ptr() + self.lo

    def guards_ok(self):
        return bool((self.raw[:self.lo] == POISON).all()) and bool((self.raw[self.lo + self.n:] == POISON).all())


def scale_base(count):
    return np.frombuffer(bytes([POISON]) * (4 * count), np.float32).copy()


def run(src, fmt, kind, host, rows, cols, side="both", offs=(0, 0, 0), what=""):
    """One quantize through the C ABI with poisoned, guarded buffers; every output against the reference.  Returns
    the device outputs (C, S, Ct, St), None for a side not asked for."""
    n = rows * cols
    es = X.STORAGE[src]().itemsize if src in ("f32", "f64") else 2
    what = f"{src}->{fmt} {kind} {rows}x{cols} {side} offs={offs} {what}"
    ab = Buf(n * es, offs[0] * es)
    ab.view(torch.uint8).copy_(torch.from_numpy(np.ascontiguousarray(host).view(np.uint8)).cuda())
    row, col = side in ("row", "both"), side in ("col", "both")
    ns, nst = BE.scale_count(rows, cols, kind), BE.scale_count(cols, rows, kind)
    cb, sb = (Buf(n, offs[1]), Buf(4 * ns)) if row else (None, None)
    tb, tsb = (Buf(n, offs[2]), Buf(4 * nst)) if col else (None, None)
    p = lambda b: b.ptr() if b is not None else None  # noqa: E731
    rc = capi.lib.b200va_quantize_fp8_blockwise(DT_CODE[src], ab.ptr(), F8_CODE[fmt], KIND[kind], rows, cols, p(cb),
                                                p(sb), p(tb), p(tsb), None)
    assert rc == 0, (what, rc)
    torch.cuda.synchronize()
    wc, ws, wct, wst = BE.quantize(host, src, fmt, kind, rows, cols, scale_base(ns), scale_base(nst))
    for b, want, name, fm in ((cb, wc, "C", fmt), (tb, wct, "Ct", fmt)):
        if b is not None:
            assert_matches(b.view(TORCH[fmt]), to_dev(want.ravel(), fmt), fm, f"{what} {name}")
            assert b.guards_ok(), f"{what} {name} guard"
    for b, want, name in ((sb, ws, "S"), (tsb, wst, "St")):
        if b is not None:
            got = b.view(torch.int32).cpu().numpy()
            bad = np.flatnonzero(got != want.view(np.int32))
            assert bad.size == 0, f"{what} {name}: {bad.size} scale mismatches, first at {bad[0]}"
            assert b.guards_ok(), f"{what} {name} guard"
    assert ab.guards_ok(), what
    return (cb.view(TORCH[fmt]) if row else None, sb.view(torch.float32) if row else None,
            tb.view(TORCH[fmt]) if col else None, tsb.view(torch.float32) if col else None)


# ------------------------------------------------------------------------------------------- quantize
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_matches_reference(src, fmt, kind):
    rng = np.random.default_rng([DT_CODE[src], F8_CODE[fmt], KIND[kind]])
    for rows, cols in SHAPES:
        host = values(src, rows * cols, rng)
        for side in SIDES:
            run(src, fmt, kind, host, rows, cols, side)
        # finite values, so that most blocks have a maximum in range
        run(src, fmt, kind, X.finite(src, rows * cols, rng, 3.0), rows, cols, "both", what="finite")
    for offs in ((1, 0, 0), (0, 3, 0), (0, 0, 5)):
        run(src, fmt, kind, X.finite(src, 128 * 256, rng, 2.0), 128, 256, "both", offs)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("src", ("f32", "f16", "f64"))
def test_planted_maximum_at_every_row_and_column_of_a_tile(src, kind):
    """128 tiles side by side; tile t holds its largest value at row t and column 53 t mod 128."""
    rng = np.random.default_rng([9, DT_CODE[src]])
    rows, cols = 128, 128 * 128
    x = rng.uniform(-1.0, 1.0, (rows, cols))
    for t in range(128):
        x[t, 128 * t + (53 * t) % 128] = -7.5 * (1 + t)
    run(src, "e4m3", kind, storage(x.ravel(), src), rows, cols, "both", what="planted")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_value_classes(src, fmt):
    rows, cols = 128, 512
    emax = {"e4m3": 8, "e5m2": 15}[fmt]
    x = np.random.default_rng(3).uniform(-1, 1, (rows, cols))
    x[:, 0:128] = 0.0                                           # an all-zero column of 1x128 blocks
    x[:, 128:256] = np.where(np.arange(128) % 2, np.inf, np.nan)   # NaN / inf only
    tiny = {"f32": 2.0 ** -149, "f64": 5e-324, "f16": 2.0 ** -24, "bf16": 2.0 ** -133}[src]
    x[:, 256:384] *= tiny * 8
    ulp = {"f32": 2.0 ** -23, "f64": 2.0 ** -52, "f16": 2.0 ** -10, "bf16": 2.0 ** -7}[src]
    for r in range(rows):
        x[r, 384 + r % 128] = 1.75 * 2.0 ** (r % 7 - 3) * (1 + (r % 3 - 1) * ulp)
    run(src, fmt, "1x128", storage(x.ravel(), src), rows, cols, "both", what="classes")
    run(src, fmt, "128x128", storage(x.ravel(), src), rows, cols, "both", what="classes")
    if src == "f64":                                            # k clamps at -126: the block saturates
        y = np.random.default_rng(4).uniform(-1, 1, (128, 256)) * 2.0 ** (126 + emax + 40)
        c, s, _, _ = run(src, fmt, "1x128", y.ravel(), 128, 256, "row", what="clamp")
        assert bool((s == 2.0 ** 126).all())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("src", ("f32", "bf16"))
def test_cross_checks(src, kind):
    rng = np.random.default_rng([5, DT_CODE[src]])
    rows, cols = 384, 256
    a = to_dev(X.finite(src, rows * cols, rng, 2.0), src).view(rows, cols)
    out, s, out_t, s_t = va.quantize_fp8_blockwise(a, "e4m3", block=kind)
    r_out, r_s, _, _ = va.quantize_fp8_blockwise(a.t().contiguous(), "e4m3", block=kind, columnwise=False)
    torch.cuda.synchronize()
    assert torch.equal(out_t.view(torch.uint8), r_out.view(torch.uint8))
    if kind == "128x128":                                       # the view's rows past ceil(K / 128) are padding
        s_t, r_s = s_t[:-(-rows // 128)], r_s[:-(-rows // 128)]
    assert torch.equal(s_t, r_s)
    if kind == "128x128":
        assert torch.equal(out_t.view(torch.uint8), out.view(torch.uint8).t().contiguous())
    else:
        q, e8 = va.quantize_mxfp8(a.reshape(-1), "e4m3", block=128, scale_rule="nosat")
        assert torch.equal(out.view(torch.uint8).reshape(-1), q.view(torch.uint8))
        want = torch.exp2(e8.to(torch.float32) - 127).view(rows, cols // 128)
        assert torch.equal(s, want)


# ------------------------------------------------------------------------------------------- dequantize
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dst", DTYPES)
def test_dequantize(dst, fmt, kind):
    rng = np.random.default_rng([7, DT_CODE[dst], F8_CODE[fmt], KIND[kind]])
    for rows, cols in ((256, 384), (130, 200), (1, 1), (40, 16)):
        q = rng.integers(0, 256, rows * cols, dtype=np.uint8)
        ns = BE.scale_count(rows, cols, kind)
        s = (rng.uniform(0.5, 2.0, ns) * np.exp2(rng.integers(-140, 120, ns))).astype(np.float32)
        s[::7] = np.float32(np.nan)
        s[1::11] = np.float32(np.inf)
        s[2::13] = np.float32(-np.inf)
        s[3::17] = 0
        s[4::19] = np.float32(2.0 ** -149)
        qd, sd = to_dev(q, fmt).view(rows, cols), torch.from_numpy(s).cuda()
        got = va.dequantize_fp8_blockwise(qd, sd, dst, block=kind)
        torch.cuda.synchronize()
        want = BE.dequantize(q, s, fmt, dst, kind, rows, cols)
        assert_matches(got.reshape(-1), to_dev(want, dst), dst, f"{dst} {fmt} {kind} {rows}x{cols}")


@pytest.mark.parametrize("kind", KINDS)
def test_round_trip(kind):
    rng = np.random.default_rng(11)
    rows, cols = 256, 512
    a = torch.from_numpy(rng.standard_normal((rows, cols)) * 2.0 ** -20).cuda()
    out, s, out_t, s_t = va.quantize_fp8_blockwise(a, "e4m3", block=kind)
    back = va.dequantize_fp8_blockwise(out, s, "f64", block=kind)
    back_t = va.dequantize_fp8_blockwise(out_t, s_t, "f64", block=kind)
    torch.cuda.synchronize()
    # elements within 2^6 of the largest magnitude are within 2^6 of their block's: E4M3 normals after scaling,
    # relative error <= 2^-4
    big = a.abs() >= a.abs().max() / 64
    for b in (back, back_t.t()):
        assert float(((b - a).abs() / a.abs())[big].max()) <= 2.0 ** -4


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_in_order_and_write_nothing():
    L = capi.lib
    buf = torch.full((1 << 20,), POISON, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    R, Cc = 128, 256
    n = R * Cc
    A_, C_, S_, T_, ST_ = base + 4096, base + 4096 + 4 * n, base + 8192 + 5 * n, base + 12288 + 6 * n, base + 16384 + 7 * n
    good = dict(src=0, a=A_, fmt=0, kind=0, rows=R, cols=Cc, c=C_, s=S_, ct=T_, st=ST_)
    # (argument, faulty value, code) in check order
    faults = [("src", 9, capi.ERR_VARIANT), ("fmt", 5, capi.ERR_VARIANT), ("kind", 2, capi.ERR_VARIANT),
              ("s", None, capi.ERR_INVALID), ("st", None, capi.ERR_INVALID), ("rows", 1 << 40, capi.ERR_INVALID),
              ("a", A_ + 2, capi.ERR_ALIGN), ("s", S_ + 2, capi.ERR_ALIGN), ("st", ST_ + 1, capi.ERR_ALIGN),
              ("c", A_ + 64, capi.ERR_OVERLAP), ("ct", C_ + 100, capi.ERR_OVERLAP), ("s", T_ + 4, capi.ERR_OVERLAP),
              ("st", S_ + 8, capi.ERR_OVERLAP)]

    def call(args):
        return L.b200va_quantize_fp8_blockwise(args["src"], args["a"], args["fmt"], args["kind"], args["rows"],
                                               args["cols"], args["c"], args["s"], args["ct"], args["st"], None)

    torch.cuda.synchronize()
    for i, (name, value, code) in enumerate(faults):
        assert call(dict(good, **{name: value})) == code, (name, value)
        for name2, value2, code2 in faults[i + 1:]:
            if name2 == name:
                continue
            assert call(dict(good, **{name: value, name2: value2})) == code, (name, value, name2, value2)
    assert call(dict(good, c=None, s=None, ct=None, st=None)) == capi.ERR_INVALID
    assert call(dict(good, rows=0, c=None, s=None, ct=None, st=None)) == 0
    torch.cuda.synchronize()
    assert bool((buf == POISON).all()), "a rejected call wrote"
    # dequantize
    D = lambda **k: L.b200va_dequantize_fp8_blockwise(k.get("fmt", 0), A_, k.get("s", S_), k.get("kind", 0),  # noqa
                                                      k.get("dst", 0), k.get("c", C_), R, Cc, None)
    assert D(dst=7) == capi.ERR_VARIANT and D(kind=3) == capi.ERR_VARIANT and D(s=None) == capi.ERR_INVALID
    assert D(c=C_ + 2) == capi.ERR_ALIGN and D(s=S_ + 1) == capi.ERR_ALIGN and D(c=A_ + 8) == capi.ERR_OVERLAP
    torch.cuda.synchronize()
    assert bool((buf == POISON).all()), "a rejected dequantize wrote"


# ------------------------------------------------------------------------------------------- streams and graphs
def test_graph_capture_and_stream_chain():
    rows, cols = 512, 1024
    a = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    outs = [torch.empty(rows, cols, dtype=torch.float8_e4m3fn, device="cuda"),
            torch.empty(BE.scale_count(rows, cols, "1x128"), dtype=torch.float32, device="cuda"),
            torch.empty(cols, rows, dtype=torch.float8_e4m3fn, device="cuda"),
            torch.empty(BE.scale_count(cols, rows, "1x128"), dtype=torch.float32, device="cuda")]
    back = torch.empty(cols, rows, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        va.quantize_fp8_blockwise(a, "e4m3", out=outs[0], scales=outs[1], out_t=outs[2], scales_t=outs[3])
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        q = va.quantize_fp8_blockwise(a, "e4m3", out=outs[0], scales=outs[1], out_t=outs[2], scales_t=outs[3])
        va.dequantize_fp8_blockwise(q[2], q[3], "f32", block="1x128", out=back)
    for scale in (1.0, 2.0 ** 20, 2.0 ** -20):
        a.copy_(torch.randn(rows, cols, device="cuda") * scale)
        g.replay()
        torch.cuda.synchronize()
        host = a.view(torch.int16).cpu().numpy().view(np.uint16).ravel()
        wc, ws, wct, wst = BE.quantize(host, "bf16", "e4m3", "1x128", rows, cols)
        assert np.array_equal(outs[2].view(torch.uint8).cpu().numpy().ravel(), wct.ravel())
        assert np.array_equal(outs[3].cpu().numpy().view(np.int32), wst.view(np.int32))
        want = BE.dequantize(wct.ravel(), wst, "e4m3", "f32", "1x128", cols, rows)
        assert np.array_equal(back.cpu().numpy().ravel().view(np.int32), want.view(np.int32))
    # a chain on one stream: convert -> blockwise quantize -> dequantize, each reading what the one before wrote
    x = torch.randn(rows, cols, device="cuda")
    for _ in range(3):
        h = va.convert(x, "f16")
        c1, s1, _, _ = va.quantize_fp8_blockwise(h.view(rows, cols), "e5m2", block="128x128", columnwise=False)
        d = va.dequantize_fp8_blockwise(c1, s1, "f32", block="128x128")
        torch.cuda.synchronize()
        host = h.view(torch.int16).cpu().numpy().view(np.uint16).ravel()
        wc, ws, _, _ = BE.quantize(host, "f16", "e5m2", "128x128", rows, cols)
        assert np.array_equal(c1.view(torch.uint8).cpu().numpy(), wc)
        want = BE.dequantize(wc.ravel(), ws, "e5m2", "f32", "128x128", rows, cols)
        assert np.array_equal(d.cpu().numpy().ravel().view(np.int32), want.view(np.int32))
        x = x * 3.0


def test_one_launch_per_call(tmp_path):
    """Each call is one launch of the block-scaled kernel of its element size, with the planned geometry: 256-thread
    CTAs, one per 128 x 128 tile for the tiled quantize, and plan_geometry's grid (one unit per 16-byte output slice)
    for the dequantize.  The outputs are made before the trace and the plan ends in a synchronize, so that the trace
    holds exactly the plan's launches."""
    rows, cols = 256, 512
    a = torch.randn(rows, cols, device="cuda")
    q = va.quantize_fp8_blockwise(a, "e4m3", block="1x128")
    r = va.quantize_fp8_blockwise(a, "e4m3", block="128x128", columnwise=False)
    d32 = torch.empty(rows, cols, dtype=torch.float32, device="cuda")
    d16 = torch.empty(rows, cols, dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()

    def plan():
        va.quantize_fp8_blockwise(a, "e4m3", block="1x128", out=q[0], scales=q[1], out_t=q[2], scales_t=q[3])
        va.dequantize_fp8_blockwise(q[0], q[1], "f32", block="1x128", out=d32)
        va.quantize_fp8_blockwise(a, "e4m3", block="128x128", columnwise=False, out=r[0], scales=r[1])
        va.dequantize_fp8_blockwise(r[0], r[1], "bf16", block="128x128", out=d16)
        torch.cuda.synchronize()

    tiles, slices = rows // 128 * (cols // 128), rows * cols // 16
    want = [("mx_quant_vec<4>", tiles, 256), ("mx_dequant_vec<4>", slices * 4 // 256, 256),
            ("mx_quant_vec<4>", tiles, 256), ("mx_dequant_vec<2>", slices * 2 // 256, 256)]
    # Late in a long session a trace can begin after the marker, and then holds nothing to find it by (the helper's
    # max() over an empty list): such a capture says nothing about the launches and is taken again, at most 3 times.
    for attempt in range(3):
        try:
            got = kernels_after_marker(tmp_path, plan, ("mx_",))
            break
        except ValueError:
            if attempt == 2:
                raise
    assert got == want


def test_ct_index_past_2_32():
    """65536 x 65664 f16 on the tiled path: Ct's last rows lie past byte 2^32.  The bottom-right 128 x 128 tile is
    checked against the reference on that tile alone (its row and column blocks lie inside it)."""
    rows, cols = 65536, 65664
    assert (cols - 1) * rows > 1 << 32
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    assert free >= 4 * rows * cols + (2 << 30), f"needs about 19 GiB of free device memory, {free >> 30} GiB free"
    block = torch.from_numpy(X.finite("f16", 1 << 20, np.random.default_rng(13), 4.0).view(np.int16)).cuda()
    a = block.repeat(-(-rows * cols // block.numel()))[:rows * cols].view(torch.float16).view(rows, cols)
    out, s, out_t, s_t = va.quantize_fp8_blockwise(a, "e4m3")
    torch.cuda.synchronize()
    i0, j0 = rows - 128, cols - 128
    host = a[i0:, j0:].contiguous().view(torch.int16).cpu().numpy().view(np.uint16).ravel()
    wc, ws, wct, wst = BE.quantize(host, "f16", "e4m3", "1x128", 128, 128)
    assert np.array_equal(out[i0:, j0:].view(torch.uint8).cpu().numpy(), wc)
    assert np.array_equal(out_t[j0:, i0:].view(torch.uint8).cpu().numpy(), wct)
    assert np.array_equal(s[i0:, -1].cpu().numpy(), ws)
    assert np.array_equal(s_t[j0:, -1].cpu().numpy(), wst)
    del a, out, out_t, block
    torch.cuda.empty_cache()
