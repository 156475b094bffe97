"""b200va_quantize_fp8_rowwise and b200va_dequantize_fp8_rowwise on the GPU, bit for bit against
tests/fp8_rowwise_exact.py.

- One real GEMM first: the three products of a linear layer through torch._scaled_mm with row-wise scales, on inputs
  whose products are exact, against an f64 reference.
- Every source type and format, row-wise only, column-wise only and both, on random bit patterns (every value class)
  with +-0, subnormals, +-inf, NaN payloads and values past the FP8 range planted.
- Tiled shapes, partial bottom tiles, ragged shapes (cols % 128 != 0, rows % 16 != 0, 1 x n, n x 1, cols = 16, rows
  and cols below and above 128 and multiples of it) and operands off a 16-byte boundary.  C, S, Ct, St and the
  workspace sit between 64 KiB poisoned guards.
- Wide rows (cols = 65536 + 128) that span many tiles and CTAs; a planted row maximum in the row's last tile and a
  column maximum in the last row band, at each position; the value classes.
- Cross-checks: S is the max of quantize_fp8_blockwise's 1x128 block scales; C's row r is quantize_fp8(row r,
  scale_exp = k_r); the column-wise side is the row-wise side of A.t().contiguous().
- Dequantize: random non-power-of-two, NaN, +-inf and 0 scales, and the round trip.
- Every rejected argument alone and in pairs returns the earlier code and writes nothing, the workspace included.
- A captured graph replayed with inputs whose magnitude moves by 2^+-20, a stream chain, a tail behind a K2d writer, a
  profiler trace of the planned launches, and a shape whose Ct byte index passes 2^32.
"""
import numpy as np
import pytest

import fp8_rowwise_exact as RE
from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import oracle as O
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    import gpu_helpers as GH
    from gpu_helpers import DT_CODE, F8_CODE, TORCH, assert_matches, kernels_after_marker, to_dev
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = V.DTYPES
FMTS = F.FORMATS8
SIDES = ("row", "col", "both")
PAD = 1 << 16                          # guard bytes on each side of every buffer
POISON = 0xA5
SHAPES = ((256, 256), (144, 384), (240, 128), (16, 128), (100, 200), (33, 130), (1, 300), (300, 1), (1, 1),
          (130, 257), (64, 16), (127, 127), (129, 129), (128, 256), (48, 384))


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


def run(src, fmt, host, rows, cols, side="both", offs=(0, 0, 0), what=""):
    """One quantize through the C ABI with poisoned, guarded buffers (the workspace too); every output against the
    reference.  Returns the device outputs (C, S, Ct, St), None for a side not asked for."""
    n = rows * cols
    es = X.STORAGE[src]().itemsize if src in ("f32", "f64") else 2
    what = f"{src}->{fmt} {rows}x{cols} {side} offs={offs} {what}"
    ab = Buf(n * es, offs[0] * es)
    ab.view(torch.uint8).copy_(torch.from_numpy(np.ascontiguousarray(host).view(np.uint8)).cuda())
    row, col = side in ("row", "both"), side in ("col", "both")
    cb, sb = (Buf(n, offs[1]), Buf(4 * rows)) if row else (None, None)
    tb, tsb = (Buf(n, offs[2]), Buf(4 * cols)) if col else (None, None)
    need = RE.workspace_bytes(rows, cols)
    wb = Buf(need)
    p = lambda b: b.ptr() if b is not None else None  # noqa: E731
    rc = capi.lib.b200va_quantize_fp8_rowwise(DT_CODE[src], ab.ptr(), F8_CODE[fmt], rows, cols, p(cb), p(sb), p(tb),
                                              p(tsb), wb.ptr(), need, None)
    assert rc == 0, (what, rc)
    torch.cuda.synchronize()
    wc, ws, wct, wst = RE.quantize(host, src, fmt, rows, cols)
    for b, want, name in ((cb, wc, "C"), (tb, wct, "Ct")):
        if b is not None:
            assert_matches(b.view(TORCH[fmt]), to_dev(want.ravel(), fmt), fmt, f"{what} {name}")
            assert b.guards_ok(), f"{what} {name} guard"
    for b, want, name in ((sb, ws, "S"), (tsb, wst, "St")):
        if b is not None:
            got = b.view(torch.int32).cpu().numpy()
            bad = np.flatnonzero(got != want.view(np.int32))
            assert bad.size == 0, f"{what} {name}: {bad.size} scale mismatches, first at {bad[0]}"
            assert b.guards_ok(), f"{what} {name} guard"
    assert ab.guards_ok() and wb.guards_ok(), what
    return (cb.view(TORCH[fmt]) if row else None, sb.view(torch.float32) if row else None,
            tb.view(TORCH[fmt]) if col else None, tsb.view(torch.float32) if col else None)


# ------------------------------------------------------------------------------------------- one real GEMM
def test_linear_layer_products_through_scaled_mm():
    """Y = X W^T, dX = dY W and dW = dY^T X through torch._scaled_mm with the row-wise operands, E4M3, bf16 out.  Each
    row of X, W and dY is {-1, 0, 1} 2^(e_row + e_tensor), e_row in [-1, 1], and every reduction is 256 long.  Every
    FP8 value is then exact whichever side it is scaled for, and every product term of a reduction is within 2^4 of
    the others, so every partial sum needs at most 13 significant bits: it is exact even in the FP8 tensor cores'
    reduced-precision accumulation (with e_row in [-4, 4], dW came out one bf16 ulp off on an H100), and the bf16
    result is the exact f64 product rounded once."""
    rng = np.random.default_rng(31)
    M, K, N = 256, 256, 256

    def operand(r, c, e):
        return rng.integers(-1, 2, (r, c)) * np.exp2(rng.integers(-1, 2, (r, 1)) + e)

    x, w, dy = operand(M, K, -3), operand(N, K, 5), operand(M, N, -20)
    q = {name: va.quantize_fp8_rowwise(torch.from_numpy(t).to("cuda", torch.bfloat16), "e4m3")
         for name, t in (("x", x), ("w", w), ("dy", dy))}
    mm = lambda a, b, sa, sb: torch._scaled_mm(a, b, scale_a=sa.view(-1, 1), scale_b=sb.view(1, -1),  # noqa: E731
                                               out_dtype=torch.bfloat16)
    cx, sx, ctx, stx = q["x"]
    cw, sw, ctw, stw = q["w"]
    cd, sd, ctd, std = q["dy"]
    got = {"forward": mm(cx, cw.t(), sx, sw), "data gradient": mm(cd, ctw.t(), sd, stw),
           "weight gradient": mm(ctd, ctx.t(), std, stx)}
    want = {"forward": x @ w.T, "data gradient": dy @ w, "weight gradient": dy.T @ x}
    torch.cuda.synchronize()
    for name in got:
        ref = torch.from_numpy(want[name]).to(torch.bfloat16)                # one RNE rounding of the exact value
        assert torch.equal(got[name].cpu().view(torch.int16), ref.view(torch.int16)), name


# ------------------------------------------------------------------------------------------- quantize
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_matches_reference(src, fmt):
    rng = np.random.default_rng([DT_CODE[src], F8_CODE[fmt], 41])
    for rows, cols in SHAPES:
        host = values(src, rows * cols, rng)
        for side in SIDES:
            run(src, fmt, host, rows, cols, side)
        run(src, fmt, X.finite(src, rows * cols, rng, 3.0), rows, cols, "both", what="finite")
    for offs in ((1, 0, 0), (0, 3, 0), (0, 0, 5)):
        for side in SIDES:
            run(src, fmt, X.finite(src, 128 * 256, rng, 2.0), 128, 256, side, offs)


@pytest.mark.parametrize("src", ("f32", "bf16", "f64"))
def test_wide_rows(src):
    rows, cols = 32, 65536 + 128
    rng = np.random.default_rng([43, DT_CODE[src]])
    x = rng.uniform(-1.0, 1.0, (rows, cols))
    for r in range(rows):                                       # each row's maximum in a different tile
        x[r, (2053 * r) % cols] = 3.0 * (r + 1)
    run(src, "e4m3", storage(x.ravel(), src), rows, cols, "both", what="wide")


@pytest.mark.parametrize("src", ("f32", "f16", "f64"))
def test_planted_maxima_in_the_last_tile_and_band(src):
    """A row's maximum at each position of the row's last tile, and a column's maximum at each row of the last band."""
    rng = np.random.default_rng([47, DT_CODE[src]])
    rows, cols = 256 + 128, 512
    x = rng.uniform(-1.0, 1.0, (rows, cols))
    for r in range(rows):
        x[r, cols - 128 + r % 128] = -5.0 * (1 + r % 9)
    for j in range(cols):
        x[rows - 128 + j % 128, j] = 40.0 * (1 + j % 5)
    for side in SIDES:
        run(src, "e4m3", storage(x.ravel(), src), rows, cols, side, what="planted")
    # the ragged per-element path
    y = x[:rows - 3, :cols - 5]
    run(src, "e5m2", storage(y.ravel(), src), *y.shape, "both", what="planted ragged")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_value_classes(src, fmt):
    rows, cols = 128, 512
    emax = {"e4m3": 8, "e5m2": 15}[fmt]
    x = np.random.default_rng(3).uniform(-1, 1, (rows, cols))
    x[0:16] = 0.0                                               # all-zero rows
    x[16:32] = np.where(np.arange(cols) % 2, np.inf, np.nan)   # NaN / inf only
    tiny = {"f32": 2.0 ** -149, "f64": 5e-324, "f16": 2.0 ** -24, "bf16": 2.0 ** -133}[src]
    x[32:48] *= tiny * 8
    ulp = {"f32": 2.0 ** -23, "f64": 2.0 ** -52, "f16": 2.0 ** -10, "bf16": 2.0 ** -7}[src]
    for r in range(48, rows):
        x[r, (7 * r) % cols] = 1.75 * 2.0 ** (r % 7 - 3) * (1 + (r % 3 - 1) * ulp)
    run(src, fmt, storage(x.ravel(), src), rows, cols, "both", what="classes")
    if src == "f64":                                            # k clamps at -126: the rows saturate
        y = np.random.default_rng(4).uniform(-1, 1, (128, 256)) * 2.0 ** (126 + emax + 40)
        _, s, _, st = run(src, fmt, y.ravel(), 128, 256, "both", what="clamp")
        assert bool((s == 2.0 ** 126).all()) and bool((st == 2.0 ** 126).all())


@pytest.mark.parametrize("src", ("f32", "bf16"))
def test_cross_checks(src):
    rng = np.random.default_rng([5, DT_CODE[src]])
    rows, cols = 384, 640
    a = to_dev(X.finite(src, rows * cols, rng, 2.0), src).view(rows, cols)
    a[7].zero_()
    out, s, out_t, s_t = va.quantize_fp8_rowwise(a, "e4m3")
    # S and St are the largest 1x128 block scales
    _, bs, _, bst = va.quantize_fp8_blockwise(a, "e4m3", block="1x128")
    assert torch.equal(s, bs.amax(dim=1)) and torch.equal(s_t, bst.amax(dim=1))
    # C's row r is quantize_fp8 of row r with k_r
    k = (127 - (s.view(torch.int32) >> 23)).cpu().tolist()
    for r in range(0, rows, 37):
        q = va.quantize_fp8(a[r].contiguous(), "e4m3", scale_exp=int(k[r]))
        assert torch.equal(out[r].view(torch.uint8), q.view(torch.uint8)), r
    # the column-wise side is the row-wise side of A^T
    r_out, r_s, _, _ = va.quantize_fp8_rowwise(a.t().contiguous(), "e4m3", columnwise=False)
    torch.cuda.synchronize()
    assert torch.equal(out_t.view(torch.uint8), r_out.view(torch.uint8)) and torch.equal(s_t, r_s)


# ------------------------------------------------------------------------------------------- dequantize
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dst", DTYPES)
def test_dequantize(dst, fmt):
    rng = np.random.default_rng([7, DT_CODE[dst], F8_CODE[fmt]])
    for rows, cols in ((256, 384), (130, 200), (1, 1), (40, 16), (300, 1)):
        q = rng.integers(0, 256, rows * cols, dtype=np.uint8)
        s = (rng.uniform(0.5, 2.0, rows) * np.exp2(rng.integers(-140, 120, rows))).astype(np.float32)
        s[::7] = np.float32(np.nan)
        s[1::11] = np.float32(np.inf)
        s[2::13] = np.float32(-np.inf)
        s[3::17] = 0
        s[4::19] = np.float32(2.0 ** -149)
        qd, sd = to_dev(q, fmt).view(rows, cols), torch.from_numpy(s).cuda()
        got = va.dequantize_fp8_rowwise(qd, sd, dst)
        torch.cuda.synchronize()
        want = RE.dequantize(q, s, fmt, dst, rows, cols)
        assert_matches(got.reshape(-1), to_dev(want, dst), dst, f"{dst} {fmt} {rows}x{cols}")


def test_round_trip():
    rng = np.random.default_rng(11)
    rows, cols = 256, 512
    a = torch.from_numpy(rng.standard_normal((rows, cols)) * np.exp2(rng.integers(-30, 30, (rows, 1)))).cuda()
    out, s, out_t, s_t = va.quantize_fp8_rowwise(a, "e4m3")
    back = va.dequantize_fp8_rowwise(out, s, "f64")
    back_t = va.dequantize_fp8_rowwise(out_t, s_t, "f64")
    torch.cuda.synchronize()
    # elements within 2^6 of their row's (or column's) largest magnitude are E4M3 normals after scaling: relative
    # error <= 2^-4
    for b, ref in ((back, a), (back_t, a.t())):
        big = ref.abs() >= ref.abs().amax(dim=1, keepdim=True) / 64
        assert float(((b - ref).abs() / ref.abs())[big].max()) <= 2.0 ** -4


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_in_order_and_write_nothing():
    L = capi.lib
    buf = torch.full((1 << 21,), POISON, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    R, Cc = 128, 256
    n = R * Cc
    need = RE.workspace_bytes(R, Cc)
    A_, C_, S_, T_, ST_ = base + 4096, base + 4096 + 4 * n, base + 8192 + 5 * n, base + 12288 + 6 * n, base + 16384 + 7 * n
    W_ = base + 20480 + 8 * n
    good = dict(src=0, a=A_, fmt=0, rows=R, cols=Cc, c=C_, s=S_, ct=T_, st=ST_, w=W_, wb=need)
    # (argument, faulty value, code) in check order
    faults = [("src", 9, capi.ERR_VARIANT), ("fmt", 5, capi.ERR_VARIANT),
              ("s", None, capi.ERR_INVALID), ("st", None, capi.ERR_INVALID), ("a", None, capi.ERR_INVALID),
              ("rows", 1 << 40, capi.ERR_INVALID), ("w", None, capi.ERR_INVALID), ("wb", need - 1, capi.ERR_INVALID),
              ("a", A_ + 2, capi.ERR_ALIGN), ("s", S_ + 2, capi.ERR_ALIGN), ("st", ST_ + 1, capi.ERR_ALIGN),
              ("w", W_ + 2, capi.ERR_ALIGN),
              ("c", A_ + 64, capi.ERR_OVERLAP), ("ct", C_ + 100, capi.ERR_OVERLAP), ("s", T_ + 4, capi.ERR_OVERLAP),
              ("st", S_ + 8, capi.ERR_OVERLAP), ("w", ST_ + 4 * Cc - 4, capi.ERR_OVERLAP)]

    def call(args):
        return L.b200va_quantize_fp8_rowwise(args["src"], args["a"], args["fmt"], args["rows"], args["cols"],
                                             args["c"], args["s"], args["ct"], args["st"], args["w"], args["wb"], None)

    torch.cuda.synchronize()
    for i, (name, value, code) in enumerate(faults):
        assert call(dict(good, **{name: value})) == code, (name, value)
        for name2, value2, code2 in faults[i + 1:]:
            if name2 == name:
                continue
            assert call(dict(good, **{name: value, name2: value2})) == code, (name, value, name2, value2)
    assert call(dict(good, c=None, s=None, ct=None, st=None)) == capi.ERR_INVALID
    assert call(dict(good, rows=0, c=None, s=None, ct=None, st=None, w=None, wb=0)) == 0
    assert call(dict(good, cols=0, w=None, wb=0)) == 0
    torch.cuda.synchronize()
    assert bool((buf == POISON).all()), "a rejected call wrote"
    # dequantize
    D = lambda **k: L.b200va_dequantize_fp8_rowwise(k.get("fmt", 0), A_, k.get("s", S_), k.get("dst", 0),  # noqa
                                                    k.get("c", C_), R, Cc, None)
    assert D(dst=7) == capi.ERR_VARIANT and D(fmt=2) == capi.ERR_VARIANT and D(s=None) == capi.ERR_INVALID
    assert D(c=C_ + 2) == capi.ERR_ALIGN and D(s=S_ + 1) == capi.ERR_ALIGN and D(c=A_ + 8) == capi.ERR_OVERLAP
    assert D(s=C_ + 4 * n - 4) == capi.ERR_OVERLAP
    torch.cuda.synchronize()
    assert bool((buf == POISON).all()), "a rejected dequantize wrote"


# ------------------------------------------------------------------------------------------- streams and graphs
def test_graph_capture_and_stream_chain():
    rows, cols = 512, 1024
    a = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    outs = [torch.empty(rows, cols, dtype=torch.float8_e4m3fn, device="cuda"),
            torch.empty(rows, dtype=torch.float32, device="cuda"),
            torch.empty(cols, rows, dtype=torch.float8_e4m3fn, device="cuda"),
            torch.empty(cols, dtype=torch.float32, device="cuda")]
    ws = torch.empty(RE.workspace_bytes(rows, cols), dtype=torch.uint8, device="cuda")
    back = torch.empty(cols, rows, dtype=torch.float32, device="cuda")
    kw = dict(out=outs[0], scales=outs[1], out_t=outs[2], scales_t=outs[3], workspace=ws)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        va.quantize_fp8_rowwise(a, "e4m3", **kw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        q = va.quantize_fp8_rowwise(a, "e4m3", **kw)
        va.dequantize_fp8_rowwise(q[2], q[3], "f32", out=back)
    for scale in (1.0, 2.0 ** 20, 2.0 ** -20):
        a.copy_(torch.randn(rows, cols, device="cuda") * scale)
        g.replay()
        torch.cuda.synchronize()
        host = a.view(torch.int16).cpu().numpy().view(np.uint16).ravel()
        wc, wsc, wct, wst = RE.quantize(host, "bf16", "e4m3", rows, cols)
        assert np.array_equal(outs[0].view(torch.uint8).cpu().numpy(), wc)
        assert np.array_equal(outs[1].cpu().numpy().view(np.int32), wsc.view(np.int32))
        assert np.array_equal(outs[2].view(torch.uint8).cpu().numpy(), wct)
        assert np.array_equal(outs[3].cpu().numpy().view(np.int32), wst.view(np.int32))
        want = RE.dequantize(wct.ravel(), wst, "e4m3", "f32", cols, rows)
        assert np.array_equal(back.cpu().numpy().ravel().view(np.int32), want.view(np.int32))
    # a chain on one stream: convert -> row-wise quantize -> dequantize, each reading what the one before wrote
    x = torch.randn(rows, cols, device="cuda")
    for _ in range(3):
        h = va.convert(x, "f16")
        c1, s1, _, _ = va.quantize_fp8_rowwise(h.view(rows, cols), "e5m2", columnwise=False, workspace=ws)
        d = va.dequantize_fp8_rowwise(c1, s1, "f32")
        torch.cuda.synchronize()
        host = h.view(torch.int16).cpu().numpy().view(np.uint16).ravel()
        wc, wsc, _, _ = RE.quantize(host, "f16", "e5m2", rows, cols)
        assert np.array_equal(c1.view(torch.uint8).cpu().numpy(), wc)
        want = RE.dequantize(wc.ravel(), wsc, "e5m2", "f32", rows, cols)
        assert np.array_equal(d.cpu().numpy().ravel().view(np.int32), want.view(np.int32))
        x = x * 3.0


def test_tail_behind_a_k2d_writer(env):  # noqa: F811
    """The row-wise quantize of X's last 2^18 elements right behind the K2d add that writes X (last, in tile order):
    each of the three launches waits for the one before, and the first for the writer."""
    rows, cols = 256, 1024
    lo = GH.N - rows * cols
    ref = O.vadd(O.fill_ctr(rows * cols, GH.SEED_P, lo), O.fill_ctr(rows * cols, GH.SEED_Q, lo))
    wc, ws, wct, wst = RE.quantize(ref, "f32", "e4m3", rows, cols)
    ws_buf = torch.empty(RE.workspace_bytes(rows, cols), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        GH._poison(env)
        va.add(env["P"], env["Q"], env["X"], variant="k2")
        c, s, ct, st = va.quantize_fp8_rowwise(env["X"][lo:].view(rows, cols), "e4m3", workspace=ws_buf)
        torch.cuda.synchronize()
        assert np.array_equal(c.view(torch.uint8).cpu().numpy(), wc)
        assert np.array_equal(ct.view(torch.uint8).cpu().numpy(), wct)
        assert np.array_equal(s.cpu().numpy().view(np.int32), ws.view(np.int32))
        assert np.array_equal(st.cpu().numpy().view(np.int32), wst.view(np.int32))


def test_planned_launches(tmp_path):
    """Quantize is three launches of the block-scaled kernel of its element size: the maxima and the cast with
    256-thread CTAs, one per 128 x 128 tile on the tiled path, and the reduction with one thread per row and column;
    dequantize is one launch with plan_geometry's grid (one unit per 16-byte output slice).  On the ragged path the
    maxima take one thread per 1x128 block and the cast one per element."""
    rows, cols = 256, 512
    a = torch.randn(rows, cols, device="cuda")
    r = torch.randn(100, 200, device="cuda", dtype=torch.float16)
    q = va.quantize_fp8_rowwise(a, "e4m3")
    qr = va.quantize_fp8_rowwise(r, "e4m3", columnwise=False)
    ws = torch.empty(RE.workspace_bytes(rows, cols), dtype=torch.uint8, device="cuda")
    d32 = torch.empty(rows, cols, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()

    def plan():
        va.quantize_fp8_rowwise(a, "e4m3", out=q[0], scales=q[1], out_t=q[2], scales_t=q[3], workspace=ws)
        va.dequantize_fp8_rowwise(q[0], q[1], "f32", out=d32)
        va.quantize_fp8_rowwise(r, "e4m3", columnwise=False, out=qr[0], scales=qr[1], workspace=ws)
        torch.cuda.synchronize()

    tiles, slices = rows // 128 * (cols // 128), rows * cols // 16
    want = [("mx_quant_vec<4>", tiles, 256), ("mx_quant_vec<4>", -(-(rows + cols) // 256), 256),
            ("mx_quant_vec<4>", tiles, 256), ("mx_dequant_vec<4>", slices * 4 // 256, 256),
            ("mx_quant_vec<2>", -(-100 * 2 // 256), 256), ("mx_quant_vec<2>", 1, 256),
            ("mx_quant_vec<2>", -(-100 * 200 // 256), 256)]
    for attempt in range(3):
        try:
            got = kernels_after_marker(tmp_path, plan, ("mx_",))
            break
        except ValueError:
            if attempt == 2:
                raise
    assert got == want


def test_ct_index_past_2_32():
    """65536 x 65664 f16 on the tiled path: Ct's last rows lie past byte 2^32.  The last 128 rows' and columns' scales
    and the bottom-right 128 x 128 corner of C and Ct are checked against the reference on the rows and columns they
    belong to (the input repeats a 2^20-element block)."""
    rows, cols = 65536, 65664
    assert (cols - 1) * rows > 1 << 32
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    assert free >= 4 * rows * cols + (2 << 30), f"needs about 19 GiB of free device memory, {free >> 30} GiB free"
    block = torch.from_numpy(X.finite("f16", 1 << 20, np.random.default_rng(13), 4.0).view(np.int16)).cuda()
    a = block.repeat(-(-rows * cols // block.numel()))[:rows * cols].view(torch.float16).view(rows, cols)
    out, s, out_t, s_t = va.quantize_fp8_rowwise(a, "e4m3")
    torch.cuda.synchronize()
    i0, j0 = rows - 128, cols - 128
    host_rows = a[i0:].contiguous().view(torch.int16).cpu().numpy().view(np.uint16).ravel()
    wc, ws, _, _ = RE.quantize(host_rows, "f16", "e4m3", 128, cols)
    assert np.array_equal(out[i0:].view(torch.uint8).cpu().numpy(), wc)
    assert np.array_equal(s[i0:].cpu().numpy(), ws)
    host_cols = a[:, j0:].contiguous().view(torch.int16).cpu().numpy().view(np.uint16).ravel()
    _, _, wct, wst = RE.quantize(host_cols, "f16", "e4m3", rows, 128)
    assert np.array_equal(out_t[j0:].view(torch.uint8).cpu().numpy(), wct)
    assert np.array_equal(s_t[j0:].cpu().numpy(), wst)
    del a, out, out_t, block
    torch.cuda.empty_cache()
