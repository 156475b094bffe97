"""b200va_quantize_fp8_transpose and b200va_quantize_fp8_transpose_auto on the GPU, bit for bit.

The reference is the 1-D one on the flattened A (oracle/fp8_exact.py, tests/fp8_auto_exact.py for k), reshaped and
transposed in numpy: C must hold its bytes (NaN matches NaN as a class) and Ct[j, i] == C[i, j]; *d_amax must hold
the bits the 1-D call leaves on the same A.  C and Ct are poisoned beforehand and their guard elements must keep the
poison.

- Every source type and format at k in {-126, -8, 0, 5, 126} (host k) and margins {0, 1, 126} (_auto), on random bit
  patterns (every value class) with +-0, subnormals, +-inf, NaN payloads and values past saturation planted.
- The tiled path: rows, cols in {16, 48, 64, 80, 128, 1040}, 16 x 65536 and 65536 x 16, partial tiles on both edges.
- The element path: rows or cols in {1, 15, 17, 63, 65, 1000}, 1 x n, n x 1, and 16-multiple shapes with A, C or Ct
  off a 16-byte boundary.
- 16384 x 16384 f16 (the HBM class) and 65536 x 65552 f16 (rows cols > 2^32, so Ct's index needs 64 bits).
- The amax: NULL accepted, a NaN gives NaN in the host form and is skipped in _auto.
- Every rejected argument writes nothing, *d_amax and *d_scale_exp included.
- A stream op -> quantize-transpose -> dequantize of Ct chain on one stream, a quantize-transpose tail behind the
  K2d writer of gpu_helpers' chains, and a captured _auto graph replayed with inputs that move by 2^+-20.
- A profiler trace of the planned launches, and the _auto amax pass equal to quantize_fp8_auto's.
- One torch._scaled_mm weight-gradient product taking out_t.t() directly.
This module's name sorts after test_gpu_typecast.py, as the other FP8 modules' do (DESIGN.md section 3).
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

    from gpu_helpers import (DT_CODE, ES, F8_CODE, GUARD, LO, POISON, TORCH, M, _chains, _run, assert_guards,
                             assert_matches, expected_cast_launch, hbm_n, kernels_after_marker, poisoned, tiled, to_dev)
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = V.DTYPES
FMTS = F.FORMATS8
KS = (-126, -8, 0, 5, 126)
MARGINS = (0, 1, 126)
K_POISON = -999
TILED = (16, 48, 64, 80, 128, 1040)
RAGGED = (1, 15, 17, 63, 65, 1000)


# ------------------------------------------------------------------------------------------- helpers
def storage(x, src):
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        return x.astype(X.STORAGE[src]) if src in ("f32", "f64") else V.round_f64(x, src)


def amax_bits(m) -> int:
    return int(m.view(torch.int64).item()) & ((1 << 64) - 1)


def values(src, n, rng):
    """Random bit patterns (every value class) with +-0, the smallest subnormals, +-inf, NaN payloads and values past
    the FP8 range planted."""
    host = V.random_bits(src, n, rng)
    tiny = {"f32": 2.0 ** -149, "f64": 5e-324, "f16": 2.0 ** -24, "bf16": 2.0 ** -133}[src]
    planted = storage([0.0, -0.0, np.inf, -np.inf, 1e5, -6e4, tiny, -tiny, 2.0 ** -20, 1.0, -1.5], src)
    for i, v in enumerate(planted):
        host[(i * 37) % n::97] = v
    return host


def transpose_bytes(flat, rows, cols):
    """The rows x cols bytes flat, transposed, flat again."""
    return np.ascontiguousarray(np.asarray(flat).reshape(rows, cols).T).reshape(-1)


def run_case(src, fmt, host, rows, cols, *, k=None, margin=None, acc=0.0, offs=(0, 0, 0), amax=True, what=""):
    """One quantize-transpose of host (rows x cols) with A, C and Ct at element offsets offs in poisoned buffers:
    host k when margin is None, else _auto.  C, Ct, the guards, the amax bits and k against the reference."""
    n = rows * cols
    oa, oc, ot = offs
    what = f"{src}->{fmt} {rows}x{cols} k={k} margin={margin} offs={offs} {what}"
    ab, a = poisoned(n, src, oa)
    a.copy_(to_dev(host, src))
    cb, c = poisoned(n, fmt, oc)
    tb, ct = poisoned(n, fmt, ot)
    m = torch.full((1,), acc, dtype=torch.float64, device="cuda") if amax else None
    if margin is None:
        out = va.quantize_fp8_transpose(a.view(rows, cols), fmt, scale_exp=k, amax=m, out=c.view(rows, cols),
                                        out_t=ct.view(cols, rows))
        want, wk = F.quantize(host, src, fmt, k), k
        m1 = torch.full((1,), acc, dtype=torch.float64, device="cuda")
        va.quantize_fp8(a, fmt, scale_exp=k, amax=m1)                  # the 1-D call's amax bits
    else:
        s = torch.full((1,), K_POISON, dtype=torch.int32, device="cuda")
        out = va.quantize_fp8_transpose_auto(a.view(rows, cols), fmt, margin=margin, amax=m, scale_exp=s,
                                             out=c.view(rows, cols), out_t=ct.view(cols, rows))
        assert out[2] is s
        want, wk, wm = A.quantize_auto(host, src, fmt, margin, acc)
    torch.cuda.synchronize()
    assert out[0].data_ptr() == c.data_ptr() and out[1].data_ptr() == ct.data_ptr()
    assert_matches(c, to_dev(want, fmt), fmt, what + " C")
    assert_matches(ct, to_dev(transpose_bytes(want, rows, cols), fmt), fmt, what + " Ct")
    assert_guards(cb, GUARD + oc, n, what + " C")
    assert_guards(tb, GUARD + ot, n, what + " Ct")
    if margin is None:
        if m is not None:
            assert amax_bits(m) == amax_bits(m1), (what, float(m.item()), float(m1.item()))
    else:
        assert int(s.item()) == wk, (what, int(s.item()), wk)
        assert amax_bits(m) == A.f64_bits(wm), (what, float(m.item()), wm)
    return want, wk


# ------------------------------------------------------------------------------------------- types, formats, scales
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_types_formats_and_scales(src, fmt):
    rng = np.random.default_rng([1, DT_CODE[src], F8_CODE[fmt]])
    for rows, cols in ((48, 80), (17, 63)):                   # the tiled path, the element path
        host = values(src, rows * cols, rng)
        for k in KS:
            run_case(src, fmt, host, rows, cols, k=k)
        for margin in MARGINS:
            run_case(src, fmt, host, rows, cols, margin=margin)
            finite = X.finite(src, rows * cols, rng, 2.0 ** (margin % 7 - 3))
            run_case(src, fmt, finite, rows, cols, margin=margin, what="finite")


# ------------------------------------------------------------------------------------------- shapes
@pytest.mark.parametrize("src", DTYPES)
def test_tiled_shapes(src):
    rng = np.random.default_rng([2, DT_CODE[src]])
    for i, rows in enumerate(TILED):
        for j, cols in enumerate(TILED):
            fmt = FMTS[(i + j) % 2]
            host = X.finite(src, rows * cols, rng, 4.0)
            if (i + j) % 3 == 0:
                run_case(src, fmt, host, rows, cols, margin=(i + j) % 2)
            else:
                run_case(src, fmt, host, rows, cols, k=KS[(i + j) % 5])


@pytest.mark.parametrize("src", DTYPES)
def test_tall_and_wide(src):
    rng = np.random.default_rng([3, DT_CODE[src]])
    for rows, cols in ((16, 65536), (65536, 16), (1040, 4112)):
        host = X.finite(src, rows * cols, rng, 8.0)
        run_case(src, "e4m3", host, rows, cols, k=2)
        run_case(src, "e5m2", host, rows, cols, margin=1)


@pytest.mark.parametrize("src", DTYPES)
def test_element_path_shapes_give_the_same_bytes(src):
    rng = np.random.default_rng([4, DT_CODE[src]])
    shapes = [(r, c) for r in RAGGED for c in (16, 65)] + [(c, r) for r in RAGGED for c in (16, 64)]
    shapes += [(1, 5003), (5003, 1), (1, 1), (1000, 1000)]
    for i, (rows, cols) in enumerate(shapes):
        host = X.finite(src, rows * cols, rng, 2.0)
        fmt = FMTS[i % 2]
        if i % 2:
            run_case(src, fmt, host, rows, cols, margin=i % 3)
        else:
            run_case(src, fmt, host, rows, cols, k=KS[i % 5])


@pytest.mark.parametrize("src", DTYPES)
def test_misaligned_operands_take_the_element_path_with_the_same_bytes(src):
    """16-multiple shapes with A, C or Ct off a 16-byte boundary: the same bytes as the aligned (tiled) call."""
    rng = np.random.default_rng([5, DT_CODE[src]])
    host = X.finite(src, 48 * 80, rng, 4.0)
    for offs in ((1, 0, 0), (0, 1, 0), (0, 0, 3), (1, 5, 7)):
        for fmt in FMTS:
            run_case(src, fmt, host, 48, 80, k=-8, offs=offs)
            run_case(src, fmt, host, 48, 80, margin=1, offs=offs)


def _check_big(a2d, block, fmt, k, what):
    """C against the tiled reference of block, then Ct against C transposed, in column chunks on the device."""
    rows, cols = a2d.shape
    q, qt = va.quantize_fp8_transpose(a2d, fmt, scale_exp=k)
    want = tiled(F.quantize(block, "f16", fmt, k), rows * cols, fmt)
    assert_matches(q.view(-1), want, fmt, what + " C")
    del want
    qb, qtb = q.view(torch.uint8), qt.view(torch.uint8)
    step = max(1, (1 << 26) // rows)
    for j in range(0, cols, step):
        if not bool(torch.equal(qtb[j:j + step], qb[:, j:j + step].t())):
            raise AssertionError(f"{what}: Ct rows {j}..{j + step} differ from C's columns")
    return q, qt


def test_the_hbm_class_16384_square_f16():
    rows = cols = 16384
    assert rows * cols >= hbm_n(2)
    block = X.finite("f16", 199_999, np.random.default_rng(6), 1.0)
    a = tiled(block, rows * cols, "f16").view(rows, cols)
    _check_big(a, block, "e4m3", 3, "16384 x 16384")


def test_rows_times_cols_past_2_32_f16():
    """65536 x 65552 f16 (16 GiB in all): Ct's index (j rows + i) passes 2^32."""
    rows, cols = 65536, 65552
    n = rows * cols
    assert n > 1 << 32
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    assert free >= 2 * n + 2 * n + n + (2 << 30), f"needs about 22 GiB of free device memory, {free >> 30} GiB free"
    block = X.finite("f16", 199_999, np.random.default_rng(7), 0.5)
    a = tiled(block, n, "f16").view(rows, cols)
    _check_big(a, block, "e5m2", -2, "65536 x 65552")


# ------------------------------------------------------------------------------------------- amax
@pytest.mark.parametrize("src", DTYPES)
def test_amax_null_and_nan(src):
    rng = np.random.default_rng([8, DT_CODE[src]])
    for rows, cols in ((64, 64), (15, 33)):
        host = X.finite(src, rows * cols, rng, 3.0)
        run_case(src, "e4m3", host, rows, cols, k=0, amax=False, what="NULL amax")
        run_case(src, "e4m3", host, rows, cols, k=0, acc=1e300, what="running amax")
        for pos in (0, rows * cols // 2, rows * cols - 1):
            nan = host.copy()
            nan[pos] = storage([np.nan], src)[0]
            run_case(src, "e5m2", nan, rows, cols, k=1, what=f"NaN at {pos}")
            _, k = run_case(src, "e5m2", nan, rows, cols, margin=0, what=f"NaN at {pos}")
            assert k == A.auto_scale_exp(float(np.abs(X.widen(host, src)[np.arange(host.size) != pos]).max()), "e5m2", 0)


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 17, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A_, R, C = buf.data_ptr() + 4096, 16, 64
    n = R * C
    C_, T_, M_, S_ = A_ + 16384, A_ + 32768, A_ + 49152, A_ + 49168
    F32, F64, F16 = 0, 1, 2
    E4, E5 = capi.F8_E4M3, capi.F8_E5M2
    big = 1 << 32
    h = [   # host form: (src, A, fmt, C, Ct, rows, cols, k, amax)
        ((4, A_, E4, C_, T_, R, C, 0, M_), capi.ERR_VARIANT), ((F32, A_, 2, C_, T_, R, C, 0, M_), capi.ERR_VARIANT),
        ((F32, A_, E4, C_, T_, R, C, -127, M_), capi.ERR_INVALID), ((F32, A_, E4, C_, T_, R, C, 127, M_), capi.ERR_INVALID),
        ((F32, None, E4, C_, T_, R, C, 0, M_), capi.ERR_INVALID), ((F32, A_, E4, None, T_, R, C, 0, M_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, None, R, C, 0, M_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, T_, 1 << 20, (1 << 20) + 16, 0, M_), capi.ERR_INVALID),        # n > 2^40
        ((F32, A_, E4, C_, T_, big, big, 0, M_), capi.ERR_INVALID),                        # wraps to 0
        ((F32, A_, E4, C_, T_, big + 1, big, 0, M_), capi.ERR_INVALID),                    # wraps to 2^32
        ((F32, A_ + 2, E4, C_, T_, R, C, 0, M_), capi.ERR_ALIGN), ((F64, A_ + 4, E4, C_, T_, R, C, 0, M_), capi.ERR_ALIGN),
        ((F16, A_ + 1, E5, C_, T_, R, C, 0, M_), capi.ERR_ALIGN), ((F32, A_, E4, C_, T_, R, C, 0, M_ + 4), capi.ERR_ALIGN),
        ((F32, A_, E4, A_ + 8, T_, R, C, 0, M_), capi.ERR_OVERLAP), ((F32, A_, E4, C_, A_ + 4 * n - 1, R, C, 0, M_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, C_ + n - 1, R, C, 0, M_), capi.ERR_OVERLAP), ((F32, A_, E4, T_ + 3, T_, R, C, 0, M_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, T_, R, C, 0, A_ + 8), capi.ERR_OVERLAP), ((F32, A_, E4, C_, T_, R, C, 0, C_ + 8), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, T_, R, C, 0, T_ + n - 8), capi.ERR_OVERLAP), ((F32, A_, E4, C_, M_ - n + 1, R, C, 0, M_), capi.ERR_OVERLAP),
    ]
    q = [   # _auto: (src, A, fmt, C, Ct, rows, cols, margin, amax, scale_exp)
        ((4, A_, E4, C_, T_, R, C, 0, M_, S_), capi.ERR_VARIANT),
        ((F32, A_, E4, C_, T_, R, C, -1, M_, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, T_, R, C, 127, M_, S_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, T_, R, C, 0, None, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, T_, R, C, 0, M_, None), capi.ERR_INVALID),
        ((F32, A_, E4, C_, None, R, C, 0, M_, S_), capi.ERR_INVALID), ((F32, A_, E4, C_, T_, big, big, 0, M_, S_), capi.ERR_INVALID),
        ((F32, A_, E4, C_, T_, R, C, 0, M_, S_ + 2), capi.ERR_ALIGN), ((F32, A_ + 2, E4, C_, T_, R, C, 0, M_, S_), capi.ERR_ALIGN),
        ((F32, A_, E4, C_, T_, R, C, 0, M_, T_ + 100), capi.ERR_OVERLAP), ((F32, A_, E4, C_, T_, R, C, 0, T_ + 8, S_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, T_, R, C, 0, M_, M_ + 4), capi.ERR_OVERLAP), ((F32, A_, E4, C_, T_, R, C, 0, M_, A_), capi.ERR_OVERLAP),
        ((F32, A_, E4, C_, A_ + 16, R, C, 0, M_, S_), capi.ERR_OVERLAP), ((F32, A_, E4, C_, C_ + 16, R, C, 0, M_, S_), capi.ERR_OVERLAP),
    ]
    for args, code in h:
        assert L.b200va_quantize_fp8_transpose(*args, None) == code, (args, code)
    for args, code in q:
        assert L.b200va_quantize_fp8_transpose_auto(*args, None) == code, (args, code)
    # rows == 0 or cols == 0: nothing to do, nothing written, nothing launched
    for rows, cols in ((0, 64), (64, 0), (0, big)):
        assert L.b200va_quantize_fp8_transpose(F32, None, E4, None, None, rows, cols, 0, M_, None) == capi.OK
        assert L.b200va_quantize_fp8_transpose_auto(F32, A_, E4, C_, T_, rows, cols, 0, M_, S_, None) == capi.OK
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == POISON).all(), "a rejected or empty call wrote to device memory"
    # right behind each other: no overlap, and the calls run
    assert L.b200va_quantize_fp8_transpose(F32, A_, E4, A_ + 4 * n, A_ + 5 * n, R, C, 0, A_ + 6 * n, None) == capi.OK
    assert L.b200va_quantize_fp8_transpose_auto(F32, A_, E4, A_ + 4 * n, A_ + 5 * n, R, C, 0, A_ + 6 * n,
                                                A_ + 6 * n + 8, None) == capi.OK
    torch.cuda.synchronize()


def test_the_wrappers_check_their_operands():
    a = torch.zeros(32, 48, dtype=torch.float16, device="cuda")
    for bad in (dict(out=torch.empty(48, 32, dtype=torch.float8_e4m3fn, device="cuda")),
                dict(out_t=torch.empty(32, 48, dtype=torch.float8_e4m3fn, device="cuda")),
                dict(out=torch.empty(32, 48, dtype=torch.float8_e5m2, device="cuda")),
                dict(out_t=torch.empty(96, 32, dtype=torch.float8_e4m3fn, device="cuda")[::2])):
        with pytest.raises(TypeError):
            va.quantize_fp8_transpose(a, "e4m3", **bad)
        with pytest.raises(TypeError):
            va.quantize_fp8_transpose_auto(a, "e4m3", **bad)
    for x in (a.view(-1), a.t(), a.view(4, 8, 48)):
        with pytest.raises(TypeError):
            va.quantize_fp8_transpose(x, "e4m3")


# ------------------------------------------------------------------------------------------- order and capture
def test_stream_op_quantize_transpose_dequantize_on_one_stream():
    """Six rounds on one stream without a host sync: b = s a (b200va_stream), (q, qt) = quantize-transpose(b, k_r),
    d_r = dequantize_fp8(qt, k_r).  Tiled and element-path shapes."""
    st = torch.cuda.Stream()
    for src, fmt, dst, (rows, cols) in (("f32", "e4m3", "f32", (1040, 2064)), ("bf16", "e5m2", "f16", (2048, 1024)),
                                        ("f64", "e4m3", "bf16", (999, 1001))):
        a0 = X.finite(src, rows * cols, np.random.default_rng(DT_CODE[src]), 8.0)
        a = to_dev(a0, src)
        b = torch.empty_like(a)
        q = torch.empty(rows, cols, dtype=TORCH[fmt], device="cuda")
        qt = torch.empty(cols, rows, dtype=TORCH[fmt], device="cuda")
        scalars = [2.0 ** (3 * r - 6) for r in range(6)]
        ks = [r - 3 for r in range(6)]
        ds = [torch.empty(rows * cols, dtype=TORCH[dst], device="cuda") for _ in scalars]
        torch.cuda.synchronize()
        for s, k, d in zip(scalars, ks, ds):
            va.stream("scale", a, None, b, scalar=s, stream=st)
            va.quantize_fp8_transpose(b.view(rows, cols), fmt, scale_exp=k, out=q, out_t=qt, stream=st)
            va.dequantize_fp8(qt.view(-1), TORCH[dst], scale_exp=k, out=d, stream=st)
        st.synchronize()
        for r, (s, k, d) in enumerate(zip(scalars, ks, ds)):
            want = F.dequantize(transpose_bytes(F.quantize(X.stream("scale", src, a0, None, s), src, fmt, k), rows, cols),
                                fmt, dst, k)
            assert_matches(d, to_dev(want, dst), dst, f"{src}->{fmt}->{dst} {rows}x{cols} round {r}")


def test_quantize_transpose_tail_reads_what_the_writer_wrote(env):
    """gpu_helpers' chains (the 2^28 K2d writer of X, then 0-3 middle launches) with a quantize-transpose of 64 x 4080
    elements of the end of X, on a 16-byte boundary (the tiled path), as the tail."""
    rows, cols = 64, 4080
    assert 3 + rows * cols <= M and (LO + 3) % 4 == 0
    middles, chains = _chains(env)
    q = torch.empty(rows, cols, dtype=torch.float8_e4m3fn, device="cuda")
    qt = torch.empty(cols, rows, dtype=torch.float8_e4m3fn, device="cuda")
    m = torch.zeros(1, dtype=torch.float64, device="cuda")
    window = env["ref_window"][3:3 + rows * cols]
    want = F.quantize(window, "f32", "e4m3", 2)
    want_t = transpose_bytes(want, rows, cols)
    want_amax = F.amax(window, "f32")

    def tail(w):
        m.zero_()
        va.quantize_fp8_transpose(w[3:3 + rows * cols].view(rows, cols), "e4m3", scale_exp=2, amax=m, out=q, out_t=qt)

    failures = []
    for names in chains:
        q.view(torch.uint8).fill_(POISON)
        qt.view(torch.uint8).fill_(POISON)
        _run(env, middles, names, tail)
        got, got_t = q.view(torch.uint8).cpu().numpy().reshape(-1), qt.view(torch.uint8).cpu().numpy().reshape(-1)
        bad, bad_t = np.flatnonzero(got != want).size, np.flatnonzero(got_t != want_t).size
        if bad or bad_t or float(m.item()) != want_amax:
            failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> quantize-transpose: {bad} C and {bad_t} Ct "
                            f"bytes differ, amax {float(m.item())!r} want {want_amax!r}")
    assert not failures, "\n".join(failures)


def test_captured_auto_graph_follows_the_scale_across_replays():
    """One graph: reset *d_amax, then quantize-transpose _auto, per case.  Between replays only the input changes, by
    2^20 either way, so each replay's k must come from its own amax on the device."""
    cases = []
    for src, fmt, (rows, cols) in (("f32", "e4m3", (256, 272)), ("bf16", "e5m2", (96, 1040)), ("f64", "e4m3", (80, 64)),
                                   ("f16", "e5m2", (63, 65))):
        a = torch.empty(rows * cols, dtype=TORCH[src], device="cuda")
        cb, c = poisoned(rows * cols, fmt)
        tb, ct = poisoned(rows * cols, fmt)
        cases.append((src, fmt, rows, cols, a, cb, c, tb, ct, torch.zeros(1, dtype=torch.float64, device="cuda"),
                      torch.zeros(1, dtype=torch.int32, device="cuda")))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for src, fmt, rows, cols, a, _, c, _, ct, m, s in cases:
                m.zero_()
                va.quantize_fp8_transpose_auto(a.view(rows, cols), fmt, margin=1, amax=m, scale_exp=s,
                                               out=c.view(rows, cols), out_t=ct.view(cols, rows))
    torch.cuda.synchronize()
    rng = np.random.default_rng(9)
    ks = {case[:2]: [] for case in cases}
    for r, e in enumerate((0, 20, 0, -20, 0)):
        hosts = []
        for src, fmt, rows, cols, a, cb, c, tb, ct, m, s in cases:
            host = X.finite(src, rows * cols, rng, 2.0 ** (e // 2 if src == "f16" else e))
            a.copy_(to_dev(host, src))
            hosts.append(host)
            cb.view(torch.uint8).fill_(POISON)
            tb.view(torch.uint8).fill_(POISON)
            m.fill_(1e300)
            s.fill_(K_POISON)
        g.replay()
        torch.cuda.synchronize()
        for host, (src, fmt, rows, cols, a, cb, c, tb, ct, m, s) in zip(hosts, cases):
            what = f"{src}->{fmt} {rows}x{cols} replay {r}"
            want, k, wm = A.quantize_auto(host, src, fmt, 1)
            assert int(s.item()) == k and amax_bits(m) == A.f64_bits(wm), (what, int(s.item()), k)
            assert_matches(c, to_dev(want, fmt), fmt, what)
            assert_matches(ct, to_dev(transpose_bytes(want, rows, cols), fmt), fmt, what + " Ct")
            assert_guards(cb, GUARD, rows * cols, what)
            assert_guards(tb, GUARD, rows * cols, what)
            ks[(src, fmt)].append(k)
    for key, seq in ks.items():
        assert len(set(seq)) == 3, (key, seq)


# ------------------------------------------------------------------------------------------- trace
def expected_transpose_launch(src, rows, cols, pa, pc, pt):
    """(kernel, grid, block) of plan_fp8_transpose (b200va_typed.cu): 256 threads and one 64 x 64 tile per CTA on
    the tiled path; else every element an edge item, 512 threads in A's HBM class and 256 below it."""
    n = rows * cols
    kernel = f"fp8_quant_vec<{DT_CODE[src]}>"
    if rows % 16 == 0 and cols % 16 == 0 and (pa | pc | pt) % 16 == 0:
        return kernel, min(-(-rows // 64) * -(-cols // 64), 2 ** 31 - 1), 256
    threads = 512 if n >= hbm_n(ES[src]) else 256
    return kernel, max(1, min(-(-n // threads), 2 ** 31 - 1)), threads


def test_trace_shows_the_planned_launches(tmp_path):
    """Per source type: tiled, ragged, misaligned and HBM-class shapes, host k and _auto.  After the marker: the
    planned launch per call and, for _auto, the amax pass first, the same launch quantize_fp8_auto makes on the same
    A; nothing else."""
    plan, want = [], []
    for i, src in enumerate(DTYPES):
        fmt = FMTS[i % 2]
        big = hbm_n(ES[src]) // 4096
        shapes = ((48, 80, 0), (1040, 16, 0), (17, 63, 0), (48, 80, 1), (4096, big, 0), (4097, big, 0))
        for rows, cols, off in shapes:
            n = rows * cols
            a = torch.zeros(n + off, dtype=TORCH[src], device="cuda")[off:].view(rows, cols)
            c = torch.empty(rows, cols, dtype=TORCH[fmt], device="cuda")
            ct = torch.empty(cols, rows, dtype=TORCH[fmt], device="cuda")
            q1 = torch.empty(n, dtype=TORCH[fmt], device="cuda")
            launch = expected_transpose_launch(src, rows, cols, a.data_ptr(), c.data_ptr(), ct.data_ptr())
            plan.append((a, fmt, c, ct, q1))
            want += [launch, "amax", launch, "amax", expected_cast_launch(f"fp8_quant_vec<{DT_CODE[src]}>", ES[src], 1, n,
                                                                                a.data_ptr(), q1.data_ptr())]
    m = torch.zeros(1, dtype=torch.float64, device="cuda")
    s = torch.zeros(1, dtype=torch.int32, device="cuda")

    def run_plan():
        for a, fmt, c, ct, q1 in plan:
            va.quantize_fp8_transpose(a, fmt, amax=m, out=c, out_t=ct)
            va.quantize_fp8_transpose_auto(a, fmt, amax=m, scale_exp=s, out=c, out_t=ct)
            va.quantize_fp8_auto(a.view(-1), fmt, amax=m, scale_exp=s, out=q1)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("fp8_",))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for j in range(0, len(want), 5):
        g, w = got[j:j + 5], want[j:j + 5]
        assert g[0] == w[0] and g[2] == w[2], (j // 5, g, w)
        assert g[1] == g[3], (j // 5, g)                 # the amax pass is quantize_fp8_auto's on the same A
        assert g[4] == w[4], (j // 5, g, w)


# ------------------------------------------------------------------------------------------- GEMM interop
def test_scaled_mm_takes_out_t_directly():
    """The weight gradient dW = dY^T X of a linear layer: torch._scaled_mm on the _auto outputs, mat1 = dY's out_t and
    mat2 = X's out_t.t() (column-major, no copy), equals the same call on out.t().contiguous() copies."""
    batch, d_out, d_in = 256, 128, 192
    gen = torch.Generator(device="cuda").manual_seed(10)
    dy = torch.randn(batch, d_out, device="cuda", generator=gen).to(torch.bfloat16)
    x = torch.randn(batch, d_in, device="cuda", generator=gen).to(torch.bfloat16) * 30
    dy_q, dy_t, dy_k = va.quantize_fp8_transpose_auto(dy, "e4m3")
    x_q, x_t, x_k = va.quantize_fp8_transpose_auto(x, "e4m3")
    sa, sb = torch.exp2(-dy_k.float()).reshape(()), torch.exp2(-x_k.float()).reshape(())
    got = torch._scaled_mm(dy_t, x_t.t(), sa, sb, out_dtype=torch.float32)
    ref = torch._scaled_mm(dy_q.t().contiguous(), x_q.t().contiguous().t(), sa, sb, out_dtype=torch.float32)
    assert torch.equal(got, ref)
    exact = (dy_t.float() * sa) @ (x_t.float() * sb).t()
    torch.testing.assert_close(got, exact, rtol=1e-2, atol=1.0)     # FP8 tensor-core accumulation is not exact f32
    assert torch.equal(dy_t.view(torch.uint8), dy_q.view(torch.uint8).t().contiguous())
