"""b200va_dot on the GPU, bit for bit against oracle/dot_exact.py (NaN matches NaN as a class).

- Every type at ragged sizes around the lane and chunk edges and on both sides of the HBM class (>= 2^25 words per
  operand, where the first rows are prefetched into L2 ahead of the wait), including a ragged HBM-class n with a
  chunk count that is no power of two.  f64 beyond the Fraction limit uses the exactly representable family.
- Every element offset within 16 bytes (the vector path with a head) and A and B in different phases (the scalar
  path) give the same bits; A == B; the adversarial, special-value and subnormal sets in both paths.
- Repeated calls, two streams, a replayed CUDA graph; ordering behind a stream op or add that writes the operands,
  with no host synchronisation; back-to-back dots sharing one workspace; f16 across byte and element 2^32.
- Argument errors, and nothing written outside d_out and the workspace bytes the call needs.
- A profiler trace of the launches: exactly the planned kernels with their grid and block, and nothing else.
"""
import json
import math

import numpy as np
import pytest

from conftest import has_gpu
from oracle import dot_exact as D
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va
    from test_gpu_parity import _profiled_kernel_name

    TORCH = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}

DTS = ["f32", "f64", "f16", "bf16"]
ES = {"f32": 4, "f64": 8, "f16": 2, "bf16": 2}
DT_CODE = {"f32": 0, "f64": 1, "f16": 2, "bf16": 3}
FORM = {"f32": (512, 4), "f64": (512, 2), "f16": (256, 4), "bf16": (256, 4)}     # dot_form: threads, rows
SMALL = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, D.LANES - 1, D.LANES + 1, D.CHUNK - 1, D.CHUNK + 1, 2 * D.CHUNK + 3,
         5_000_011]
POISON = 0x5A


def to_dev(x, dtype):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t.view(TORCH[dtype]) if dtype in ("f16", "bf16") else t


def hbm_n(dtype):
    """The smallest n in the HBM class: n * sizeof(T) / 4 >= 2^25."""
    return (1 << 25) * 4 // ES[dtype]


def bits(x: float) -> int:
    return int(np.float64(x).view(np.uint64))


def assert_same(got: float, want: float, what=""):
    assert (math.isnan(got) and math.isnan(want)) or bits(got) == bits(want), f"{what}: got {got!r} want {want!r}"


def dot(a, b, **kw) -> float:
    r = va.dot(a, b, **kw)
    torch.cuda.synchronize()
    return float(r.item())


def inputs(dtype, n, seed):
    """(host a, host b, the contract's value): random finite values, or the exact family for f64 beyond the
    Fraction limit."""
    if dtype == "f64" and n > X.FRACTION_LIMIT:
        a, b = D.family(dtype, n, seed)
        return a, b, D.family_sum(a, b, dtype)
    rng = np.random.default_rng([seed, DT_CODE[dtype]])
    a, b = X.finite(dtype, n, rng), X.finite(dtype, n, rng)
    return a, b, D.dot(a, b, dtype)


@pytest.mark.parametrize("dtype", DTS)
def test_sizes_and_both_sides_of_the_hbm_class(dtype):
    h = hbm_n(dtype)
    ragged = h + 5 * D.CHUNK + 1234                   # 2^25 words + 5 chunks: a chunk count that is no power of two
    for n in SMALL + [h - 1, h, ragged]:
        a, b, want = inputs(dtype, n, n)
        assert_same(dot(to_dev(a, dtype), to_dev(b, dtype)), want, f"{dtype} n={n}")


def placed(x, dtype, off):
    """A device copy of x starting `off` elements past a 256-byte boundary."""
    buf = torch.empty(x.size + off + 16, dtype=TORCH[dtype], device="cuda")
    view = buf[off:off + x.size]
    view.copy_(to_dev(x, dtype))
    return buf, view


@pytest.mark.parametrize("dtype", DTS)
def test_every_offset_and_relative_phase_gives_the_same_bits(dtype):
    """The same values at every element offset within 16 bytes for A and B together (the vector path with every
    head), and with B one to EPV - 1 elements further than A (the scalar path)."""
    epv = 16 // ES[dtype]
    for name, a, b in [("cancellation", *D.cancellation(dtype))] + [("random", *inputs(dtype, 2 * D.CHUNK + 3, 5)[:2])]:
        want = D.dot(a, b, dtype)
        for oa in range(epv):
            for ob in range(epv):
                _, da = placed(a, dtype, oa)
                _, db = placed(b, dtype, ob)
                assert_same(dot(da, db), want, f"{dtype} {name} offsets {oa},{ob}")


@pytest.mark.parametrize("dtype", DTS)
def test_a_equals_b_is_a_sum_of_squares(dtype):
    for n in (D.LANES + 1, 3 * D.CHUNK + 5):
        a, _, _ = inputs(dtype, n, 3)
        if dtype == "f64":
            a = D.family(dtype, n, 3)[0]
        x = to_dev(a, dtype)
        assert_same(dot(x, x), D.dot(a, a, dtype), f"{dtype} n={n}")
        _, v = placed(a, dtype, 1)
        assert_same(dot(v, v), D.dot(a, a, dtype), f"{dtype} n={n} offset 1")


@pytest.mark.parametrize("dtype", DTS)
def test_adversarial_special_and_subnormal_sets(dtype):
    """Cancellation, NaN, +-inf, inf * 0, inf - inf and subnormal operands, in the vector and the scalar path."""
    for name, a, b in D.adversarial(dtype):
        want = D.dot(a, b, dtype)
        da = to_dev(a, dtype)
        _, db1 = placed(b, dtype, 1)
        assert_same(dot(da, to_dev(b, dtype)), want, f"{dtype} {name} (vector)")
        assert_same(dot(da, db1), want, f"{dtype} {name} (scalar)")


@pytest.mark.parametrize("dtype", DTS)
def test_repeated_calls_two_streams_and_graph_replay(dtype):
    n = 3 * D.CHUNK + 5
    a, b = D.cancellation(dtype, n, seed=7)
    want = D.dot(a, b, dtype)
    da, db = to_dev(a, dtype), to_dev(b, dtype)
    for _ in range(3):
        assert_same(dot(da, db), want, "repeat")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = [va.dot(da, db, stream=s) for s in (s1, s2, s1, s2)]
    torch.cuda.synchronize()
    for r in outs:
        assert_same(float(r.item()), want, "two streams")
    out = torch.full((), 7.0, dtype=torch.float64, device="cuda")
    ws = torch.empty(capi.lib.b200va_dot_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            va.dot(da, db, out=out, workspace=ws)
    torch.cuda.synchronize()
    for _ in range(3):
        out.fill_(7.0)
        g.replay()
        torch.cuda.synchronize()
        assert_same(float(out.item()), want, "graph replay")


def test_dot_after_a_stream_op_and_an_add_on_one_stream():
    """b200va_stream and b200va_add_f32 write the operands and the dot follows on the same stream with no host
    synchronisation, at an L2-resident size and in the HBM class; ten rounds with a different scalar each."""
    st = torch.cuda.Stream()
    for n in ((1 << 20) + 5, (1 << 25) + 5):
        rng = np.random.default_rng(n)
        pa = X.finite("f32", 49_999, rng, 1.0)
        a = to_dev(np.resize(pa, n), "f32")
        c, d = torch.empty_like(a), torch.empty_like(a)
        scalars = [1.0 + k / 8 for k in range(10)]
        outs = torch.full((2, 10), 7.0, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        for k, s in enumerate(scalars):
            va.stream("scale", a, None, c, scalar=s, stream=st)          # c = s a
            va.dot(c, a, out=outs[0, k:k + 1], stream=st)
            va.add(c, a, d, stream=st)                                   # d = c + a
            va.dot(d, c, out=outs[1, k:k + 1], stream=st)
        st.synchronize()
        ha = np.resize(pa, n)
        for k, s in enumerate(scalars):
            hc = X.stream("scale", "f32", ha, None, s)
            hd = X.stream("add", "f32", hc, ha)
            assert_same(float(outs[0, k]), D.dot(hc, ha, "f32"), f"n={n} scale, round {k}")
            assert_same(float(outs[1, k]), D.dot(hd, hc, "f32"), f"n={n} add, round {k}")


@pytest.mark.parametrize("dtype", DTS)
def test_small_dot_reading_the_end_of_a_large_stream_op(dtype):
    """A large HBM-class stream op writes C, and a one-chunk dot right behind it reads the last elements of C,
    which the large launch's last CTAs write last: only the dot's wait keeps it from loading stale values.  Ten
    pairs with a different scalar each, so a stale load finds the previous pair's values."""
    n = hbm_n(dtype) + 5
    m = D.CHUNK - 3
    rng = np.random.default_rng(31)
    pa, pb = X.finite(dtype, 49_999, rng, 1.0), X.finite(dtype, m, rng, 1.0)
    a, b = to_dev(np.resize(pa, n), dtype), to_dev(pb, dtype)
    c = torch.empty_like(a)
    tail = np.resize(pa, n)[n - m:]
    st = torch.cuda.Stream()
    scalars = [1.0 + k / 8 for k in range(10)]
    outs = torch.full((10,), 7.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    for k, s in enumerate(scalars):
        va.stream("scale", a, None, c, scalar=s, stream=st)
        va.dot(c[n - m:], b, out=outs[k:k + 1], stream=st)
    st.synchronize()
    for k, s in enumerate(scalars):
        assert_same(float(outs[k]), D.dot(X.stream("scale", dtype, tail, None, s), pb, dtype), f"{dtype} pair {k}")


def test_back_to_back_dots_share_a_workspace_and_write_neighbouring_slots():
    n = 3 * D.CHUNK + 5
    need = capi.lib.b200va_dot_workspace_bytes(n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(12, dtype=torch.float64, device="cuda")
    out.view(torch.uint8).fill_(POISON)
    cases = []
    for k in range(10):
        dtype = DTS[k % 4]
        a, b = D.cancellation(dtype, n - 1000 * k, seed=k)
        cases.append((dtype, a, b, to_dev(a, dtype), to_dev(b, dtype)))
    torch.cuda.synchronize()
    for k, (dtype, _, _, da, db) in enumerate(cases):
        va.dot(da, db, out=out[k + 1:k + 2], workspace=ws)
    torch.cuda.synchronize()
    for k, (dtype, a, b, _, _) in enumerate(cases):
        assert_same(float(out[k + 1]), D.dot(a, b, dtype), f"slot {k + 1}")
    u8 = out.view(torch.uint8)
    assert bool((u8[:8] == POISON).all()) and bool((u8[88:] == POISON).all())


def test_f16_beyond_32_bit_offsets():
    """f16 at n = 2^32 + 4099 (two 8 GiB arrays) with exact-family inputs: element 2^31 is byte 2^32 and element
    2^32 needs a 64-bit index.  The inputs repeat a block of odd length, so a wrapped index reads another element
    and changes the exact sum.  65 537 chunk values take two pass-2 levels."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * 2 * n + (4 << 30):
        pytest.skip("needs ~20 GiB of free device memory")
    pa, pb = D.family("f16", 199_999, 43)
    a = to_dev(pa, "f16").repeat(-(-n // pa.size))[:n]
    b = to_dev(pb, "f16").repeat(-(-n // pb.size))[:n]
    want = D.family_sum(pa, pb, "f16", n)
    assert_same(dot(a, b), want, "n = 2^32 + 4099")
    m = (1 << 32) + 1                                   # one element past element 2^32
    assert_same(dot(a[:m], b[:m]), D.family_sum(pa, pb, "f16", m), "n = 2^32 + 1")


def test_argument_errors_and_nothing_written_outside_the_result_and_the_workspace():
    L = capi.lib
    n = 3 * D.CHUNK + 5
    need = L.b200va_dot_workspace_bytes(n)
    assert need == 8 * 4
    a = torch.ones(n + 64, dtype=torch.float32, device="cuda")
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    ws.fill_(POISON)
    out = torch.empty(5, dtype=torch.float64, device="cuda")
    out.view(torch.uint8).fill_(POISON)
    A, W, O = a.data_ptr(), ws.data_ptr(), out.data_ptr() + 16
    assert L.b200va_dot(9, A, A, n, O, W, need, None) == capi.ERR_VARIANT
    assert L.b200va_dot(-1, A, A, n, O, W, need, None) == capi.ERR_VARIANT
    assert L.b200va_dot(0, None, A, n, O, W, need, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A, None, n, O, W, need, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A, A, n, None, W, need, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A, A, n, O, None, need, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A, A, n, O, W, need - 1, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A, A, (1 << 40) + 1, O, W, 1 << 30, None) == capi.ERR_INVALID
    assert L.b200va_dot(0, A + 2, A, n, O, W, need, None) == capi.ERR_ALIGN
    assert L.b200va_dot(1, A + 4, A + 4, n // 2, O, W, need, None) == capi.ERR_ALIGN    # f64 needs 8 bytes
    assert L.b200va_dot(0, A, A + 2, n, O, W, need, None) == capi.ERR_ALIGN
    assert L.b200va_dot(0, A, A, n, O + 4, W, need, None) == capi.ERR_ALIGN
    assert L.b200va_dot(0, A, A, n, O, W + 4, need, None) == capi.ERR_ALIGN
    assert L.b200va_dot(0, A, A, n, A + 64, W, need, None) == capi.ERR_OVERLAP       # d_out inside A
    assert L.b200va_dot(0, A + 4 * 64, A, n, A, W, need, None) == capi.ERR_OVERLAP   # d_out inside B
    assert L.b200va_dot(0, A, A, n, O, A + 8, need, None) == capi.ERR_OVERLAP        # workspace inside A
    assert L.b200va_dot(0, A, A, n, W + 8, W, need, None) == capi.ERR_OVERLAP        # d_out inside the workspace
    assert L.b200va_dot(0, A, A, n, W + need, W, need + 8, None) == capi.OK           # right behind it is fine
    torch.cuda.synchronize()
    ws[need:].fill_(POISON)
    assert L.b200va_dot(0, None, None, 0, O, None, 0, None) == capi.OK                # n = 0: +0.0, no workspace
    torch.cuda.synchronize()
    assert bits(float(out[2])) == 0
    out.view(torch.uint8).fill_(POISON)
    assert L.b200va_dot(0, A, A, n, O, W, need + 256, None) == capi.OK                # A == B, larger workspace
    torch.cuda.synchronize()
    assert float(out[2]) == float(n)
    assert bool((ws[need:] == POISON).all()), "the workspace past the needed bytes was written"
    u8 = out.view(torch.uint8)
    assert bool((u8[:16] == POISON).all()) and bool((u8[24:] == POISON).all()), "a guard word around d_out was written"


def test_trace_shows_exactly_the_planned_kernels(tmp_path):
    """One call per type and class (n = 0, one chunk, several chunks, the HBM class, the scalar path, and f16 with
    more than 8192 chunks, whose pass 2 takes two levels) under the profiler: the kernels in the trace, with their
    grid and block, are exactly the planned ones, and there is no memset or other kernel."""
    plan, want = [], []

    def final(k):
        out = []
        while k > 8192:
            k = -(-k // 8192)
            out.append(("dot_final", k, 1024))
        return out + [("dot_final", 1, 1024)]

    bufs = {}
    for dtype in DTS:
        nmax = hbm_n(dtype) + 64
        bufs[dtype] = (torch.zeros(nmax, dtype=TORCH[dtype], device="cuda"), torch.zeros(nmax, dtype=TORCH[dtype], device="cuda"))
        threads, rows = FORM[dtype]
        for n, off in ((0, 0), (1000, 0), (3 * D.CHUNK + 5, 0), (hbm_n(dtype), 0), (hbm_n(dtype) - 1, 0), (5000, 1)):
            k = -(-n // D.CHUNK)
            plan.append((dtype, n, off))
            if n and off:
                want.append((f"dot_scalar<{DT_CODE[dtype]}>", k, 512))
            elif n:
                want.append((f"dot_vec<{DT_CODE[dtype]},{threads},{rows}>", k, threads))
            want += final(k)
    big_n = 8193 * D.CHUNK + 7
    big = torch.zeros(big_n, dtype=torch.float16, device="cuda")
    plan.append(("f16", big_n, -1))
    want += [("dot_vec<2,256,4>", 8194, 256)] + final(8194)
    out = torch.empty(1, dtype=torch.float64, device="cuda")
    ws = torch.empty(capi.lib.b200va_dot_workspace_bytes(big_n), dtype=torch.uint8, device="cuda")
    marker = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()

    def run_plan():
        for dtype, n, off in plan:
            if off < 0:
                va.dot(big, big, out=out, workspace=ws)
            else:
                a, b = bufs[dtype]
                va.dot(a[:n], b[off:off + n], out=out, workspace=ws)
        torch.cuda.synchronize()

    # Late in a long test session the trace can miss the first kernels after the profiler starts.  So the plan
    # runs twice, a fill kernel marks the start of the second pass, and the second pass is checked.
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_plan()
        marker.fill_(1.0)
        torch.cuda.synchronize()
        run_plan()
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    events = sorted((e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset")),
                    key=lambda e: e["ts"])
    m = max(i for i, e in enumerate(events) if "dot_" not in e["name"])   # the marker: nothing but dot kernels after it
    assert events[m].get("cat") == "kernel" and "ill" in events[m]["name"], events[m]["name"]
    got = [(_profiled_kernel_name(e["name"]), e["args"]["grid"][0], e["args"]["block"][0]) for e in events[m + 1:]]
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w in zip(got, want):
        assert g == w, (g, w)
