"""b200va_convert on the GPU, element by element against oracle/convert_exact.py (NaN matches NaN as a class, except
in the same-type copy, which keeps every bit).  Outputs are poisoned beforehand and guard elements on both sides
must keep the poison.

- Every ordered pair at ragged sizes around the group size G and 16-byte edges, at every element offset of A and
  of C within 16 bytes: the vector body with every head, and the mixed-phase scalar path.
- All 65536 patterns of each 16-bit source; for f32 and f64 sources, high parts of the pattern joined with the low
  parts that decide the rounding (0, 1, half - 1, half, half + 1, all ones).
- Both sides of the HBM class edge per pair and a ragged, misaligned n in it.  Large inputs repeat a random block
  of odd length, so the reference of the whole array is the block's reference repeated.
- Same-type copies keep NaN payloads; f16 <-> bf16 in place; every rejected argument writes nothing.
- A stream op writes A, the convert reads it and a stream op reads C, on one stream without a host sync; a
  captured and replayed graph; f16 -> bf16 at n = 2^32 + 4099.
- A profiler trace of the planned kernel, grid and block.
This module's name sorts after test_gpu_stream_dot.py: a module with profiler traces that runs before the parity
and stream modules makes their traces lose kernels (DESIGN.md section 3).
"""
import numpy as np
import pytest

from conftest import has_gpu
from oracle import convert_exact as V
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import (DT_CODE, ES, GUARD, POISON, TORCH, assert_guards, assert_matches, expected_cast_launch,
                             hbm_n, kernels_after_marker, poisoned, tiled, to_dev)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

PAIRS = V.PAIRS
PERIOD = 199_999


def group(src, dst):
    return 16 // min(ES[src], ES[dst])


def convert(a, dst, out, **kw):
    return va.convert(a, TORCH[dst], out, **kw)


def check(src, dst, a_host, a_dev, off_c=0, what=""):
    """Convert a_dev into a poisoned output at element offset off_c; compare with the reference of a_host."""
    n = a_host.size
    buf, out = poisoned(n, dst, off_c)
    convert(a_dev, dst, out)
    torch.cuda.synchronize()
    want = to_dev(V.convert(a_host, src, dst), dst)
    assert_matches(out, want, dst, what, nan_class=src != dst)
    assert_guards(buf, GUARD + off_c, n, what)


@pytest.mark.parametrize("src,dst", PAIRS)
def test_sizes_around_the_group_at_every_offset(src, dst):
    G = group(src, dst)
    sizes = sorted({0, 1, 2, 3, G - 1, G, G + 1, 2 * G - 1, 2 * G + 1, 15, 16, 17, 3 * G + 5, 4099, 70_001})
    rng = np.random.default_rng([DT_CODE[src], DT_CODE[dst]])
    host = V.random_bits(src, max(sizes) + 16, rng)
    for oa in range(16 // ES[src]):
        abuf, _ = poisoned(host.size, src)
        abuf[GUARD:GUARD + host.size].copy_(to_dev(host, src))
        for oc in range(16 // ES[dst]):
            for n in sizes:
                a = abuf[GUARD + oa:GUARD + oa + n]
                check(src, dst, host[oa:oa + n], a, oc, f"{src}->{dst} n={n} offsets A {oa} C {oc}")


@pytest.mark.parametrize("src", ["f16", "bf16"])
def test_every_16_bit_pattern(src):
    x = np.arange(1 << 16, dtype=np.uint16)
    a = to_dev(x, src)
    for dst in V.DTYPES:
        if dst != src:
            for off_c in (0, 1):                      # C one element off: mixed phase for the wider types
                check(src, dst, x, a, off_c, f"{src}->{dst} all patterns, C offset {off_c}")


def _highs(src, dst):
    """High parts (sign, exponent and the bits dst keeps in its normal range) of the rounding patterns: all of
    them where they number at most 2^22; for f64 -> f32 (2^35) every sign and exponent with 64 significand high
    parts: 0, 1, the top bit alone, the two largest and 59 random ones."""
    _, eb, mb = X.BITS[src]
    kept = X.FORMATS[dst][0] - 1
    if 1 + eb + kept <= 22:
        return np.arange(1 << (1 + eb + kept), dtype=np.uint64)
    rng = np.random.default_rng(5)
    mh = np.concatenate([np.array([0, 1, 1 << (kept - 1), (1 << kept) - 2, (1 << kept) - 1], np.uint64),
                         rng.integers(0, 1 << kept, 59, dtype=np.uint64)])
    se = np.arange(1 << (1 + eb), dtype=np.uint64)
    return ((se[:, None] << np.uint64(kept)) | mh[None, :]).ravel()


@pytest.mark.parametrize("src,dst", [("f32", "f16"), ("f32", "bf16"), ("f64", "f32"), ("f64", "f16"), ("f64", "bf16")])
def test_the_low_parts_that_decide_the_rounding(src, dst):
    highs = _highs(src, dst)
    for lo in range(0, highs.size, 1 << 19):
        x = V.rounding_patterns(src, dst, highs[lo:lo + (1 << 19)])
        check(src, dst, x, to_dev(x, src), 0, f"{src}->{dst} patterns from high part {int(highs[lo]):#x}")


@pytest.mark.parametrize("src,dst", PAIRS)
def test_both_sides_of_the_hbm_edge(src, dst):
    """n = h - 1 and h at aligned pointers, then h + 37 with A and C one element past a 16-byte boundary: the
    vector body with a head, in the HBM class (L2 prefetch ahead of the wait, no-allocate stores)."""
    h = hbm_n(max(ES[src], ES[dst]))
    big = h + 37
    block = V.random_bits(src, PERIOD, np.random.default_rng([7, DT_CODE[src], DT_CODE[dst]]))
    a, want = tiled(block, big + 1, src), tiled(V.convert(block, src, dst), big + 1, dst)
    for n, off in ((h - 1, 0), (h, 0), (big, 1)):
        buf, out = poisoned(n, dst, off)
        convert(a[off:off + n], dst, out)
        torch.cuda.synchronize()
        what = f"{src}->{dst} n={n} offset {off}"
        assert_matches(out, want[off:off + n], dst, what)
        assert_guards(buf, GUARD + off, n, what)
        del buf, out


@pytest.mark.parametrize("dtype", V.DTYPES)
def test_same_type_is_a_bit_copy_with_nan_payloads(dtype):
    x = np.tile(np.arange(1 << 16, dtype=np.uint16), 3) if dtype in ("f16", "bf16") else X.nan_payloads(dtype, 300_001, 5)
    n = x.size - 1
    a = to_dev(x, dtype)
    for name, src, off in (("vector", a[:n], 0), ("scalar", a[1:], 0), ("vector, head", a[1:], 1)):
        buf, out = poisoned(n, dtype, off)
        convert(src, dtype, out)
        torch.cuda.synchronize()
        assert_matches(out, src, dtype, f"{dtype} copy {name}", nan_class=False)
        assert_guards(buf, GUARD + off, n, name)


def test_f16_bf16_in_place():
    x = V.random_bits("f16", 100_003, np.random.default_rng(9))
    for src, dst in (("f16", "bf16"), ("bf16", "f16")):
        for off in (0, 1, 5):
            buf, v = poisoned(x.size, src, off)
            v.copy_(to_dev(x, src))
            convert(v, dst, v.view(TORCH[dst]))
            torch.cuda.synchronize()
            what = f"{src}->{dst} in place, offset {off}"
            assert_matches(v.view(TORCH[dst]), to_dev(V.convert(x, src, dst), dst), dst, what)
            assert_guards(buf, GUARD + off, x.size, what)


def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A, n = buf.data_ptr() + 4096, 1000
    F32, F64, F16, BF16 = 0, 1, 2, 3
    cases = [
        ((4, A, F32, A + 16384, n), capi.ERR_VARIANT), ((-1, A, F32, A + 16384, n), capi.ERR_VARIANT),
        ((F32, A, 9, A + 16384, n), capi.ERR_VARIANT), ((F16, A, -2, A + 16384, n), capi.ERR_VARIANT),
        ((F32, None, F16, A + 16384, n), capi.ERR_INVALID), ((F32, A, F16, None, n), capi.ERR_INVALID),
        ((F16, A, F16, None, n), capi.ERR_INVALID),
        ((F32, A, F16, A + 16384, (1 << 40) + 1), capi.ERR_INVALID),
        ((F32, A + 2, F16, A + 16384, n), capi.ERR_ALIGN), ((F32, A, F64, A + 16384 + 4, n), capi.ERR_ALIGN),
        ((F16, A + 1, BF16, A + 16384, n), capi.ERR_ALIGN), ((F64, A + 4, F64, A + 16384, n), capi.ERR_ALIGN),
        ((F32, A, F16, A, n), capi.ERR_OVERLAP),                       # exact aliasing of different sizes
        ((F16, A, F32, A, n), capi.ERR_OVERLAP),
        ((F32, A, F64, A + 4 * n - 8, n), capi.ERR_OVERLAP),           # C starts inside A
        ((F64, A + 8, F16, A, n), capi.ERR_OVERLAP),                   # C ends inside A
        ((F16, A + 2 * n, F32, A, n), capi.ERR_OVERLAP),               # C's wide tail meets A
        ((F16, A, BF16, A + 2, n), capi.ERR_OVERLAP),                  # equal sizes, partial overlap
        ((F32, A, F32, A + 4, n), capi.ERR_OVERLAP),
    ]
    for args, code in cases:
        assert L.b200va_convert(*args, None) == code, (args, code)
    assert L.b200va_convert(F32, None, F16, None, 0, None) == capi.OK  # n = 0: nothing to check or do
    assert L.b200va_convert(F16, A + 2 * n, F32, A, n // 2, None) == capi.OK      # right behind: no overlap
    torch.cuda.synchronize()
    u8 = buf.cpu().numpy()
    outside = np.ones(u8.size, bool)
    outside[4096:4096 + 2 * n] = False                                  # what the last call wrote
    assert (u8[outside] == POISON).all(), "a rejected call wrote to device memory"


def test_stream_op_convert_stream_op_on_one_stream():
    """Ten rounds on one stream with no host synchronisation: b = s a (b200va_stream), c = convert(b), d_k = c / 2
    (b200va_stream), at an L2-resident size and in the HBM class of the pair.  A different s per round, so a
    convert that read b before the scale finished, or a scale that read c before the convert finished, gives
    another round's values."""
    st = torch.cuda.Stream()
    for src, dst in (("f32", "bf16"), ("f64", "f16"), ("f16", "f32")):
        period = 49_999
        a0 = X.finite(src, period, np.random.default_rng(DT_CODE[src]), 1.0)
        scalars = [1.0 + k / 8 for k in range(10)]
        wants = []
        for s in scalars:
            c = V.convert(X.stream("scale", src, a0, None, s), src, dst)
            wants.append(X.stream("scale", dst, c, None, 0.5))
        for n in ((1 << 20) + 5, hbm_n(max(ES[src], ES[dst])) + 5):
            a = tiled(a0, n, src)
            b = torch.empty_like(a)
            c = torch.empty(n, dtype=TORCH[dst], device="cuda")
            ds = [torch.empty_like(c) for _ in scalars]
            torch.cuda.synchronize()
            for s, d in zip(scalars, ds):
                va.stream("scale", a, None, b, scalar=s, stream=st)
                convert(b, dst, c, stream=st)
                va.stream("scale", c, None, d, scalar=0.5, stream=st)
            st.synchronize()
            for k, (d, w) in enumerate(zip(ds, wants)):
                assert_matches(d, tiled(w, n, dst), dst, f"{src}->{dst} n={n} round {k}")
            del a, b, c, ds


def test_captured_graph_replays():
    cases = []
    for src, dst in (("f32", "f16"), ("f64", "bf16"), ("bf16", "f64")):
        x = V.random_bits(src, 100_003, np.random.default_rng(DT_CODE[dst]))
        buf, out = poisoned(x.size, dst, 1)
        cases.append((src, dst, x, to_dev(x, src), buf, out))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for src, dst, _, a, _, out in cases:
                convert(a, dst, out)
    torch.cuda.synchronize()
    for r in range(3):
        for _, _, _, _, buf, _ in cases:
            buf.view(torch.uint8).fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        for src, dst, x, _, buf, out in cases:
            what = f"{src}->{dst} replay {r}"
            assert_matches(out, to_dev(V.convert(x, src, dst), dst), dst, what)
            assert_guards(buf, GUARD + 1, x.size, what)


def test_f16_to_bf16_beyond_32_bit_offsets():
    """n = 2^32 + 4099 (two 8 GiB arrays and the 8 GiB reference): element 2^31 is byte 2^32 and element 2^32 needs
    a 64-bit index.  The input repeats a random block of odd length, so a wrapped index or byte offset converts
    another element."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * 2 * n + (4 << 30):
        pytest.skip("needs ~28 GiB of free device memory")
    block = V.random_bits("f16", PERIOD, np.random.default_rng(23))
    a = tiled(block, n, "f16")
    c = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    c.view(torch.uint8).fill_(POISON)
    convert(a, "bf16", c)
    want = tiled(V.convert(block, "f16", "bf16"), n, "bf16")
    for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - 8192):
        assert_matches(c[lo:lo + 8192], want[lo:lo + 8192], "bf16", f"window at {lo}")
    assert_matches(c, want, "bf16", "n = 2^32 + 4099")


def test_trace_shows_the_planned_kernels(tmp_path):
    """Per pair: n = 1000, the HBM class, n = 1001 in mixed phase, and an odd n with a head; per type the same-type
    call, which is the COPY stream kernel.  Under the profiler the kernels after the marker are exactly the
    planned ones with their grid and block."""
    nmax = max(hbm_n(max(ES[s], ES[d])) for s, d in PAIRS) + 64
    bufs = {dt: torch.zeros(nmax, dtype=TORCH[dt], device="cuda") for dt in V.DTYPES}
    outs = {dt: torch.zeros_like(bufs[dt]) for dt in V.DTYPES}
    plan, want = [], []
    for src, dst in PAIRS:
        for n, oa, oc in ((1000, 0, 0), (hbm_n(max(ES[src], ES[dst])), 0, 0), (1001, 0, 1), (4099, 1, 1)):
            a, c = bufs[src][oa:oa + n], outs[dst][oc:oc + n]
            plan.append((src, dst, a, c))
            want.append(expected_cast_launch(f"convert_vec<{DT_CODE[src]},{DT_CODE[dst]}>", ES[src], ES[dst], n,
                                             a.data_ptr(), c.data_ptr()))
    for dt in V.DTYPES:
        plan.append((dt, dt, bufs[dt][:1000], outs[dt][:1000]))
        want.append((f"stream_vec<{DT_CODE[dt]},0,1,0,0>", -(-1000 * ES[dt] // 16 // 128), 128))

    def run_plan():
        for _, dst, a, c in plan:
            convert(a, dst, c)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("convert_vec", "stream_vec"))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w, p in zip(got, want, plan):
        assert g == w, (p[:2], g, w)
