"""Row f4 on the GPU: b200va_stream (copy/scale/add/triad x f32/f64/f16/bf16) through the C ABI.

The first five tests compare with the C oracle (vadd_oracle.c) at ragged sizes, misaligned pointers and special
values.  The rest compare with the exact reference of oracle/stream_exact.py, which shares no arithmetic with the
kernels or the C oracle:
- every size class of launch_stream_typed and both sides of each class edge, up to the HBM class (m >= 2^25 words),
  and a profiler trace showing that every stream kernel of the library is launched with the table's geometry;
- COPY bit for bit (NaN payloads, signalling NaNs); the scalar rule (f32(s) for f32/f16/bf16, the double for f64);
- every aliasing of A, B and C; dependent chains of launches on one stream; 64-bit element and byte offsets.
Large inputs repeat a random block of PERIOD elements (odd, so it never lines up with a tile or a power of two): the
reference of an elementwise op is then the block's reference repeated, exact at every element for little host work.
Outputs are filled with a finite byte pattern beforehand, and guard elements on both sides must keep it.
"""
import re

import numpy as np
import pytest

import oracle
import sass
from conftest import has_gpu
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    import k8s_gpu_hpa_b200 as pkg
    from gpu_helpers import (DT_CODE, ES, GUARD, POISON, TORCH, assert_guards, assert_matches, expected_stream_launch,
                             kernels_after_marker, poisoned, tiled, to_dev)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

OPS = ["copy", "scale", "add", "triad"]
DTS = ["f32", "f64", "f16", "bf16"]
SIZES = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 1023, 4097, 50000, (1 << 20) + 3, 5_000_011]
OP_CODE = {"copy": 0, "scale": 1, "add": 2, "triad": 3}
BINARY = ("add", "triad")
PERIOD = 199_999            # <= X.FRACTION_LIMIT: f64 TRIAD is exact through Fraction over a whole period
SCALARS = [0.1, 1 / 3, 1 + 2.0 ** -24, 1 + 2.0 ** -24 + 2.0 ** -52, 3.5e38, 1e-45, 1e-50, -0.0,
           float("inf"), float("-inf"), float("nan")]


def host_inputs(dtype, n, seed):
    rng = np.random.default_rng(seed)
    if dtype == "f32":
        return (rng.standard_normal(n) * 4).astype(np.float32), (rng.standard_normal(n) * 4).astype(np.float32)
    if dtype == "f64":
        return rng.standard_normal(n) * 4, rng.standard_normal(n) * 4
    # half types: every bit pattern class incl. subnormals / inf / nan
    return (rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16),
            rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16))


def to_host(t, dtype):
    if dtype in ("f16", "bf16"):
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


def run(op, a, b, c, s=0.0, stream=None):
    va.stream(op, a, b if op in BINARY else None, c, scalar=s, stream=stream)


def n_from(dtype, m_words):
    """The smallest n whose footprint n * sizeof(T) / 4 (integer division, as the dispatcher computes it) is >= m."""
    return -(-m_words * 4 // ES[dtype])


def class_edges(dtype):
    """n on both sides of every class edge of launch_stream_typed: m >= 2^19, m >= 2^21, m > 2^23, m >= 2^25."""
    out = []
    for m in (1 << 19, 1 << 21, (1 << 23) + 1, 1 << 25):
        n = n_from(dtype, m)
        out += [n - 1, n]
    return out


def period_inputs(op, dtype, seed, period=PERIOD):
    """One PERIOD block of random inputs (half types: every bit pattern) and its exact reference."""
    if dtype in ("f16", "bf16"):
        a, b = host_inputs(dtype, period, seed)
    else:
        rng = np.random.default_rng(seed)
        a, b = X.finite(dtype, period, rng), X.finite(dtype, period, rng)
    s = 0.7001953125 if dtype != "f64" else 0.1
    return a, b, s, X.stream(op, dtype, a, b if op in BINARY else None, s)


# ------------------------------------------------------------------------------------ against the C oracle
@pytest.mark.parametrize("dtype", DTS)
@pytest.mark.parametrize("op", OPS)
def test_stream_ops_ragged_sizes(op, dtype):
    nmax = max(SIZES)
    ha, hb = host_inputs(dtype, nmax, 11)
    a, b = to_dev(ha, dtype), to_dev(hb, dtype)
    s = 0.7001953125 if op in ("scale", "triad") else 0.0
    want = oracle.stream(op, dtype, ha, hb if op in ("add", "triad") else None, s)
    for n in SIZES:
        buf, out = poisoned(n, dtype)
        va.stream(op, a[:n], b[:n] if op in ("add", "triad") else None, out, scalar=s)
        torch.cuda.synchronize()
        bad = oracle.first_mismatch_bits(to_host(out, dtype), want[:n], dtype)
        assert bad < 0, f"{op} {dtype} n={n}: first mismatch at {bad}"
        assert_guards(buf, GUARD, n, f"{op} {dtype} n={n}")


@pytest.mark.parametrize("dtype", DTS)
def test_stream_misaligned_and_aliased(dtype):
    n = 20_011
    ha, hb = host_inputs(dtype, n + 32, 12)
    a, b = to_dev(ha, dtype), to_dev(hb, dtype)
    for oa, ob, oc in [(0, 0, 0), (1, 1, 1), (3, 3, 3), (5, 5, 5), (1, 2, 3), (0, 1, 0), (7, 7, 0)]:
        buf, out = poisoned(n, dtype, oc)
        va.stream("triad", a[oa:oa + n], b[ob:ob + n], out, scalar=-1.5)
        torch.cuda.synchronize()
        want = oracle.stream("triad", dtype, ha[oa:oa + n].copy(), hb[ob:ob + n].copy(), -1.5)
        assert oracle.first_mismatch_bits(to_host(out, dtype), want, dtype) == -1, (oa, ob, oc)
        assert_guards(buf, GUARD + oc, n, str((oa, ob, oc)))
    x = to_dev(ha[:n], dtype)
    va.stream("triad", x, b[:n], x, scalar=2.0)                       # y = y + 2*x in place (axpy)
    assert oracle.first_mismatch_bits(to_host(x, dtype), oracle.stream("triad", dtype, ha[:n].copy(), hb[:n].copy(), 2.0), dtype) == -1


def test_stream_f32_add_is_bit_identical_to_the_hot_path():
    n = 3_000_017
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    c1, c2 = va.add(a, b), va.stream("add", a, b)
    assert bool((c1.view(torch.int32) == c2.view(torch.int32)).all())
    assert va.digest(c2) == oracle.ctr_vadd_digest(n)


def test_stream_special_values_f32_and_f64():
    g = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "special_values.npz"))
    ua, ub = np.tile(g["a_bits"], 9), np.tile(g["b_bits"], 9)
    a, b = to_dev(ua.view(np.float32), "f32"), to_dev(ub.view(np.float32), "f32")
    for op, s in (("add", 0.0), ("triad", 1.0), ("triad", -0.5), ("scale", 2.0 ** -10)):
        got = to_host(va.stream(op, a, b if op != "scale" else None, scalar=s), "f32")
        want = oracle.stream(op, "f32", ua.view(np.float32), ub.view(np.float32) if op != "scale" else None, s)
        assert oracle.first_mismatch_bits(got, want, "f32") == -1, op
    da = np.array([0.0, -0.0, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, np.inf, -np.inf, np.nan, 1.0, 1 + 2 ** -52])
    xa, xb = np.repeat(da, len(da)), np.tile(da, len(da))
    for op, s in (("add", 0.0), ("triad", 3.0), ("scale", 0.5)):
        got = to_host(va.stream(op, to_dev(xa, "f64"), to_dev(xb, "f64") if op != "scale" else None, scalar=s), "f64")
        assert oracle.first_mismatch_bits(got, oracle.stream(op, "f64", xa, xb if op != "scale" else None, s), "f64") == -1, op


def test_stream_argument_errors():
    a = torch.zeros(64, dtype=torch.float32, device="cuda")
    L = capi.lib
    assert L.b200va_stream(9, 0, a.data_ptr(), a.data_ptr(), a.data_ptr(), 64, 0.0, None) == capi.ERR_VARIANT
    assert L.b200va_stream(2, 7, a.data_ptr(), a.data_ptr(), a.data_ptr(), 64, 0.0, None) == capi.ERR_VARIANT
    assert L.b200va_stream(2, 0, a.data_ptr(), None, a.data_ptr(), 64, 0.0, None) == capi.ERR_INVALID     # add needs b
    assert L.b200va_stream(0, 0, a.data_ptr(), None, a.data_ptr(), 64, 0.0, None) == capi.OK             # copy does not
    assert L.b200va_stream(2, 1, a.data_ptr() + 4, a.data_ptr(), a.data_ptr(), 4, 0.0, None) == capi.ERR_ALIGN  # f64 needs 8 B
    assert L.b200va_stream(2, 0, a.data_ptr(), a.data_ptr(), a.data_ptr() + 8, 32, 0.0, None) == capi.ERR_OVERLAP


# ------------------------------------------------------------------------------------ against the exact reference
@pytest.mark.parametrize("dtype", DTS)
@pytest.mark.parametrize("op", OPS)
def test_every_size_class_and_both_sides_of_each_edge(op, dtype):
    """n on both sides of each class edge (m >= 2^19, >= 2^21, > 2^23, >= 2^25 words), then one n in the HBM class
    with a misaligned head (one element) and a ragged tail, each compared with the exact reference at every
    element.  The HBM class is the one with L1::no_allocate stores and the L2 prefetch ahead of the wait."""
    sizes = class_edges(dtype)
    big = sizes[-1] + 37
    pa, pb, s, pw = period_inputs(op, dtype, 101)
    a, b, want = tiled(pa, big + 1, dtype), tiled(pb, big + 1, dtype), tiled(pw, big + 1, dtype)
    for n, off in [(n, 0) for n in sizes] + [(big, 1)]:
        buf, out = poisoned(n, dtype, off)
        run(op, a[off:off + n], b[off:off + n], out, s)
        torch.cuda.synchronize()
        what = f"{op} {dtype} n={n} offset {off}"
        assert_matches(out, want[off:off + n], dtype, what, nan_class=op != "copy")
        assert_guards(buf, GUARD + off, n, what)


def library_stream_kernels(path):
    """stream_* kernels in a library, as the profiler names them: stream_vec<DT,OP,UNROLL,LD,ST>, stream_scalar<DT,OP>."""
    out = set()
    for fn in sass.functions(path):
        m = re.match(r"_ZN6b200va\d+(stream_vec|stream_scalar)I((?:Li-?\d+E)+)E", fn)
        if m:
            out.add(f"{m[1]}<{','.join(re.findall(r'Li(-?\d+)E', m[2]))}>")
    return out


def test_every_stream_kernel_of_the_library_is_launched_with_the_dispatchers_geometry(tmp_path):
    """One launch per dtype, op and size class, plus one through the mixed-misalignment scalar path, under the
    profiler: each kernel's template arguments, grid and block are the table's in launch_stream_typed, and the
    kernels launched are exactly the stream kernels in the SASS of libb200va.so.  prefetch_first is a runtime
    argument the trace cannot show; the dispatcher sets it under the m >= 2^25 condition that picks the ST_NA
    (store hint 1) kernels, so a launched ST_NA kernel ran the prefetch."""
    plan, want = [], []
    for dtype in DTS:
        sizes = [1000] + [n_from(dtype, m) for m in (1 << 19, 1 << 21, (1 << 23) + 1, 1 << 25)]
        for op in OPS:
            for n in sizes:
                plan.append((op, dtype, n, 0))
                want.append(expected_stream_launch(op, dtype, n))
            plan.append((op, dtype, 1001, 1))                 # A one element past C: the scalar fallback
            want.append((f"stream_scalar<{DT_CODE[dtype]},{OP_CODE[op]}>", -(-1001 // 256), 256))
    bufs = {}
    for dtype in DTS:
        nmax = max(n for _, d, n, _ in plan if d == dtype) + 1
        bufs[dtype] = [torch.zeros(nmax, dtype=TORCH[dtype], device="cuda") for _ in range(3)]

    def run_plan():
        for op, dtype, n, off in plan:
            a, b, c = bufs[dtype]
            run(op, a[off:off + n], b[off:off + n], c[:n], 0.5)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("stream_",))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w, p in zip(got, want, plan):
        assert g == w, (p, g, w)
    launched = {g[0] for g in got}
    shipped = library_stream_kernels(capi.LIB_PATH)
    assert len(shipped) == 64 and launched == shipped, (sorted(shipped - launched), sorted(launched - shipped))


@pytest.mark.parametrize("dtype", DTS)
def test_copy_is_bit_exact_nan_payloads_included(dtype):
    """COPY keeps every bit: all 65536 half patterns, random 32/64-bit patterns a third of which are NaNs with
    random payloads (quiet and signalling), in the vector path and in the scalar path."""
    if dtype in ("f16", "bf16"):
        x = np.tile(np.arange(1 << 16, dtype=np.uint16), 3)
    else:
        x = X.nan_payloads(dtype, 300_001, 5)
    n = x.size - 1
    a = to_dev(x, dtype)
    for name, src, off in (("vector", a[:n], 0), ("scalar", a[1:], 0), ("vector, head", a[1:], 1)):
        buf, out = poisoned(n, dtype, off)
        run("copy", src, None, out)
        torch.cuda.synchronize()
        assert_matches(out, src, dtype, f"copy {dtype} {name}", nan_class=False)
        assert_guards(buf, GUARD + off, n, name)


@pytest.mark.parametrize("dtype", DTS)
@pytest.mark.parametrize("op", ["scale", "triad"])
def test_scalar_is_rounded_to_f32_except_for_f64(op, dtype):
    """f32/f16/bf16 use f32(s), f64 the double as given: scalars that are no floats, a double exactly between two
    floats and the double just above it, one that overflows f32, f32-subnormal and f32-zero ones, -0, +-inf, NaN.
    Random operands plus the edge set (zeros, subnormals, the largest values, inf, NaN)."""
    rng = np.random.default_rng(7)
    n = 20_011
    a = np.concatenate([X.finite(dtype, n, rng), X.edge_values(dtype, 4096, 8)])
    b = np.concatenate([X.finite(dtype, n, rng), X.edge_values(dtype, 4096, 9)])
    da, db = to_dev(a, dtype), to_dev(b, dtype)
    for s in SCALARS:
        buf, out = poisoned(a.size, dtype)
        run(op, da, db, out, s)
        torch.cuda.synchronize()
        want = X.stream(op, dtype, a, b if op in BINARY else None, s)
        assert_matches(out, to_dev(want, dtype), dtype, f"{op} {dtype} s={s!r}")
        assert_guards(buf, GUARD, a.size, repr(s))


@pytest.mark.parametrize("dtype", DTS)
@pytest.mark.parametrize("op", OPS)
def test_adversarial_inputs(op, dtype):
    """The adversarial sets of oracle/stream_exact.py: fma cancellation, f16/bf16 TRIAD results on a storage-type
    midpoint (where rounding twice differs from rounding once), the overflow threshold, subnormal results, signed
    zeros, NaN payloads for COPY; in the vector path and in the scalar path."""
    for name, s, a, b in X.adversarial(op, dtype):
        da, db = to_dev(a, dtype), to_dev(b, dtype)
        want = to_dev(X.stream(op, dtype, a, b if op in BINARY else None, s), dtype)
        for path, off in (("vector", 0), ("scalar", 1)):      # scalar: C one element off A and B
            buf, out = poisoned(a.size, dtype, off)
            run(op, da, db, out, s)
            torch.cuda.synchronize()
            assert_matches(out, want, dtype, f"{op} {dtype} {name} ({path})", nan_class=op != "copy")
            assert_guards(buf, GUARD + off, a.size, name)


# (name, then (buffer, offset in elements) of A, B and C).  Buffers p and q hold the inputs, r is a fresh output.
ALIASES = [("vector C==A", ("p", 0), ("q", 0), ("p", 0)), ("vector C==B", ("p", 0), ("q", 0), ("q", 0)),
           ("vector A==B", ("p", 0), ("p", 0), ("r", 0)), ("vector A==B==C", ("p", 0), ("p", 0), ("p", 0)),
           ("scalar C==A", ("p", 0), ("q", 1), ("p", 0)), ("scalar C==B", ("p", 1), ("q", 0), ("q", 0)),
           ("scalar A==B", ("p", 0), ("p", 0), ("r", 1))]


@pytest.mark.parametrize("dtype", DTS)
@pytest.mark.parametrize("op", OPS)
def test_aliased_operands(op, dtype):
    """C == A, C == B, A == B and A == B == C in the vector path; in the scalar path C == A and C == B with the
    other input one element off, and A == B with C one element off.  Inputs that are not C stay unchanged."""
    n = 100_003
    rng = np.random.default_rng(13)
    ha, hb = X.finite(dtype, n, rng), X.finite(dtype, n, rng)
    s = -1.5 if dtype != "f64" else 0.1
    for name, A, B, C in ALIASES:
        if name in ("scalar C==A", "scalar C==B") and op not in BINARY:
            continue                                           # B is not read: these stay in the vector path
        bufs, views = {}, {}
        for key, host in (("p", ha), ("q", hb), ("r", None)):
            off = max(o for k, o in (A, B, C) if k == key) if key in (A[0], B[0], C[0]) else 0
            bufs[key], v = poisoned(n, dtype, off)
            if host is not None:
                v.copy_(to_dev(host, dtype))
        view = lambda kv: bufs[kv[0]][GUARD + kv[1]:GUARD + kv[1] + n]
        host_of = {"p": ha, "q": hb}
        wa, wb = host_of[A[0]], host_of[B[0]]
        run(op, view(A), view(B), view(C), s)
        torch.cuda.synchronize()
        what = f"{op} {dtype} {name}"
        assert_matches(view(C), to_dev(X.stream(op, dtype, wa, wb if op in BINARY else None, s), dtype), dtype, what)
        assert_guards(bufs[C[0]], GUARD + C[1], n, what)
        for kv in {A, B} - {C}:
            assert_matches(view(kv), to_dev(host_of[kv[0]], dtype), dtype, f"{what}: input {kv} changed", nan_class=False)


STREAM_S = 2 ** 0.5 - 1     # s (2 + s) = 1: a STREAM iteration maps a to s (2 + s) a, so values neither grow nor fade


def stream_iterations(a, b, c, s, iters, run_op):
    """The STREAM loop: c = a; b = s c; c = a + b; a = b + s c."""
    for _ in range(iters):
        c = run_op("copy", a, None, c, 0.0)
        b = run_op("scale", c, None, b, s)
        c = run_op("add", a, b, c, 0.0)
        a = run_op("triad", b, c, a, s)
    return a, b, c


@pytest.mark.parametrize("dtype", DTS)
def test_dependent_stream_loop_on_one_stream(dtype):
    """Ten iterations of the STREAM loop on one non-default stream with no host synchronisation inside: every launch
    consumes the previous one's output across the programmatic (PDL) edge.  Once at an L2-resident size and once in
    the HBM class, where the L2 prefetch runs ahead of the wait.  Checked against the exact reference iterated on
    the host; most f16 elements stay finite over the ten iterations."""
    period = 49_999
    rng = np.random.default_rng(17)
    a0, b0, c0 = (X.finite(dtype, period, rng, 1.0) for _ in range(3))

    def host_op(op, x, y, out, s):
        return X.stream(op, dtype, x, y, s)

    wa, wb, wc = stream_iterations(a0, b0, c0, STREAM_S, 10, host_op)
    if dtype == "f16":
        assert np.isfinite(X.widen(wa, dtype)).mean() > 0.99
    st = torch.cuda.Stream()
    for n in (n_from(dtype, 1 << 20) + 5, n_from(dtype, 1 << 25) + 5):
        a, b, c = (tiled(x, n, dtype) for x in (a0, b0, c0))
        torch.cuda.synchronize()

        def dev_op(op, x, y, out, s):
            run(op, x, y, out, s, stream=st)
            return out

        with torch.cuda.stream(st):
            stream_iterations(a, b, c, STREAM_S, 10, dev_op)
        st.synchronize()
        for name, got, want in (("a", a, wa), ("b", b, wb), ("c", c, wc)):
            assert_matches(got, tiled(want, n, dtype), dtype, f"{dtype} n={n} {name}")


def test_f32_add_then_stream_ops_on_one_stream():
    """The f32 add hot path (AUTO) writes C and stream ops read it, ten times over on one stream without a host
    synchronisation: c = a + b (b200va_add_f32); b = s c; a = b + s c."""
    period = 49_999
    rng = np.random.default_rng(19)
    a0, b0 = X.finite("f32", period, rng), X.finite("f32", period, rng)
    wa, wb = a0, b0
    for _ in range(10):
        wc = X.stream("add", "f32", wa, wb)
        wb = X.stream("scale", "f32", wc, None, STREAM_S)
        wa = X.stream("triad", "f32", wb, wc, STREAM_S)
    st = torch.cuda.Stream()
    for n in ((1 << 20) + 5, (1 << 25) + 5):
        a, b = tiled(a0, n, "f32"), tiled(b0, n, "f32")
        c = torch.empty_like(a)
        torch.cuda.synchronize()
        for _ in range(10):
            va.add(a, b, c, stream=st)
            run("scale", c, None, b, STREAM_S, stream=st)
            run("triad", b, c, a, STREAM_S, stream=st)
        st.synchronize()
        assert_matches(a, tiled(wa, n, "f32"), "f32", f"n={n} a")
        assert_matches(b, tiled(wb, n, "f32"), "f32", f"n={n} b")
        assert_matches(c, tiled(wc, n, "f32"), "f32", f"n={n} c")


def test_f16_beyond_32_bit_offsets():
    """f16 at n = 2^32 + 4099 (three 8 GiB arrays): element 2^31 is byte 2^32, element 2^32 needs a 64-bit index.
    The inputs repeat a block of odd length, so an index or byte offset that wrapped at 2^31 or 2^32 would read a
    different element.  All four ops are compared with the exact reference over the whole array."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()                           # earlier tests' blocks held by the caching allocator
    free, _ = torch.cuda.mem_get_info()
    if free < 4 * 2 * n + (4 << 30):
        pytest.skip("needs ~38 GiB of free device memory")
    pa, pb = host_inputs("f16", PERIOD, 23)
    a, b = tiled(pa, n, "f16"), tiled(pb, n, "f16")
    c = torch.empty_like(a)
    for op in OPS:
        c.view(torch.uint8).fill_(POISON)
        run(op, a, b, c, 0.7001953125)
        want = tiled(X.stream(op, "f16", pa, pb if op in BINARY else None, 0.7001953125), n, "f16")
        for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - 8192):      # windows across byte 2^32, element 2^32, the tail
            assert_matches(c[lo:lo + 8192], want[lo:lo + 8192], "f16", f"{op} window at {lo}", nan_class=op != "copy")
        assert_matches(c, want, "f16", op, nan_class=op != "copy")
        del want
        if op == "add":       # widen, one f32 RNE add, RNE narrow: torch's own statement of the contract
            for lo in range(0, n, 1 << 28):
                hi = min(n, lo + (1 << 28))
                ref = (a[lo:hi].float() + b[lo:hi].float()).half()
                assert_matches(c[lo:hi], ref, "f16", f"add vs torch at {lo}")


@pytest.mark.parametrize("dtype", DTS)
def test_small_launch_reading_the_end_of_a_large_one(dtype):
    """A large launch in the HBM class writes C, and a small launch right behind it on the same stream reads the last
    elements of C, which the large launch's last CTAs write last.  The small launch can start while those CTAs still
    run (programmatic dependent launch), so only its wait on the large one keeps it from loading stale values.
    Ten such pairs with a different scalar each, so a stale load finds the previous pair's values."""
    n = n_from(dtype, 1 << 25) + 5
    m = n - (n - 3 * 4096) // 8 * 8                    # C[n - m:] stays 16-byte aligned: the vector kernel reads it
    rng = np.random.default_rng(29)
    pa, pb = X.finite(dtype, PERIOD, rng, 1.0), X.finite(dtype, m, rng, 1.0)
    a, b = tiled(pa, n, dtype), to_dev(pb, dtype)
    buf, c = poisoned(n, dtype)
    outs = [poisoned(m, dtype) for _ in range(10)]
    tail = np.resize(pa, n)[n - m:]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    scalars = [1.0 + k / 8 for k in range(10)]
    for s, (_, d) in zip(scalars, outs):
        run("scale", a, None, c, s, stream=st)
        run("add", c[n - m:], b, d, stream=st)      # expected_stream_launch: a stream_vec kernel, launched with PDL
    st.synchronize()
    for k, (s, (obuf, d)) in enumerate(zip(scalars, outs)):
        want = X.stream("add", dtype, X.stream("scale", dtype, tail, None, s), pb)
        assert_matches(d, to_dev(want, dtype), dtype, f"{dtype} pair {k}")
        assert_guards(obuf, GUARD, m, f"pair {k}")
