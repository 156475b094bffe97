"""The reductions on the GPU -- the amax of b200va_quantize_fp8 and b200va_quantize_fp8_sr_f32, the MXFP8 block scales,
b200va_dot and b200va_verify_f32 / b200va_digest_f32 -- with planted extremes and poisoned neighbours.

An element-wise kernel that drops or misreads an element shows up as a wrong output element.  A reduction shows it
only if that element would have changed the answer, so every test here makes it change the answer:
- Every operand sits inside a buffer with a 64 KiB margin on both sides (more than a tile of the widest vector unit),
  filled so that reading it changes the result: NaN for amax and dot, the source type's largest finite value for
  MXFP8 quantize (NaN and +-inf are excluded from a block maximum), 0xFF (NaN) scale bytes around the scales for
  MXFP8 dequantize, C elements that do not equal A + B for verify, nonzero words for digest.  Each result equals
  the oracle of [0, n) alone, bit for bit.
- amax: small background values and one larger magnitude planted in turn at every position of the launch plan where
  a path begins or ends (restated here from plan_cast in b200va_typed.cu): the head, group 0, the last thread of the
  first unroll slot, the second unroll slot of the HBM class, the last full tile, the partial tile, the tail, and in
  mixed phase the first element of every edge-loop CTA.  Each case asserts it reaches the path it is meant for.
- MXFP8: block b holds its maximum at position (7 b) mod len_b, so one launch covers every position in a block; the
  short final block has 1, 2, block / 2 and block - 1 elements.
- dot: NaN margins at every head and in the scalar path, a NaN-filled workspace larger than the call needs, and the
  pass-2 level edges: 8192 chunk values (one level), 8193 (two) and 16385 (two, with a partial second block).
- verify: single mismatches at every position where the vector form changes what it does, and sets of them.
- The vector_add wrapper checks the length and device of every operand before it calls the library.
"""
import math

import numpy as np
import pytest

import oracle
from conftest import has_gpu
from oracle import dot_exact as D
from oracle import fp8_exact as F
from oracle import mxfp8_exact as MX
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import INT, POISON, TORCH, assert_matches, hbm_n, tiled, to_dev
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = ["f32", "f64", "f16", "bf16"]
FMTS = ["e4m3", "e5m2"]
ES = {"f32": 4, "f64": 8, "f16": 2, "bf16": 2, "e4m3": 1, "e5m2": 1, "u8": 1}
MARGIN = 1 << 16                    # bytes on each side of every operand
PERIOD = 49_999                     # background values repeat with this odd period

NAN = {"f32": 0x7FC00000, "f64": 0x7FF8000000000000, "f16": 0x7E00, "bf16": 0x7FC0}
INF = {"f32": 0x7F800000, "f64": 0x7FF0000000000000, "f16": 0x7C00, "bf16": 0x7F80}
MAX_FINITE = {"f32": 0x7F7FFFFF, "f64": 0x7FEFFFFFFFFFFFFF, "f16": 0x7BFF, "bf16": 0x7F7F}
SIGN = {"f32": 1 << 31, "f64": 1 << 63, "f16": 1 << 15, "bf16": 1 << 15}
PLANT = 3.25                        # the planted magnitude: exact in every type, far above the background


# ------------------------------------------------------------------------------------------- helpers
def signed(bits: int, fmt: str) -> int:
    """An unsigned bit pattern as the value of fmt's integer view (signed for 2, 4 and 8 bytes)."""
    w = 8 * ES[fmt]
    return bits - (1 << w) if w > 8 and bits >> (w - 1) else bits


def storage_bits(x: float, fmt: str) -> int:
    """The bit pattern of the value x rounded to fmt."""
    if fmt in ("f32", "f64"):
        return int(np.array([x], X.STORAGE[fmt]).view({"f32": np.uint32, "f64": np.uint64}[fmt])[0])
    return int(X.narrow(np.array([x], np.float32), fmt)[0])


def poison_bits(fmt: str) -> int:
    """The element pattern of a buffer whose bytes are all POISON."""
    return int.from_bytes(bytes([POISON]) * ES[fmt], "little")


def f64_bits(x: float) -> int:
    return int(np.float64(x).view(np.uint64))


def margined(n, fmt, off, fill):
    """(buffer, view): the view is n elements of fmt starting `off` elements past a MARGIN-byte margin, and every
    element of the buffer outside it (both margins and the off elements) holds the bit pattern fill."""
    m = MARGIN // ES[fmt]
    buf = torch.empty(m + off + n + m, dtype=TORCH[fmt], device="cuda")
    buf.view(INT[fmt]).fill_(signed(fill, fmt))
    return buf, buf[m + off:m + off + n]


def assert_margins(buf, view, fill, what=""):
    """Every element of buf outside view still holds the bit pattern fill."""
    es = buf.element_size()
    fmt = {1: "u8", 2: "f16", 4: "f32", 8: "f64"}[es]
    start = (view.data_ptr() - buf.data_ptr()) // es
    ints = buf.view(INT[fmt])
    for part in (ints[:start], ints[start + view.numel():]):
        assert bool((part == signed(fill, fmt)).all()), f"{what}: an element outside the operand was written"


def put(view, host, fmt):
    """Copy host storage (values, or patterns for f16 / bf16 / FP8) of view's length into view."""
    view.view(INT[fmt]).copy_(to_dev(host, fmt).view(INT[fmt]))


def background(src, scale=0.25, seed=0):
    """PERIOD small finite values of src (|x| < 2, normal with sigma `scale`)."""
    return X.finite(src, PERIOD, np.random.default_rng([seed, DTYPES.index(src)]), scale)


def same_f64(got: float, want: float) -> bool:
    return (math.isnan(got) and math.isnan(want)) or f64_bits(got) == f64_bits(want)


# ------------------------------------------------------------------------------------------- the cast launch plan
class CastPlan:
    """plan_cast (b200va_typed.cu) for n elements of esa bytes at address pa cast to esc bytes at pc: the head, the
    groups of the vector body and the launch geometry."""

    def __init__(self, esa, esc, n, pa, pc):
        self.G = 16 // min(esa, esc)
        head, h = n, ((16 - pa % 16) % 16) // esa
        while h < self.G:
            if (pc + h * esc) % 16 == 0:
                head = h
                break
            h += 16 // esa
        self.n, self.head = n, min(head, n)
        self.ngroups = (n - self.head) // self.G
        hbm = n >= hbm_n(max(esa, esc))
        self.threads, self.unroll = (512, 2) if hbm else (256, 1)
        self.tile = self.threads * self.unroll
        edges = n - self.ngroups * self.G
        self.grid = max(1, -(-self.ngroups // self.tile), -(-edges // self.threads))

    @property
    def mixed(self):
        return self.head == self.n

    def positions(self):
        """The elements where a path of the kernel begins or ends, in increasing order."""
        n, G, T = self.n, self.G, self.threads
        if n <= 2 * G:
            return list(range(n))
        if self.mixed:
            # cast_edges takes element i in thread i of the grid: the first element of every CTA, and of its last warp
            pos = {0, n - 1} | {c * T for c in range(self.grid)} | {c * T + T - 32 for c in range(self.grid)}
            return sorted(p for p in pos if p < n)
        first = lambda g: self.head + G * g                                  # noqa: E731
        pos = set(range(self.head)) | set(range(first(self.ngroups), n))     # the head and the tail
        if self.ngroups:
            pos |= {first(0), first(0) + G - 1}
            full = self.ngroups // self.tile
            if self.ngroups > T - 1:
                pos.add(first(T - 1))                                        # the last thread, unroll slot 0
            if self.unroll == 2 and self.ngroups > T:
                pos.add(first(T))                                            # thread 0, unroll slot 1
            if full:
                pos.add(first(full * self.tile) - 1)                         # the last group of the last full tile
            if self.ngroups % self.tile:
                pos |= {first(full * self.tile), first(self.ngroups) - 1}    # the first and last group of the partial tile
        return sorted(pos)


# Element offsets of A and C from a 16-byte boundary: with both one element in, the head is 15 for every type
# (A and C meet a boundary together 15 elements on); A aligned and C one byte in never meet one (mixed phase).
LAYOUTS = {"aligned": (0, 0), "head": (1, 1), "mixed": (0, 1)}


def amax_cases(es):
    """(n, layout, what the plan must show) for a source of es bytes into FP8."""
    t = 256                                                  # groups per tile below the HBM class
    cases = [(n, lay, ("head",) if lay == "head" and n > 15 else ()) for n in (1, 15, 16, 17) for lay in LAYOUTS]
    cases += [(16 * (t + 1), "aligned", ("partial",)), (16 * (t - 1), "aligned", ("partial",)),
              (15 + 16 * (t + 1) + 3, "head", ("head", "partial")), (15 + 16 * (t - 1) + 3, "head", ("head", "partial")),
              (16 * (3 * t + 7) + 9, "aligned", ("partial",)), (15 + 16 * (3 * t + 7) + 9, "head", ("head", "partial")),
              (3 * 256 + 77, "mixed", ("mixed",)),
              (hbm_n(es), "head", ("head", "unroll2", "partial")), (hbm_n(es) + 37, "head", ("head", "unroll2", "partial"))]
    return cases


def assert_reaches(p: CastPlan, expect, what):
    if "head" in expect:
        assert 0 < p.head < p.n, f"{what}: no head ({p.head})"
    if "mixed" in expect:
        assert p.mixed and p.grid > 1, f"{what}: not mixed phase over several CTAs"
    if "unroll2" in expect:
        assert p.unroll == 2 and p.ngroups > p.threads, f"{what}: no second unroll slot"
    if "partial" in expect:
        assert p.ngroups % p.tile, f"{what}: no partial tile"


def run_planted_amax(src, fmt, launch, what):
    """Every amax case of src into fmt: per case one launch per planted position (and an unplanted one, a NaN and a
    +inf), each into its own f64 slot, with one synchronise per case."""
    bg = background(src)
    bg_amax = F.amax(bg, src)
    mag, sgn = storage_bits(PLANT, src), SIGN[src]
    for n, layout, expect in amax_cases(ES[src]):
        oa, oc = LAYOUTS[layout]
        abuf, a = margined(n, src, oa, NAN[src])
        a.view(INT[src]).copy_(tiled(bg, n, src).view(INT[src]))
        cbuf, c = margined(n, fmt, oc, POISON)
        p = CastPlan(ES[src], 1, n, a.data_ptr(), c.data_ptr())
        case = f"{what} n={n} {layout} (head {p.head}, {p.ngroups} groups, grid {p.grid} x {p.threads}, unroll {p.unroll})"
        assert_reaches(p, expect, case)
        pos = p.positions()
        plants = [(None, None, bg_amax if n >= PERIOD else F.amax(bg[:n], src))]
        plants += [(q, mag | (sgn if k % 2 else 0), PLANT) for k, q in enumerate(pos)]
        plants += [(pos[0], NAN[src], math.nan), (pos[-1], INF[src], math.inf)]
        slots = torch.zeros(len(plants), dtype=torch.float64, device="cuda")
        ai = a.view(INT[src])
        for k, (q, bits, _) in enumerate(plants):
            if q is None:
                launch(a, c, slots[k:k + 1])
                continue
            keep = ai[q:q + 1].clone()
            ai[q:q + 1].fill_(signed(bits, src))
            launch(a, c, slots[k:k + 1])
            ai[q:q + 1].copy_(keep)
        torch.cuda.synchronize()
        got = slots.cpu().numpy()
        bad = [f"planted {bits:#x} at {q}: amax {g!r}, want {w!r}" for (q, bits, w), g in zip(plants, got.tolist())
               if not same_f64(g, w)]
        assert not bad, f"{case}: {len(bad)} of {len(plants)} wrong:\n" + "\n".join(bad[:10])
        assert_margins(cbuf, c, POISON, case)
        del abuf, cbuf, a, c, slots


# ------------------------------------------------------------------------------------------- amax
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_amax_finds_a_maximum_planted_at_every_path_edge(src, fmt):
    run_planted_amax(src, fmt, lambda a, c, m: va.quantize_fp8(a, TORCH[fmt], scale_exp=0, amax=m, out=c),
                     f"quantize {src}->{fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_sr_quantize_amax_finds_a_maximum_planted_at_every_path_edge(fmt):
    run_planted_amax("f32", fmt, lambda a, c, m: va.quantize_fp8_sr(a, TORCH[fmt], seed=5, amax=m, out=c),
                     f"SR quantize f32->{fmt}")


@pytest.mark.parametrize("src", DTYPES + ["sr"])
def test_amax_of_adjacent_shards_equals_the_amax_of_the_whole(src):
    """Three calls over adjacent slices (a ragged first slice, so the others start off a 16-byte boundary) max-
    accumulate into one amax: the same bits as one call over the whole array, with and without a planted maximum."""
    t = "f32" if src == "sr" else src
    n = 15 + 16 * (3 * 256 + 7) + 9
    bounds = [0, 1001, 1001 + 2 * 4096 + 5, n]
    assert bounds == sorted(set(bounds))
    abuf, a = margined(n, t, 0, NAN[t])
    put(a, background(t, seed=3)[:n], t)
    c = torch.empty(n, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)

    def quant(lo, hi, m):
        if src == "sr":
            va.quantize_fp8_sr(a[lo:hi], torch.float8_e4m3fn, seed=9, offset=lo, amax=m, out=c[lo:hi])
        else:
            va.quantize_fp8(a[lo:hi], torch.float8_e4m3fn, amax=m, out=c[lo:hi])

    for plant in (None, bounds[1] + 7, bounds[2] - 1, bounds[2]):
        if plant is not None:
            a.view(INT[t])[plant:plant + 1].fill_(signed(storage_bits(PLANT, t) | SIGN[t], t))
        m = torch.zeros(2, dtype=torch.float64, device="cuda")
        quant(0, n, m[0:1])
        for lo, hi in zip(bounds, bounds[1:]):
            quant(lo, hi, m[1:2])
        torch.cuda.synchronize()
        whole, shards = m.tolist()
        assert f64_bits(whole) == f64_bits(shards), (src, plant, whole, shards)
        if plant is not None:
            assert whole == PLANT, (src, plant, whole)
            put(a, background(t, seed=3)[:n], t)
    del abuf


# ------------------------------------------------------------------------------------------- MXFP8
def mx_top(b):
    """The magnitude block b's maximum has: 1 + (b mod 8) / 8 times 2^(1 + (b / 8) mod 8), so the scales vary and the
    significands cross 1.75 (where the two scale rules differ).  It repeats every 128 blocks."""
    return (1 + (b % 8) / 8) * 2.0 ** (1 + (b // 8) % 8)


def mx_blocks(src, first, count, length, seed):
    """`count` blocks of `length` elements of src, global block indices first..: background below 1 in magnitude, and
    block b's maximum, of sign (-1)^b, at position (7 b) mod length."""
    x = np.random.default_rng([seed, first, length]).uniform(-0.99, 0.99, count * length)
    for k in range(count):
        b = first + k
        x[k * length + (7 * b) % length] = mx_top(b) * (-1) ** b
    return X.narrow(x.astype(np.float32), src) if src in ("f16", "bf16") else x.astype(X.STORAGE[src])


def run_mx(src, fmt, block, rule, off, n, what):
    """One quantize and one dequantize of n elements at element offset off, against the oracle bit for bit: whole
    blocks repeat a 128-block period (the oracle of the period, tiled), the short final block is its own."""
    K, r = divmod(n, block)
    period = mx_blocks(src, 0, 128, block, 1)
    last = mx_blocks(src, K, 1, r, 2) if r else None
    qp, sp = MX.quantize(period, src, fmt, block, rule)
    dp = MX.dequantize(qp, sp, fmt, src, block)
    abuf, a = margined(n, src, off, MAX_FINITE[src])
    a.view(INT[src])[:K * block].copy_(tiled(period, K * block, src).view(INT[src]))
    if r:
        put(a[K * block:], last, src)
    nsc = MX.scale_count(n, block)
    cbuf, c = margined(n, fmt, off, POISON)
    sbuf, s = margined(nsc, "u8", 0, POISON)
    if off == 0:
        assert a.data_ptr() % 16 == 0 and c.data_ptr() % 16 == 0, what
    va.quantize_mxfp8(a, TORCH[fmt], block=block, scale_rule=rule, out=c, scales=s)
    want_q = tiled(qp, K * block, fmt).view(torch.uint8)
    want_s = tiled(sp, K, "u8")
    if r:
        ql, sl = MX.quantize(last, src, fmt, block, rule)
        want_q = torch.cat([want_q, to_dev(ql, "u8")])
        want_s = torch.cat([want_s, to_dev(sl, "u8")])
    torch.cuda.synchronize()
    assert_matches(c.view(torch.uint8), want_q, "u8", f"{what}: C", nan_class=False)
    assert_matches(s, want_s, "u8", f"{what}: scales", nan_class=False)
    assert_margins(cbuf, c, POISON, f"{what}: C")
    assert_margins(sbuf, s, POISON, f"{what}: scales")
    del abuf
    # dequantize the same bytes with 0xFF (NaN) scale bytes right before and after the scales
    s2buf, s2 = margined(nsc, "u8", 0, 0xFF)
    s2.copy_(s)
    dbuf, d = margined(n, src, off, poison_bits(src))
    va.dequantize_mxfp8(c, s2, TORCH[src], block=block, out=d)
    want_d = tiled(dp, K * block, src)
    if r:
        want_d = torch.cat([want_d, to_dev(MX.dequantize(ql, sl, fmt, src, block), src)])
    torch.cuda.synchronize()
    assert_matches(d, want_d, src, f"{what}: dequantize", nan_class=False)
    assert_margins(dbuf, d, poison_bits(src), f"{what}: dequantize")
    del cbuf, sbuf, s2buf, dbuf


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_mx_block_maximum_at_every_position_with_poisoned_margins(src, fmt):
    """Every block size and rule, the vector path (A and C 16-byte aligned) and the edge path (offset 1), and short
    final blocks of 1, 2, block / 2 and block - 1 elements, after three tiles and more of whole blocks."""
    for block in MX.BLOCKS:
        K = 3 * 4096 // block + 5
        for rule in MX.RULES:
            for off in (0, 1):
                for r in (1, 2, block // 2, block - 1):
                    run_mx(src, fmt, block, rule, off, K * block + r,
                           f"{src}->{fmt} block {block} {rule} offset {off} n={K * block + r}")


@pytest.mark.parametrize("src", DTYPES)
def test_mx_block_maximum_at_every_position_in_the_hbm_class(src):
    h = hbm_n(ES[src])
    for k, block in enumerate(MX.BLOCKS):
        fmt, rule = FMTS[k % 2], MX.RULES[(k // 2 + DTYPES.index(src)) % 2]
        for off in (0, 1):
            run_mx(src, fmt, block, rule, off, h + block - 1, f"{src}->{fmt} block {block} {rule} offset {off} HBM class")
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- dot
def nan_workspace(nbytes):
    return torch.empty(nbytes + 4096, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("dtype", DTYPES)
def test_dot_with_nan_margins_and_a_nan_workspace_at_every_head(dtype):
    """A and B inside NaN margins, at every element offset within 16 bytes together (the vector form with every head)
    and one element apart (the scalar form); the workspace is filled with NaN before every call."""
    epv = 16 // ES[dtype]
    sizes = [1, D.LANES - 1, D.LANES + 1, D.CHUNK - 1, D.CHUNK + 1, 3 * D.CHUNK + 5]
    rng = np.random.default_rng([11, DTYPES.index(dtype)])
    ha, hb = X.finite(dtype, max(sizes), rng, 1.0), X.finite(dtype, max(sizes), rng, 1.0)
    ws = nan_workspace(capi.lib.b200va_dot_workspace_bytes(max(sizes)))
    for n in sizes:
        want = D.dot(ha[:n], hb[:n], dtype)
        layouts = [(o, o) for o in range(epv)] + [(0, 1), (1, 0)]
        outs = torch.full((len(layouts),), 7.0, dtype=torch.float64, device="cuda")
        keep = []
        for k, (oa, ob) in enumerate(layouts):
            abuf, a = margined(n, dtype, oa, NAN[dtype])
            bbuf, b = margined(n, dtype, ob, NAN[dtype])
            put(a, ha[:n], dtype)
            put(b, hb[:n], dtype)
            ws.fill_(0xFF)
            va.dot(a, b, out=outs[k:k + 1], workspace=ws)
            keep.append((abuf, bbuf))
        torch.cuda.synchronize()
        for (oa, ob), got in zip(layouts, outs.tolist()):
            assert same_f64(got, want), f"{dtype} n={n} offsets {oa},{ob}: got {got!r} want {want!r}"


def _chunk_values(a, b, dtype, lo, hi):
    """D.chunk_values of the device operands' elements [lo, hi), copied to the host a block of chunks at a time."""
    out = []
    step = D.BLOCK_CHUNKS * D.CHUNK
    for s in range(lo, hi, step):
        e = min(hi, s + step)
        ha, hb = (x[s:e].view(INT[dtype]).cpu().numpy().view(X.STORAGE[dtype]) for x in (a, b))
        out.append(D.chunk_values(ha, hb, dtype))
    return np.concatenate(out) if out else np.zeros(0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_dot_pass_2_level_edges(dtype):
    """k = 8192 chunk values (the last count pass 2 sums in one level), 8193 (the first with two levels: a second block
    of one partial) and, for f16 and bf16, 16385 (a third block at level 1).  Random finite values against D.dot for
    f32, f16 and bf16, the exactly representable family for f64.  The workspace is NaN before every call and larger
    than the call needs, so a partial that pass 1 does not write, or that pass 2 drops, shows."""
    ks = [8192, 8193] + ([16385] if dtype in ("f16", "bf16") else [])
    ns = [ks[0] * D.CHUNK] + [(k - 1) * D.CHUNK + 1 for k in ks[1:]]
    N = max(ns)
    need = 2 * N * ES[dtype] + (1 << 30)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    if dtype == "f64":
        pa, pb = D.family(dtype, 199_999, 17)
        a, b = tiled(pa, N, dtype), tiled(pb, N, dtype)
        wants = [D.family_sum(pa, pb, dtype, n) for n in ns]
    else:
        g = torch.Generator(device="cuda")
        g.manual_seed(1000 + DTYPES.index(dtype))
        a = torch.randn(N, dtype=TORCH[dtype], device="cuda", generator=g)
        b = torch.randn(N, dtype=TORCH[dtype], device="cuda", generator=g)
        full = _chunk_values(a, b, dtype, 0, N // D.CHUNK * D.CHUNK)
        wants = []
        for n in ns:
            cv = full[:n // D.CHUNK]
            if n % D.CHUNK:
                cv = np.concatenate([cv, _chunk_values(a, b, dtype, n // D.CHUNK * D.CHUNK, n)])
            wants.append(float(D.tree(cv)))
    ws = nan_workspace(capi.lib.b200va_dot_workspace_bytes(N))
    outs = torch.full((len(ns),), 7.0, dtype=torch.float64, device="cuda")
    for k, n in enumerate(ns):
        assert D.chunks(n) == ks[k]
        ws.fill_(0xFF)
        va.dot(a[:n], b[:n], out=outs[k:k + 1], workspace=ws)
    torch.cuda.synchronize()
    for k, n, got, want in zip(ks, ns, outs.tolist(), wants):
        assert same_f64(got, want), f"{dtype} k={k} n={n}: got {got!r} want {want!r}"
    del a, b, ws
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- verify and digest
ONE, FIVE = 0x3F800000, 0x40A00000      # A and B margins hold 1.0, C margins 5.0: mismatches verify must not count


def verify_case(r, off):
    """(A, B, C views, host C, the grid stride of verify_bits_vec in vectors, n) for n mod 4 = r at element offset off,
    with n large enough that thread 0 of verify_bits_vec reaches its second grid-stride slot."""
    stride = torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256
    n = 4 * (2 * stride + 1000) + r
    ha, hb = oracle.fill_ctr(n, 0x51), oracle.fill_ctr(n, 0x52)
    hc = oracle.vadd(ha, hb)
    bufs = []
    views = []
    for h, fill in ((ha, ONE), (hb, ONE), (hc, FIVE)):
        buf, v = margined(n, "f32", off, fill)
        v.copy_(torch.from_numpy(h).cuda())
        bufs.append(buf)
        views.append(v)
    return bufs, views, hc, stride, n


def verify_positions(n, stride):
    nvec = n // 4
    pos = {0, 1, 2, 3, 4 * stride, 4 * stride + 3, 4 * (nvec - 1), 4 * (nvec - 1) + 3, n - 1} | set(range(4 * nvec, n))
    return sorted(pos)


@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "offset1"])
@pytest.mark.parametrize("r", [0, 1, 2, 3])
def test_verify_counts_every_planted_mismatch_and_nothing_outside(r, off):
    bufs, (a, b, c), hc, stride, n = verify_case(r, off)
    if off == 0:
        assert all(x.data_ptr() % 16 == 0 for x in (a, b, c))
    pos = verify_positions(n, stride)
    ci = c.view(torch.int32)
    st = torch.cuda.current_stream().cuda_stream
    plant_sets = [()] + [(p,) for p in pos] + [tuple(pos), (n - 1, 4 * stride, 3), (4 * stride + 3, 4 * (n // 4 - 1))]
    res = torch.empty((len(plant_sets), 2), dtype=torch.int64, device="cuda")
    for k, ps in enumerate(plant_sets):
        for p in ps:
            ci[p:p + 1].bitwise_xor_(1)
        capi.check(capi.lib.b200va_verify_f32(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, res[k].data_ptr(), st),
                   "b200va_verify_f32")
        for p in ps:
            ci[p:p + 1].bitwise_xor_(1)
    torch.cuda.synchronize()
    got = [(int(x), int(y) & (2**64 - 1)) for x, y in res.tolist()]
    bad = []
    for ps, (count, first) in zip(plant_sets, got):
        want = (len(ps), min(ps) if ps else 2**64 - 1)
        if (count, first) != want:
            bad.append(f"planted at {list(ps)[:6]}: ({count}, {first}) want {want}")
    assert not bad, f"n={n} offset {off}: {len(bad)} wrong:\n" + "\n".join(bad[:10])

    # a NaN sum against a NaN of another payload is a match; -0 against +0 and a non-NaN against a NaN sum are not
    ai, bi = a.view(torch.int32), b.view(torch.int32)
    p, q = pos[len(pos) // 2], n - 1
    ai[p:p + 1].fill_(0x7FC00001)
    ci[p:p + 1].fill_(signed(0xFFC12345, "f32"))
    assert va.verify(a, b, c) == (0, -1)
    ci[p:p + 1].fill_(0x3F800000)
    assert va.verify(a, b, c) == (1, p)
    ai[q:q + 1].fill_(0)
    bi[q:q + 1].fill_(0)
    ci[q:q + 1].fill_(signed(0x80000000, "f32"))
    assert va.verify(a, b, c) == (2, p)
    del bufs


@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "offset1"])
@pytest.mark.parametrize("r", [0, 1, 2, 3])
def test_digest_of_an_operand_with_nonzero_margins(r, off):
    bufs, (_, _, c), hc, _, n = verify_case(r, off)
    assert va.digest(c) == oracle.bits_digest(hc), (n, off)
    ci = c.view(torch.int32)
    for p in (0, n - 1):
        ci[p:p + 1].bitwise_xor_(0x10)
        h2 = hc.copy()
        h2.view(np.uint32)[p] ^= 0x10
        assert va.digest(c) == oracle.bits_digest(h2), (n, off, p)
        ci[p:p + 1].bitwise_xor_(0x10)
    del bufs


# ------------------------------------------------------------------------------------------- the wrapper
def test_wrapper_rejects_a_short_or_misplaced_operand_before_calling_the_library():
    n = 4099
    a = torch.ones(n, device="cuda")
    b = torch.ones(n, device="cuda")
    c = torch.zeros(n, device="cuda")
    poison = torch.full((n + 64,), -7.0, device="cuda")
    short = poison[:n - 1]
    cpu = torch.ones(n)
    f64 = torch.ones(n, dtype=torch.float64, device="cuda")
    strided = torch.ones(2 * n, device="cuda")[::2]
    torch.cuda.synchronize()
    calls = [
        ("verify, short b", lambda: va.verify(a, short, c), ValueError),
        ("verify, short c", lambda: va.verify(a, b, short), ValueError),
        ("verify, short a", lambda: va.verify(short, b, c), ValueError),
        ("verify, b on the host", lambda: va.verify(a, cpu, c), TypeError),
        ("add, short out", lambda: va.add(a, b, short), ValueError),
        ("add, short b", lambda: va.add(a, short, c), ValueError),
        ("add_loop, short out", lambda: va.add_loop(a, b, short, 2), ValueError),
        ("add_loop, short b", lambda: va.add_loop(a, short, c, 2), ValueError),
        ("add_loop, out on the host", lambda: va.add_loop(a, b, cpu, 2), TypeError),
        ("Loop, short out", lambda: va.Loop(a, b, short, graph_batch=2), ValueError),
        ("Loop, short a", lambda: va.Loop(short, b, c, graph_batch=2), ValueError),
        ("probe read2, short a", lambda: va.probe("read2", short, b, c), ValueError),
        ("probe read2, short b", lambda: va.probe("read2", a, short, c), ValueError),
        ("probe copy, short a", lambda: va.probe("copy", short, None, c), ValueError),
        ("probe copy, short c", lambda: va.probe("copy", a, None, short), ValueError),
        ("probe read2, f64 a", lambda: va.probe("read2", f64, b, c), TypeError),
        ("probe copy, strided a", lambda: va.probe("copy", strided, None, c), ValueError),
        ("probe read2, b on the host", lambda: va.probe("read2", a, cpu, c), TypeError),
    ]
    for what, call, exc in calls:
        with pytest.raises(exc):
            call()
        torch.cuda.synchronize()
        assert bool((poison == -7.0).all()), f"{what}: the short operand or its neighbours were written"
        assert bool((c == 0).all()), f"{what}: c was written"
    # the unused operands of a probe are not checked, and a full-length call runs
    va.probe("fill", short, None, c)
    va.probe("copy", a, cpu, c)
    torch.cuda.synchronize()


@pytest.mark.skipif(not has_gpu() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_wrapper_rejects_operands_on_two_devices():
    n = 4099
    a, b = torch.ones(n, device="cuda:0"), torch.ones(n, device="cuda:1")
    out = torch.full((n,), -7.0, device="cuda:1")
    for call in (lambda: va.add(a, b), lambda: va.add(a, a, out), lambda: va.add_loop(a, a, out, 2),
                 lambda: va.Loop(a, a, out, graph_batch=2), lambda: va.verify(a, a, out), lambda: va.verify(a, b, a),
                 lambda: va.probe("read2", a, b, out)):
        with pytest.raises(ValueError):
            call()
    torch.cuda.synchronize(1)
    assert bool((out == -7.0).all())
