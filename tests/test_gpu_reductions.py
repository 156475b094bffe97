"""The reductions on the GPU -- the amax of b200va_quantize_fp8 and b200va_quantize_fp8_sr_f32, the amax pass of
b200va_quantize_fp8_auto and _transpose_auto, the fused amax of b200va_quantize_fp8_transpose, the row and column
maxima of b200va_quantize_fp8_rowwise, the MXFP8 block scales, b200va_dot and b200va_verify_f32 / b200va_digest_f32 --
with planted extremes and poisoned neighbours.

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
- The amax pass of the device-chosen scale has its own plan (plan_fp8_amax, restated as AmaxPlan): A's head alone,
  so its head, groups and tail differ from the quantize launch's.  The same cases at margins 0 and 3, every plant
  checked in the amax bits and in k; NaN and +inf are left out of this maximum, so A's margins hold the largest
  finite value.  The transposed form also checks the planted byte in C and Ct under the chosen k.
- The quantize-transpose's amax (plan_fp8_transpose, restated as TransposePlan): on the tiled path a plant in each
  warp's rows and each group of a row, and the corners of the first, a middle, each partial and the last tile, on
  shapes with partial right and bottom tiles and one with more tiles than the SMs hold at once; on the element path
  the first element of every CTA and of its last warp.
- Row-wise: for nb = 1 .. 9 blocks on the row side and on the column side, each line's maximum in block u mod nb, on
  the tiled and the per-block path, so the reduction's unroll remainder holds some line's maximum (ReducePlan).
- Each restated plan's grid and block are pinned to a profiler trace, and tests/test_reduction_coverage.py models on
  the CPU which elements each path covers, showing that a kernel dropping one path misses a planted position.
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

import fp8_auto_exact as AU
import fp8_rowwise_exact as RE
import oracle
from conftest import has_gpu
from oracle import dot_exact as D
from oracle import fp8_exact as F
from oracle import mxfp8_exact as MX
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import DT_CODE, INT, POISON, TORCH, assert_matches, kernels_after_marker, tiled, to_dev
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


# ------------------------------------------------------------------------------------------- the launch plans
# Restated from b200va_typed.cu.  They need no GPU: tests/test_reduction_coverage.py models on the CPU which elements
# each path of a plan covers, and shows that the planted positions below catch a kernel that drops one path.
def hbm_n(es):
    """The smallest n in the HBM class (hbm_class, b200va_internal.h): n elements of es bytes (the wider operand's)
    hold at least 2^25 four-byte words."""
    return (1 << 25) * 4 // es


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
        self._place(n, head, max(esa, esc))

    def _place(self, n, head, es):
        """The vector body from element min(head, n) on in groups of G, and plan_geometry's launch for the HBM class of
        n elements of es bytes, a group being one unit and every element outside the body an edge item."""
        self.n, self.head = n, min(head, n)
        self.ngroups = (n - self.head) // self.G
        hbm = n >= hbm_n(es)
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


class AmaxPlan(CastPlan):
    """plan_fp8_amax (b200va_typed.cu): the amax pass of b200va_quantize_fp8_auto and _transpose_auto over n elements
    of es bytes at pa.  There is no C, so the head is A's own (the elements before A's next 16-byte boundary) and the
    groups are 16 elements; the geometry is A's HBM class.  Its head, groups and tail differ from the quantize
    launch's whenever C's phase differs from A's: with A aligned and C one byte in, the quantize launch is in mixed
    phase and this pass has a full vector body.  It is never in mixed phase past 32 elements, so positions() is
    CastPlan's without the mixed-phase rule."""

    def __init__(self, es, n, pa):
        self.G = 16
        self._place(n, ((16 - pa % 16) % 16) // es, es)


class TransposePlan(CastPlan):
    """plan_fp8_transpose (b200va_typed.cu) for rows x cols elements of es bytes at pa, C at pc and Ct at pt.  The
    tiled path when rows and cols are multiples of 16 and A, C and Ct sit on 16-byte boundaries: one 256-thread CTA
    per 64 x 64 tile (no head, no unroll), thread t taking group t % 4 of tile row t / 4, so warp w takes tile rows
    8 w .. 8 w + 7; tiles on the right and bottom edges are partial in steps of 16.  Otherwise the element path: head
    = n, every element an edge item of plan_geometry's grid for A's HBM class, as CastPlan in mixed phase."""
    T = 64

    def __init__(self, es, rows, cols, pa, pc, pt):
        self.rows, self.cols, self.G = rows, cols, 16
        self.tiled = rows % 16 == 0 and cols % 16 == 0 and (pa | pc | pt) % 16 == 0
        if not self.tiled:
            self._place(rows * cols, rows * cols, es)
            return
        self.n, self.head, self.ngroups = rows * cols, 0, rows * cols // 16
        self.threads, self.unroll = 256, 1
        self.tiles_c = -(-cols // self.T)
        self.grid = -(-rows // self.T) * self.tiles_c

    def box(self, t):
        """(first row, first column, rows, columns) of tile t."""
        i0, j0 = t // self.tiles_c * self.T, t % self.tiles_c * self.T
        return i0, j0, min(self.T, self.rows - i0), min(self.T, self.cols - j0)

    def positions(self):
        """The element path: CastPlan's mixed-phase positions.  The tiled path: in tile 0, one element in each warp's
        rows (row 9 w of the tile, group w % 4), and the four corners of tile 0, of a middle tile, of the first
        partial right tile, of the first partial bottom tile and of the last tile."""
        if not self.tiled:
            return super().positions()
        at = lambda i, j: i * self.cols + j                                  # noqa: E731
        tiles_r = self.grid // self.tiles_c
        tiles = {0, tiles_r // 2 * self.tiles_c + self.tiles_c // 2, self.grid - 1}
        tiles |= {self.tiles_c - 1} if self.cols % self.T else set()
        tiles |= {self.grid - self.tiles_c} if self.rows % self.T else set()
        pos = set()
        for t in tiles:
            i0, j0, tr, tc = self.box(t)
            pos |= {at(i0, j0), at(i0, j0 + tc - 1), at(i0 + tr - 1, j0), at(i0 + tr - 1, j0 + tc - 1)}
        _, _, tr, tc = self.box(0)
        pos |= {at(9 * w, 16 * (w % 4) + 5 * w % 16) for w in range(8) if 9 * w < tr and 16 * (w % 4) < tc}
        return sorted(pos)


class ReducePlan:
    """The FP8R_REDUCE launch of b200va_quantize_fp8_rowwise with both sides asked for: plan_geometry below the HBM
    class with one edge item per row (S), then per column (St).  The thread of a row walks the row's nb = ceil(cols /
    128) 1x128 block scales, that of a column its ceil(rows / 128), in fp8r_reduce's loop under `#pragma unroll 4`."""
    threads = 256

    def __init__(self, rows, cols):
        self.nb_row, self.nb_col = -(-cols // 128), -(-rows // 128)
        self.grid = max(1, -(-(rows + cols) // self.threads))


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
    if "whole" in expect:
        assert p.ngroups and p.ngroups % p.tile == 0, f"{what}: not whole tiles"


def amax_pass_expect(es, n, expect):
    """What the amax pass of an amax case must show: the case's expectations but mixed phase, which only the quantize
    launch has (A aligned and C one byte in give the amax pass a full vector body).  An f64 A one element in has a
    head of 1, so the amax pass over 15 + 16 (t - 1) + 3 elements has one whole tile of t groups, not a partial one."""
    expect = tuple(e for e in expect if e != "mixed")
    return tuple(e for e in expect if e != "partial") + ("whole",) if (es, n) == (8, 15 + 16 * 255 + 3) else expect


# (rows, cols, element offsets of A, C and Ct, what the plan must show) of the quantize-transpose amax cases
TRANSPOSE_CASES = [(128, 192, (0, 0, 0), ("tiled",)),
                   (192, 208, (0, 0, 0), ("tiled", "right")),            # cols % 64 = 16
                   (176, 128, (0, 0, 0), ("tiled", "bottom")),           # rows % 64 = 48
                   (144, 240, (0, 0, 0), ("tiled", "right", "bottom")),  # 16 and 48
                   (80, 112, (0, 0, 0), ("tiled", "right", "bottom")),   # 16 and 48, one full tile
                   (2112, 4096, (0, 0, 0), ("tiled", "resident")),       # 2112 tiles
                   (100, 203, (0, 0, 0), ("element",)),
                   (64, 80, (0, 0, 1), ("element",))]                    # Ct one byte off a 16-byte boundary
# 2048 threads per SM: at most 8 of the tiled path's 256-thread CTAs are resident on one
CTAS_PER_SM = 2048 // 256


def assert_transpose_reaches(p: TransposePlan, expect, sms, what):
    assert p.tiled == ("tiled" in expect), f"{what}: tiled {p.tiled}"
    if "right" in expect:
        assert p.cols % 64 in (16, 48), f"{what}: no partial right tile"
    if "bottom" in expect:
        assert p.rows % 64 in (16, 48), f"{what}: no partial bottom tile"
    if "resident" in expect:
        assert p.grid > sms * CTAS_PER_SM, f"{what}: {p.grid} tiles fit in {sms} SMs at once"
    if "element" in expect:
        assert p.grid > 1, f"{what}: one CTA"


def rowwise_cases():
    """(side, nb, rows, cols, A's element offset, path): for nb = 1 .. 9 blocks on the row side (cols = 128 nb) and on
    the column side (rows = 128 nb), the tiled path and the per-block path (cols = 128 nb - 5, or A one element off a
    16-byte boundary)."""
    cases = []
    for nb in range(1, 10):
        cases += [("row", nb, 16 * (1 + nb % 2), 128 * nb, 0, "tiled"), ("row", nb, 16, 128 * nb - 5, 0, "per-block"),
                  ("col", nb, 128 * nb, 128, 0, "tiled"), ("col", nb, 128 * nb, 128, 1, "per-block")]
    return cases


def rowwise_plants(side, nb, rows, cols):
    """[(row, column)]: line u of the side (row u, or column u, of A) holds its maximum in block u mod nb along it, at
    37 u modulo the block's length."""
    if side == "row":
        return [(u, 128 * (u % nb) + 37 * u % min(128, cols - 128 * (u % nb))) for u in range(rows)]
    return [(128 * (u % nb) + 37 * u % min(128, rows - 128 * (u % nb)), u) for u in range(cols)]


def plant_each(a, src, plants, launch):
    """launch(k) for each plant k = (position, bit pattern) with that element of a holding the pattern (None: a as
    it is), restored after the launch.  No synchronise."""
    ai = a.view(INT[src])
    for k, (q, bits) in enumerate(plants):
        if q is None:
            launch(k)
            continue
        keep = ai[q:q + 1].clone()
        ai[q:q + 1].fill_(signed(bits, src))
        launch(k)
        ai[q:q + 1].copy_(keep)


def planted(src, pos, bg_amax):
    """[(position, bit pattern, the amax the call must give)] of the host-k calls, whose amax takes NaN and +inf:
    none (the background's amax), PLANT of alternating sign at every position, a NaN at the first and last and a
    +inf at the last."""
    mag, sgn = storage_bits(PLANT, src), SIGN[src]
    plants = [(None, None, bg_amax)] + [(q, mag | (sgn if k % 2 else 0), PLANT) for k, q in enumerate(pos)]
    return plants + [(pos[0], NAN[src], math.nan), (pos[-1], NAN[src], math.nan), (pos[-1], INF[src], math.inf)]


def run_plants(a, src, plants, launch, case):
    """launch(a, amax) once per plant, each into its own zeroed f64 slot, one synchronise; every slot against its
    want."""
    slots = torch.zeros(len(plants), dtype=torch.float64, device="cuda")
    plant_each(a, src, [(q, bits) for q, bits, _ in plants], lambda k: launch(slots[k:k + 1]))
    torch.cuda.synchronize()
    bad = [f"planted {bits:#x} at {q}: amax {g!r}, want {w!r}" for (q, bits, w), g in zip(plants, slots.tolist())
           if not same_f64(g, w)]
    assert not bad, f"{case}: {len(bad)} of {len(plants)} wrong:\n" + "\n".join(bad[:10])


def run_planted_amax(src, fmt, launch, what):
    """Every amax case of src into fmt, NaN margins around A: per case one launch per plant, each into its own f64
    slot, with one synchronise per case."""
    bg = background(src)
    for n, layout, expect in amax_cases(ES[src]):
        oa, oc = LAYOUTS[layout]
        abuf, a = margined(n, src, oa, NAN[src])
        a.view(INT[src]).copy_(tiled(bg, n, src).view(INT[src]))
        cbuf, c = margined(n, fmt, oc, POISON)
        p = CastPlan(ES[src], 1, n, a.data_ptr(), c.data_ptr())
        case = f"{what} n={n} {layout} (head {p.head}, {p.ngroups} groups, grid {p.grid} x {p.threads}, unroll {p.unroll})"
        assert_reaches(p, expect, case)
        run_plants(a, src, planted(src, p.positions(), F.amax(bg[:n], src)), lambda m: launch(a, c, m), case)
        assert_margins(cbuf, c, POISON, case)
        del abuf, cbuf, a, c


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


# ------------------------------------------------------------------------------------------- the device-chosen scale
def host_element(bits, src):
    """The one-element host storage of src whose bit pattern is bits."""
    return np.array([bits], {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[ES[src]]).view(X.STORAGE[src])


def finite_amax_without(bg, n, q, src):
    """The amax pass's result over n elements of the background (bg repeated) with element q taken out (a NaN or
    +inf planted there).  Past PERIOD elements, q's value is still held by q +- PERIOD when that is in range."""
    if n > PERIOD and (q >= PERIOD or q + PERIOD < n):
        return AU.finite_amax(bg, src)
    return AU.finite_amax(np.delete(bg[:n], q), src)


@pytest.mark.parametrize("form", ["1-D", "transpose"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_auto_amax_pass_finds_a_maximum_planted_at_every_path_edge(src, fmt, form):
    """quantize_fp8_auto, or quantize_fp8_transpose_auto of A as 1 x n, over every amax case at margins 0 and 3, the
    plants at AmaxPlan's positions.  Each launch has its own zeroed amax and its own k slot.  The background stays
    below 2, so k differs with and without PLANT: a missed plant shows in k too.  The pass takes finite values only,
    so a NaN or +inf plant gives the amax and k of the background without that element, and A's margins hold the
    largest finite value.  The
    planted element's byte in C (and Ct) is the reference's under the planted k: the quantize took the pass's k."""
    bg = background(src)
    mag, sgn = storage_bits(PLANT, src), SIGN[src]
    for n, layout, expect in amax_cases(ES[src]):
        oa, oc = LAYOUTS[layout]
        abuf, a = margined(n, src, oa, MAX_FINITE[src])
        a.view(INT[src]).copy_(tiled(bg, n, src).view(INT[src]))
        cbuf, c = margined(n, fmt, oc, POISON)
        tbuf, ct = margined(n, fmt, oc, POISON) if form == "transpose" else (None, None)
        p = AmaxPlan(ES[src], n, a.data_ptr())
        case = f"{form} auto {src}->{fmt} n={n} {layout} (amax pass: head {p.head}, {p.ngroups} groups, grid {p.grid} x " \
               f"{p.threads}, unroll {p.unroll})"
        assert_reaches(p, amax_pass_expect(ES[src], n, expect), case)
        pos = p.positions()
        bg_amax = AU.finite_amax(bg[:n], src)
        plants = [(None, None, bg_amax)] + [(q, mag | (sgn if k % 2 else 0), PLANT) for k, q in enumerate(pos)]
        plants += [(q, bits, finite_amax_without(bg, n, q, src)) for bits in (NAN[src], INF[src]) for q in (pos[0], pos[-1])]
        for margin in (0, 3):
            what = f"{case} margin {margin}"
            assert AU.auto_scale_exp(PLANT, fmt, margin) != AU.auto_scale_exp(bg_amax, fmt, margin), what
            m = torch.zeros(len(plants), dtype=torch.float64, device="cuda")
            s = torch.full((len(plants),), -999, dtype=torch.int32, device="cuda")
            got = torch.zeros((len(plants), 2), dtype=torch.uint8, device="cuda")

            def launch(k):
                if form == "1-D":
                    va.quantize_fp8_auto(a, TORCH[fmt], margin=margin, amax=m[k:k + 1], scale_exp=s[k:k + 1], out=c)
                else:
                    va.quantize_fp8_transpose_auto(a.view(1, n), TORCH[fmt], margin=margin, amax=m[k:k + 1],
                                                   scale_exp=s[k:k + 1], out=c.view(1, n), out_t=ct.view(n, 1))
                q = plants[k][0]
                if q is not None:                    # element (0, q) is C[q] and, in the n x 1 transpose, Ct[q]
                    got[k, 0:1].copy_(c.view(torch.uint8)[q:q + 1])
                    if ct is not None:
                        got[k, 1:2].copy_(ct.view(torch.uint8)[q:q + 1])

            plant_each(a, src, [(q, bits) for q, bits, _ in plants], launch)
            torch.cuda.synchronize()
            bad = []
            for (q, bits, want), gm, gk, gb in zip(plants, m.tolist(), s.tolist(), got.tolist()):
                wk = AU.auto_scale_exp(want, fmt, margin)
                if not same_f64(gm, want) or gk != wk:
                    bad.append(f"planted {bits!r} at {q}: amax {gm!r} k {gk}, want {want!r} k {wk}")
                elif want == PLANT:
                    wb = int(F.quantize(host_element(bits, src), src, fmt, wk)[0])
                    if gb[0] != wb or (ct is not None and gb[1] != wb):
                        bad.append(f"planted {bits:#x} at {q}: bytes C {gb[0]:#x} Ct {gb[1]:#x}, want {wb:#x}")
            assert not bad, f"{what}: {len(bad)} of {len(plants)} wrong:\n" + "\n".join(bad[:10])
        assert_margins(cbuf, c, POISON, case + " C")
        if ct is not None:
            assert_margins(tbuf, ct, POISON, case + " Ct")
        del abuf, cbuf, tbuf, a, c, ct


# ------------------------------------------------------------------------------------------- the quantize-transpose
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", DTYPES)
def test_quantize_transpose_amax_finds_a_maximum_planted_at_every_tile_and_warp_edge(src, fmt):
    """quantize_fp8_transpose (host k) over TRANSPOSE_CASES, NaN margins around A, the plants at TransposePlan's
    positions: on the tiled path every warp's rows, every group of a row and the corners of the first, a middle, each
    partial and the last tile; on the element path the first element of every CTA and of its last warp.  Its amax
    takes NaN (a NaN plant gives NaN).  C's and Ct's margins keep their poison."""
    bg = background(src)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for rows, cols, (oa, oc, ot), expect in TRANSPOSE_CASES:
        n = rows * cols
        abuf, a = margined(n, src, oa, NAN[src])
        a.view(INT[src]).copy_(tiled(bg, n, src).view(INT[src]))
        cbuf, c = margined(n, fmt, oc, POISON)
        tbuf, ct = margined(n, fmt, ot, POISON)
        p = TransposePlan(ES[src], rows, cols, a.data_ptr(), c.data_ptr(), ct.data_ptr())
        case = f"transpose {src}->{fmt} {rows}x{cols} offsets {oa},{oc},{ot} ({'tiled' if p.tiled else 'element'} path, " \
               f"grid {p.grid} x {p.threads})"
        assert_transpose_reaches(p, expect, sms, case)
        run_plants(a, src, planted(src, p.positions(), F.amax(bg[:n], src)),
                   lambda m: va.quantize_fp8_transpose(a.view(rows, cols), TORCH[fmt], scale_exp=0, amax=m,
                                                       out=c.view(rows, cols), out_t=ct.view(cols, rows)), case)
        assert_margins(cbuf, c, POISON, case + " C")
        assert_margins(tbuf, ct, POISON, case + " Ct")
        del abuf, cbuf, tbuf, a, c, ct


# ------------------------------------------------------------------------------------------- the row-wise scales
def line_top(u):
    """The magnitude line u's maximum has: 1 + (u mod 8) / 8 times 2^(1 + (u / 8) mod 4), above the background's 1, so
    each line's k differs from the background's and the k of neighbouring lines differ."""
    return (1 + (u % 8) / 8) * 2.0 ** (1 + (u // 8) % 4)


@pytest.mark.parametrize("src", DTYPES)
def test_rowwise_reduction_finds_a_line_maximum_planted_in_every_block(src):
    """quantize_fp8_rowwise, both sides, over rowwise_cases(): each line of the side under test holds its maximum in
    block u mod nb, so for nb = 1 .. 9 every block of a row (or column) holds some line's maximum, the unroll
    remainder of fp8r_reduce's loop included.  C, S, Ct and St bit for bit against tests/fp8_rowwise_exact.py; A's
    margins hold the largest finite value, and the margins of C, Ct, S, St and the workspace keep their poison."""
    for side, nb, rows, cols, oa, path in rowwise_cases():
        fmt = FMTS[nb % 2]
        n = rows * cols
        x = np.random.default_rng([19, nb, rows, cols]).uniform(-0.99, 0.99, (rows, cols))
        for u, (i, j) in enumerate(rowwise_plants(side, nb, rows, cols)):
            x[i, j] = line_top(u) * (-1) ** u
        host = (X.narrow(x.astype(np.float32), src) if src in ("f16", "bf16") else x.astype(X.STORAGE[src])).ravel()
        abuf, a = margined(n, src, oa, MAX_FINITE[src])
        put(a, host, src)
        bufs = {"C": margined(n, fmt, 0, POISON), "Ct": margined(n, fmt, 0, POISON),
                "S": margined(rows, "f32", 0, poison_bits("f32")), "St": margined(cols, "f32", 0, poison_bits("f32")),
                "workspace": margined(RE.workspace_bytes(rows, cols), "u8", 0, POISON)}
        v = {k: b[1] for k, b in bufs.items()}
        tiled_path = cols % 128 == 0 and rows % 16 == 0 and a.data_ptr() % 16 == 0
        case = f"row-wise {src}->{fmt} {rows}x{cols} offset {oa}: {side} side, {nb} blocks, {path} path"
        assert tiled_path == (path == "tiled"), case
        va.quantize_fp8_rowwise(a.view(rows, cols), TORCH[fmt], out=v["C"].view(rows, cols), scales=v["S"],
                                out_t=v["Ct"].view(cols, rows), scales_t=v["St"], workspace=v["workspace"])
        wc, ws, wct, wst = RE.quantize(host, src, fmt, rows, cols)
        torch.cuda.synchronize()
        for name, want in (("C", wc), ("Ct", wct)):
            assert_matches(v[name].view(torch.uint8), to_dev(want.ravel(), "u8"), "u8", f"{case}: {name}", nan_class=False)
        for name, want in (("S", ws), ("St", wst)):
            assert_matches(v[name], to_dev(want, "f32"), "f32", f"{case}: {name}", nan_class=False)
        for name, (buf, view) in bufs.items():
            assert_margins(buf, view, POISON if buf.element_size() == 1 else poison_bits("f32"), f"{case}: {name}")
        del abuf, a, bufs, v


# ------------------------------------------------------------------------------------------- the plans in the trace
def test_restated_plans_match_the_traced_launches(tmp_path):
    """The grid and block of every launch the plants above rely on, against the restated plan that placed them:
    AmaxPlan (the amax pass, with CastPlan's quantize launch behind it) for a head, a mixed-phase and an HBM-class
    case of every element size; TransposePlan for every case of TRANSPOSE_CASES in f32; ReducePlan for a row side and
    a column side.  A restatement that disagrees fails naming its plan."""
    calls, want = [], []
    keep = []
    for src in ("f16", "f32", "f64"):
        for n, layout, _ in amax_cases(ES[src]):
            if layout == "aligned" or n < 3 * 256 or (n >= hbm_n(ES[src]) and src != "f16"):
                continue
            oa, oc = LAYOUTS[layout]
            _, a = margined(n, src, oa, 0)
            _, c = margined(n, "e4m3", oc, 0)
            m, s = torch.zeros(1, dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
            keep += [a, c, m, s]
            calls.append(lambda a=a, c=c, m=m, s=s: va.quantize_fp8_auto(a, torch.float8_e4m3fn, amax=m, scale_exp=s, out=c))
            pa, pq = AmaxPlan(ES[src], n, a.data_ptr()), CastPlan(ES[src], 1, n, a.data_ptr(), c.data_ptr())
            kernel = f"fp8_quant_vec<{DT_CODE[src]}>"
            want += [(f"AmaxPlan {src} n={n} {layout}", kernel, pa.grid, pa.threads),
                     (f"CastPlan {src} n={n} {layout}", kernel, pq.grid, pq.threads)]
    for rows, cols, (oa, oc, ot), _ in TRANSPOSE_CASES:
        n = rows * cols
        _, a = margined(n, "f32", oa, 0)
        _, c = margined(n, "e4m3", oc, 0)
        _, ct = margined(n, "e4m3", ot, 0)
        keep += [a, c, ct]
        calls.append(lambda a=a, c=c, ct=ct, r=rows, k=cols: va.quantize_fp8_transpose(
            a.view(r, k), torch.float8_e4m3fn, out=c.view(r, k), out_t=ct.view(k, r)))
        p = TransposePlan(4, rows, cols, a.data_ptr(), c.data_ptr(), ct.data_ptr())
        want.append((f"TransposePlan {rows}x{cols} offsets {oa},{oc},{ot}", "fp8_quant_vec<0>", p.grid, p.threads))
    for side, nb, rows, cols, oa, path in rowwise_cases():
        if nb != 9:
            continue
        a = torch.zeros(rows * cols + oa, device="cuda")[oa:].view(rows, cols)
        keep.append(a)
        calls.append(lambda a=a: va.quantize_fp8_rowwise(a, torch.float8_e4m3fn))
        p = ReducePlan(rows, cols)
        want += [None, (f"ReducePlan {rows}x{cols} offset {oa} ({side} side, {path} path)", "mx_quant_vec<4>", p.grid,
                        p.threads), None]
    for call in calls:
        call()
    torch.cuda.synchronize()

    def plan():
        for call in calls:
            call()
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, plan, ("fp8_", "mx_"))
    assert len(got) == len(want), (len(got), len(want))
    for g, w in zip(got, want):
        if w is not None:
            assert g == w[1:], f"{w[0]}: traced {g}, restated {w[1:]}"
    del keep

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
