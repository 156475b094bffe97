"""Every add kernel both libraries carry, launched through the C ABI and compared with the oracle; the STREAM kernels
only the tune library's B200VA_STREAM_GEOMETRY reaches, compared with the exact reference.

test_kernel_inventory.py restates which kernels each library carries.  Here each of the 1174 add kernels of
libb200va_tune.so runs at one geometry it accepts, and the 88 of libb200va.so run from that library:
- Two input pools from oracle.fill_ctr, one element in 61 replaced by a special pair (signed zeros, subnormals,
  finite values that overflow, infinities, NaN); a third of B negated, so sums cancel.  The expected sum of the
  whole pools comes from oracle.vadd once and is uploaded once.
- A kernel's shapes are windows at the same positions in A, B and an output arena, with poisoned elements between
  them.  Per kernel the arena is poisoned, every shape is launched back to back on one stream, and one device-side
  comparison checks the whole arena: the windows against the oracle (NaN as a class), the rest still poisoned.
- Copies of the pools whose element 0 lies 4, 8 or 16 bytes past an aligned address put A, B and C in different
  phases at the same index: 16 bytes (K3 drops to the 16-byte body) and no common 16-byte phase (the K4 path).
The shapes follow from each kernel's plan, restated in gpu_helpers.expected_add_launch, and the test asserts per
kernel what they cover: no vector body, every head, exactly one tile and one vector either side of it, a ragged
last tile, and more tiles than CTAs (for the TMA ring, a ring that wraps at least twice per CTA).

This module sorts after test_gpu_parity.py and test_gpu_stream.py: its profiler traces come after theirs (DESIGN.md
section 3).
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from conftest import ROOT, has_gpu
from oracle import stream_exact as X
from test_kernel_inventory import add_kernels, add_tunes, sass_kernels

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import (ES, GUARD, assert_guards, assert_matches, expected_add_launch,
                             expected_stream_launch, geometry, kernels_after_marker, poisoned, tiled)
    from k8s_gpu_hpa_b200 import capi

POOL = 1 << 25                      # elements per input pool and in the output arena
GAP = 16                            # poisoned elements at least between two windows
POISON32 = 0x5A5A5A5A               # the arena's f32 word (gpu_helpers.POISON bytes): finite, about 1.5e16
SPECIAL_STRIDE = 61
F32_MAX, F32_INF, F32_QNAN = 0x7F7FFFFF, 0x7F800000, 0x7FC00001
SPECIALS = [  # (A bits, B bits)
    (0x00000000, 0x80000000), (0x80000000, 0x80000000), (0x80000000, 0x00000000), (0x3F800000, 0xBF800000),
    (0x00000001, 0x00000001), (0x007FFFFF, 0x00000001), (0x80000003, 0x00000001), (0x00400000, 0x80400001),
    (F32_MAX, F32_MAX), (F32_MAX | 1 << 31, F32_MAX | 1 << 31), (F32_MAX, 0x73000000), (F32_MAX, 0x72FFFFFF),
    (F32_INF, 0x3F800000), (F32_INF | 1 << 31, 0xBF800000), (F32_INF, F32_INF | 1 << 31), (F32_INF, F32_INF),
    (F32_QNAN, 0x3F800000), (0x3F800000, F32_QNAN | 1 << 31)]
A_SHIFTS, B_SHIFTS = (0, 1), (0, 2, 4)      # elements past a 256-byte boundary of each pool copy
THREADS = (32, 64, 96, 128, 192, 256, 320, 384, 512, 640, 768, 1024)
STAGES, TILES, CONSUMERS = (2, 3, 5, 8), (2048, 6144, 8192, 28672), (32, 128, 992)
K4_THREADS = (32, 96, 256, 640, 1024)


# ------------------------------------------------------------------------------------------- inputs and arena
class Matrix:
    """The pools, their shifted copies, the arena, the expected sums and each library's tunes with a geometry."""

    def __init__(self):
        a = oracle.fill_ctr(POOL, 0x0A).view(np.uint32)
        b = oracle.fill_ctr(POOL, 0x0B).view(np.uint32)
        b[::3] |= np.uint32(1 << 31)
        idx = np.arange(7, POOL, SPECIAL_STRIDE)
        sp = np.array(SPECIALS, dtype=np.uint32)
        a[idx], b[idx] = sp[idx % len(sp), 0], sp[idx % len(sp), 1]
        ha, hb = a.view(np.float32), b.view(np.float32)
        self.A = {s: self._shifted(ha, s) for s in A_SHIFTS}
        self.B = {s: self._shifted(hb, s) for s in B_SHIFTS}
        self.E = self._shifted(oracle.vadd(ha, hb), 0)          # the expected C = A + B at every index
        self.EAA = self._shifted(oracle.vadd(ha, ha), 0)        # A + A, for A == B == C
        self.arena = self._shifted(np.zeros(POOL, np.float32), 0)
        self.want = torch.empty_like(self.arena)
        self.want_layout = None
        self.stream = torch.cuda.Stream()
        self.tunes = choose_geometries(add_tunes("tune"), capi.tune_lib())

    @staticmethod
    def _shifted(host, s):
        raw = torch.empty(host.size + 8, dtype=torch.float32, device="cuda")
        view = raw[s:s + host.size]
        view.copy_(torch.from_numpy(host))
        return view

    def ptrs(self, p, sa=0, sb=0):
        return (self.A[sa].data_ptr() + 4 * p, self.B[sb].data_ptr() + 4 * p, self.arena.data_ptr() + 4 * p)

    def expect(self, windows, extent):
        """self.want[:extent]: poison, and over each (p, n, "E" or "EAA") window that expected sum."""
        if self.want_layout != (windows, extent):
            w = self.want[:extent]
            w.view(torch.int32).fill_(POISON32)
            for p, n, src in windows:
                w[p:p + n].copy_(getattr(self, src)[p:p + n])
            self.want_layout = (windows, extent)

    def first_bad(self, extent):
        """The first arena index whose bits differ from self.want (NaN as a class), or -1."""
        g, w = self.arena[:extent].view(torch.int32), self.want[:extent].view(torch.int32)
        bad = g != w
        bad &= ~(((g & 0x7FFFFFFF) > 0x7F800000) & ((w & 0x7FFFFFFF) > 0x7F800000))
        return int(torch.nonzero(bad)[0]) if bool(bad.any()) else -1


@pytest.fixture(scope="module")
def mx():
    free, _ = torch.cuda.mem_get_info()
    if free < (3 << 30):
        pytest.skip(f"needs about 3 GiB of free device memory, {free >> 20} MiB free")
    m = Matrix()
    torch.cuda.synchronize()
    yield m
    del m
    torch.cuda.empty_cache()


def choose_geometries(tunes, lib):
    """Each tune with a geometry the library accepts (b200va_geometry), rotated over the kernels: vec threads over
    THREADS and ctas_per_sm over 0, 1, 2 (0 under the dynamic scheduler), TMA stages, tile bytes and consumer threads
    over STAGES, TILES and CONSUMERS.  A refused geometry steps the threads (vec, K4) or the stages (TMA) down.
    Returns [(tune, None)] for the kernels no geometry could launch, so that they are reported, not dropped."""
    out = []
    for i, base in enumerate(tunes):
        t = capi.Tune(**base.as_dict())
        if t.kind == capi.K0_SCALAR:
            t.threads, t.unroll = 256, 1
            cands = [t]
        elif t.kind == capi.K2_TMA:
            t.ctas_per_sm = 1
            t.threads = CONSUMERS[i % 3]
            t.tile_bytes = TILES[(i // 3) % 4]
            first = STAGES[(i // 12 + i) % 4]
            cands = []
            for s in [s for s in STAGES if s <= first][::-1]:
                c = capi.Tune(**t.as_dict())
                c.stages = s
                cands.append(c)
        else:
            if t.kind != capi.K4_SCALAR_MLP:
                t.ctas_per_sm = 0 if t.scheduler else (i // len(THREADS)) % 3
            first = THREADS[i % len(THREADS)]
            cands = []
            for th in [th for th in THREADS if th <= first][::-1]:
                c = capi.Tune(**t.as_dict())
                c.threads = th
                cands.append(c)
        chosen = None
        for c in cands:
            if geometry(c, 1 << 20, lib)[0] == geometry(alias_twin(c), 1 << 20, lib)[0] == capi.OK:
                chosen = c
                break
        out.append((base, chosen))
    return out


def alias_twin(t):
    """The tune plan_launch runs for t when C is A or B: plain loads for .nc ones, the L2 prefetch for early register
    loads.  A geometry is chosen that both accept, so that the aliased launches run too."""
    e = capi.Tune(**t.as_dict())
    if e.kind in (capi.K1_VEC128, capi.K3_VEC256):
        e.ld_hint = 0 if e.ld_hint == 4 else e.ld_hint
        e.early_loads = 2 if e.early_loads == 1 else e.early_loads
    return e


# ------------------------------------------------------------------------------------------- shapes
def vec_width(t):
    return {capi.K3_VEC256: 8, capi.K1_VEC128: 4, capi.K2_TMA: 4}.get(t.kind, 1)


def tile_elems(t):
    """Elements of one tile: threads x unroll vectors (vec, K4, K0), tile_bytes of each operand (TMA)."""
    if t.kind == capi.K2_TMA:
        return t.tile_bytes // 4
    return t.threads * t.unroll * vec_width(t)


def head_of(vw, off):
    return (vw - off % vw) % vw


def big_tiles(t, lib):
    """Tiles of the shape that makes a persistent grid loop: 1.5 times the CTAs of the grid at a huge n plus one; for
    the TMA ring, enough that every CTA's ring wraps at least twice.  A grid of one CTA per tile gets 5 tiles."""
    huge = 1 << 30
    _, grid, _ = geometry(t, huge, lib)
    if t.kind == capi.K2_TMA:
        return 2 * grid * t.stages + grid + 1
    if grid >= -(-huge // tile_elems(t)):
        return 5
    return grid + grid // 2 + 1


def shapes(t, lib):
    """[(n, off, sa, sb)]: n elements at a window starting off elements past a 32-byte boundary, A from the pool copy
    shifted by sa elements, B by sb."""
    vw, te = vec_width(t), tile_elems(t)
    out = [(1, 0, 0, 0), (2, 1, 0, 0), (3, 0, 0, 0), (5, 3, 0, 0), (7, 1, 0, 0)]     # no vector body
    out += [(4133 + 3 * off, off, 0, 0) for off in range(8)]                          # every head
    for off in (2, 5):                                                                # one tile, and one vector either side
        h = head_of(vw, off)
        out += [(h + te, off, 0, 0), (h + te - vw, off, 0, 0), (h + te + vw, off, 0, 0)]
    h = head_of(vw, 6)
    out.append((h + 3 * te + 5 * vw + 3 % vw, 6, 0, 0))                               # a ragged last tile
    out += [(4133, 0, 0, 4), (4133 + 5, 1, 0, 4)]                                     # equal mod 16, not mod 32
    h = head_of(vw, 1)
    out.append((h + (big_tiles(t, lib) - 1) * te + te // 2 + 3 % vw, 1, 0, 0))        # more tiles than CTAs
    return out


def layout(shape_list, src_of=None):
    """[(p, n, sa, sb)] at increasing positions and the arena extent they need."""
    pos, out = 0, []
    for n, off, sa, sb in shape_list:
        p = -(-(pos + GAP) // 64) * 64 + off
        out.append((p, n, sa, sb))
        pos = p + n
    extent = pos + GAP
    assert extent + 8 <= POOL, f"the shapes need {extent} arena elements"
    return out, extent


def covered(t, shape_list, mx, lib):
    """What the shapes give kernel t, from its restated plan: the missing properties (empty when all are there)."""
    vw, te = vec_width(t), tile_elems(t)
    if t.kind in (capi.K0_SCALAR, capi.K4_SCALAR_MLP):
        return []
    tile_vecs = te // vw
    heads, bodies, missing = set(), [], []
    no_body_short = no_body_head = fallback = ragged = loops = False
    for n, off, sa, sb in shape_list:
        pa, pb, pc = mx.ptrs(off, sa, sb)
        rc, name, grid, _ = expected_add_launch(t, n, pa, pb, pc, lib)
        w = 8 if "<8," in name else 4
        head = min(n, ((w * 4 - (pa & (w * 4 - 1))) & (w * 4 - 1)) // 4)
        nvec = (n - head) // w
        fallback |= vw == 8 and w == 4
        if w != vw:
            continue
        no_body_short |= n < vw
        no_body_head |= 0 < n <= head
        if nvec:
            heads.add(head)
            bodies.append(nvec)
        if t.kind == capi.K2_TMA:
            ntiles = -(-(nvec * 16) // t.tile_bytes)
            ragged |= nvec * 16 > t.tile_bytes and (nvec * 16) % t.tile_bytes != 0
            loops |= ntiles >= grid * (2 * t.stages + 1)
        else:
            ntiles = -(-nvec // tile_vecs)
            ragged |= nvec > tile_vecs and nvec % tile_vecs != 0
            loops |= ntiles > grid or (ntiles >= 5 and grid == ntiles)
    tile_nvec = t.tile_bytes // 16 if t.kind == capi.K2_TMA else tile_vecs
    checks = {"no vector body, n < VW": no_body_short, "no vector body, head >= n": no_body_head,
              f"every head 0..{vw - 1}": heads >= set(range(vw)),
              "one tile": tile_nvec in bodies, "one tile + 1 vector": tile_nvec + 1 in bodies,
              "one tile - 1 vector": tile_nvec - 1 in bodies, "a ragged last tile": ragged,
              "more tiles than CTAs": loops}
    if vw == 8:
        checks["the 16-byte fallback"] = fallback
    return [k for k, ok in checks.items() if not ok]


def run_kernel(mx, lib, t, shape_list):
    """Poison the arena, launch every shape back to back on one stream, compare once.  None, or what went wrong."""
    wins, extent = layout(shape_list)
    st = mx.stream
    with torch.cuda.stream(st):
        mx.expect(tuple((p, n, "E") for p, n, _, _ in wins), extent)
        mx.arena[:extent].view(torch.int32).fill_(POISON32)
        for p, n, sa, sb in wins:
            rc = lib.b200va_add_f32_tuned(*mx.ptrs(p, sa, sb), n, C.byref(t), st.cuda_stream)
            if rc != capi.OK:
                return f"n={n} at {p} (A +{sa}, B +{sb}): {capi.strerror(rc)} ({rc})"
        bad = mx.first_bad(extent)
    if bad < 0:
        return None
    win = next(((p, n, sa, sb) for p, n, sa, sb in wins if p - GAP <= bad < p + n + GAP), None)
    g, w = int(mx.arena.view(torch.int32)[bad]) & 0xFFFFFFFF, int(mx.want.view(torch.int32)[bad]) & 0xFFFFFFFF
    return f"arena[{bad}] = {g:#010x}, want {w:#010x}; window (p, n, A shift, B shift) = {win}"


# ------------------------------------------------------------------------------------------- the add kernels
def test_every_add_kernel_of_the_tune_library_matches_the_oracle(mx):
    """All 1174: each at its geometry over every shape, on one stream without a host synchronisation in between."""
    lib = capi.tune_lib()
    unlaunchable = [base.kernel_name() for base, t in mx.tunes if t is None]
    assert not unlaunchable, f"no geometry is accepted for {unlaunchable}"
    failures, ran = [], set()
    for _, t in mx.tunes:
        sl = shapes(t, lib)
        gaps = covered(t, sl, mx, lib)
        assert not gaps, f"{t.kernel_name()} {t.as_dict()}: the shapes miss {gaps}"
        err = run_kernel(mx, lib, t, sl)
        if err:
            failures.append(f"{t.kernel_name()} {t.as_dict()}: {err}")
        ran.add(t.kernel_name())
    assert not failures, f"{len(failures)} kernels differ from the oracle:\n" + "\n".join(failures[:20])
    assert ran == add_kernels("tune") and len(ran) == 1174


def test_mixed_phase_runs_the_four_byte_kernel(mx):
    """vadd_scalar_unrolled<4|8|16> at 32 to 1024 threads, and the K4 path that a vec or TMA tune takes when A, B and
    C share no 16-byte phase, over ragged sizes and offsets."""
    lib = capi.tune_lib()
    mixed = [(n, off, 1, 2) for off in range(4) for n in (1, 3, 255, 2048, 2049, 100_003)]
    mixed += [(n, off, 1, 0) for off in (0, 3) for n in (7, 70_001)]
    tunes = [capi.Tune(kind=capi.K4_SCALAR_MLP, threads=th, unroll=u) for u in (4, 8, 16) for th in K4_THREADS]
    tunes += [t for _, t in mx.tunes if t.kind != capi.K4_SCALAR_MLP][::97]
    failures = []
    for t in tunes:
        for n, off, sa, sb in mixed[:2]:
            pa, pb, pc = mx.ptrs(off, sa, sb)
            rc, name, _, block = expected_add_launch(t, n, pa, pb, pc, lib)
            assert rc == capi.OK and name.startswith("vadd_scalar"), (t.as_dict(), name)
            if t.kind not in (capi.K0_SCALAR, capi.K4_SCALAR_MLP):
                assert (name, block) == ("vadd_scalar_unrolled<8>", 256), (t.as_dict(), name, block)
        err = run_kernel(mx, lib, t, mixed)
        if err:
            failures.append(f"{t.as_dict()}: {err}")
    assert not failures, "\n".join(failures[:20])


def alias_tunes(mx):
    """Every tune with .nc loads or early register loads, which plan_launch changes when C is A or B, and a sample
    of the others."""
    out = []
    for i, (_, t) in enumerate(mx.tunes):
        if t.kind in (capi.K1_VEC128, capi.K3_VEC256) and (t.ld_hint == 4 or t.early_loads == 1):
            out.append(t)
        elif i % 29 == 0:
            out.append(t)
    return out


ALIAS_N, ALIAS_OFF = 150_001, 1


def alias_windows():
    (p1, _, _, _), (p2, _, _, _), (p3, _, _, _) = layout([(ALIAS_N, ALIAS_OFF, 0, 0)] * 3)[0]
    return p1, p2, p3


def test_aliased_operands(mx):
    """C == A, C == B and A == B == C, each on a fresh copy of its input, for every tune with .nc loads or early
    register loads and a sample of the others."""
    lib = capi.tune_lib()
    n = ALIAS_N
    (p1, p2, p3), extent = alias_windows(), layout([(n, ALIAS_OFF, 0, 0)] * 3)[1]
    A, B, arena, st = mx.A[0], mx.B[0], mx.arena, mx.stream
    failures = []
    tunes = alias_tunes(mx)
    assert len(tunes) > 512
    with torch.cuda.stream(st):
        for t in tunes:
            mx.expect(((p1, n, "E"), (p2, n, "E"), (p3, n, "EAA")), extent)
            arena[:extent].view(torch.int32).fill_(POISON32)
            arena[p1:p1 + n].copy_(A[p1:p1 + n])
            arena[p2:p2 + n].copy_(B[p2:p2 + n])
            arena[p3:p3 + n].copy_(A[p3:p3 + n])
            c1, c2, c3 = (arena.data_ptr() + 4 * p for p in (p1, p2, p3))
            rcs = [lib.b200va_add_f32_tuned(c1, B.data_ptr() + 4 * p1, c1, n, C.byref(t), st.cuda_stream),
                   lib.b200va_add_f32_tuned(A.data_ptr() + 4 * p2, c2, c2, n, C.byref(t), st.cuda_stream),
                   lib.b200va_add_f32_tuned(c3, c3, c3, n, C.byref(t), st.cuda_stream)]
            assert rcs == [capi.OK] * 3, (t.as_dict(), rcs)
            bad = mx.first_bad(extent)
            if bad >= 0:
                which = "C == A" if bad < p2 - GAP else "C == B" if bad < p3 - GAP else "A == B == C"
                failures.append(f"{t.kernel_name()} {t.as_dict()}: {which}, first bad element {bad}")
    assert not failures, f"{len(failures)} aliased launches differ:\n" + "\n".join(failures[:20])


def test_in_place_launch_is_refused_where_the_swapped_kernel_takes_no_such_block(mx):
    """The kernel plan_launch swaps in when C is A or B can need more registers than the tune's own: the .nc loads
    let ptxas sink them next to their use.  At a CTA size only the tune's own kernel runs, the out-of-place launch
    runs and the in-place one is refused with ERR_VARIANT, as b200va_geometry of the swapped tune says, and writes
    nothing.  (So the matrix above chooses geometries that both kernels take.)"""
    lib = capi.tune_lib()
    cases = []
    for _, t in mx.tunes:
        if t.kind not in (capi.K1_VEC128, capi.K3_VEC256) or not (t.ld_hint == 4 or t.early_loads == 1):
            continue
        for th in THREADS[::-1]:
            c = capi.Tune(**t.as_dict())
            c.threads = th
            if geometry(c, 1 << 20, lib)[0] == capi.OK:
                if geometry(alias_twin(c), 1 << 20, lib)[0] == capi.ERR_VARIANT:
                    cases.append(c)
                break
    assert cases, "every CTA size a .nc or early-load kernel takes fits its swapped kernel too"
    n = ALIAS_N
    (p, _, _, _), extent = layout([(n, ALIAS_OFF, 0, 0)])[0][0], layout([(n, ALIAS_OFF, 0, 0)])[1]
    A, B, arena, st = mx.A[0], mx.B[0], mx.arena, mx.stream
    with torch.cuda.stream(st):
        for t in cases:
            mx.expect(((p, n, "E"),), extent)
            arena[:extent].view(torch.int32).fill_(POISON32)
            arena[p:p + n].copy_(A[p:p + n])
            before = arena[:extent].clone()
            pc = arena.data_ptr() + 4 * p
            rc = lib.b200va_add_f32_tuned(pc, B.data_ptr() + 4 * p, pc, n, C.byref(t), st.cuda_stream)
            assert rc == capi.ERR_VARIANT == expected_add_launch(t, n, pc, B.data_ptr() + 4 * p, pc, lib)[0], \
                (t.as_dict(), rc)
            assert torch.equal(arena[:extent].view(torch.int32), before.view(torch.int32)), t.as_dict()
            assert lib.b200va_add_f32_tuned(*mx.ptrs(p), n, C.byref(t), st.cuda_stream) == capi.OK
            assert mx.first_bad(extent) < 0, t.as_dict()


def test_production_library_runs_its_88_and_refuses_the_rest(mx):
    """Each tune of the matrix through libb200va.so: OK exactly for the 88 kernels it carries, which then match the
    oracle over every shape; ERR_VARIANT from the launch and from b200va_geometry for every other, with nothing
    written and no CUDA error left latched."""
    prod, tune_lib = capi.lib, capi.tune_lib()
    carried = add_kernels("production")
    n, off = 4133, 3
    (wins, extent) = layout([(n, off, 0, 0)])
    p = wins[0][0]
    st = mx.stream
    with torch.cuda.stream(st):
        mx.expect((), extent)
        mx.arena[:extent].view(torch.int32).fill_(POISON32)
        refused = 0
        for _, t in mx.tunes:
            if t.kernel_name() in carried:
                continue
            rc = prod.b200va_add_f32_tuned(*mx.ptrs(p), n, C.byref(t), st.cuda_stream)
            assert rc == capi.ERR_VARIANT and geometry(t, n, prod)[0] == capi.ERR_VARIANT, (t.kernel_name(), rc)
            refused += 1
        bad = mx.first_bad(extent)
    assert refused == 1174 - 88 and bad < 0, (refused, bad)
    # K0 reports cudaGetLastError() after its launch: a refusal that left an error latched would show here
    k0 = capi.Tune(kind=capi.K0_SCALAR)
    assert prod.b200va_add_f32_tuned(*mx.ptrs(p), n, C.byref(k0), st.cuda_stream) == capi.OK
    failures, ran = [], set()
    for _, t in mx.tunes:
        if t.kernel_name() not in carried:
            continue
        assert geometry(t, n, prod) == geometry(t, n, tune_lib), t.kernel_name()
        err = run_kernel(mx, prod, t, shapes(t, prod))
        if err:
            failures.append(f"{t.kernel_name()} {t.as_dict()}: {err}")
        ran.add(t.kernel_name())
    assert not failures, "\n".join(failures[:20])
    assert ran == carried and len(ran) == 88


def test_every_add_kernel_is_launched_as_planned(mx, tmp_path):
    """Under the profiler, per library: each kernel once at its shape with a head and more tiles than CTAs, each K3
    tune at a shape equal mod 16 but not mod 32, the C == A and A == B == C launches of the alias tunes, and the
    mixed-phase path.  Each launch has the name, grid and block of the restated plan, so the trace shows the
    16-byte fallback and plan_launch's swap to plain loads and the L2 prefetch; and the launched vadd_* kernels
    are the library's whole inventory."""
    for lib_name, lib in (("tune", capi.tune_lib()), ("production", capi.lib)):
        carried = add_kernels(lib_name)
        plan = []                                       # (ptrs, n, tune)
        for _, t in mx.tunes:
            if t.kernel_name() not in carried:
                continue
            n, off, sa, sb = shapes(t, lib)[-1]
            plan.append((mx.ptrs(off, sa, sb), n, t))
            if t.kind == capi.K3_VEC256:
                plan.append((mx.ptrs(1, 0, 4), 4133, t))
        for t in alias_tunes(mx) + [t for _, t in mx.tunes if t.kind == capi.K1_VEC128][:3]:
            if t.kernel_name() not in carried:
                continue
            pa, pb, pc = mx.ptrs(ALIAS_OFF)
            plan += [((pc, pb, pc), ALIAS_N, t), ((pc, pc, pc), ALIAS_N, t)]
        plan += [(mx.ptrs(off, 1, 2), 70_001, t) for off, (_, t) in enumerate(mx.tunes[:600:150])]
        want = []
        for (pa, pb, pc), n, t in plan:
            rc, name, grid, block = expected_add_launch(t, n, pa, pb, pc, lib)
            assert rc == capi.OK, (t.as_dict(), rc)
            want.append((name, grid, block))

        def run_plan():
            st = torch.cuda.current_stream().cuda_stream
            for (pa, pb, pc), n, t in plan:
                assert lib.b200va_add_f32_tuned(pa, pb, pc, n, C.byref(t), st) == capi.OK
            torch.cuda.synchronize()

        got = kernels_after_marker(tmp_path, run_plan, ("vadd_",))
        assert len(got) == len(want), (lib_name, len(got), len(want))
        for g, w, (_, n, t) in zip(got, want, plan):
            assert g == w, (lib_name, t.as_dict(), n, g, w)
        launched = {g[0] for g in got}
        assert launched == carried == sass_kernels(lib_name, "vadd_"), (lib_name, sorted(carried - launched)[:8])


# ------------------------------------------------------------------------------------------- STREAM geometry override
STREAM_OVERRIDES = ["96,1,1", "256,2,1", "1024,4,0", "32,4,1", "48,3,1"]
STREAM_OPS, STREAM_DTS = ("copy", "scale", "add", "triad"), ("f32", "f64", "f16", "bf16")
STREAM_PERIOD = 20_011


def _stream_sizes(dtype):
    """(n, element offset of A, B and the vector output, vector path): below 2^19 words, at 2^21 words and more (the
    table's unroll-2 class), and a mixed-phase n."""
    return [(50_001, 1, True), (-(-(1 << 23) // ES[dtype]) + 3, 1, True), (20_003, 1, False)]


def stream_child(tmp):
    """One process under one B200VA_STREAM_GEOMETRY: all 16 op x dtype pairs through libb200va_tune.so, each
    compared with stream_exact at every element with guards; prints each launch's (kernel, grid, block) as JSON."""
    lib = capi.tune_lib()
    env = os.environ.get("B200VA_STREAM_GEOMETRY")
    override = tuple(int(v) for v in env.split(",")) if env else None
    cases = []
    for dtype in STREAM_DTS:
        rng = np.random.default_rng(5)
        if dtype in ("f16", "bf16"):
            pa, pb = (rng.integers(0, 1 << 16, STREAM_PERIOD, dtype=np.uint32).astype(np.uint16) for _ in range(2))
        else:
            pa, pb = X.finite(dtype, STREAM_PERIOD, rng), X.finite(dtype, STREAM_PERIOD, rng)
        s = 0.7001953125 if dtype != "f64" else 0.1
        for op in STREAM_OPS:
            binary = op in ("add", "triad")
            want_block = X.stream(op, dtype, pa, pb if binary else None, s)
            for n, off, vector in _stream_sizes(dtype):
                a, b, want = (tiled(x, n + off, dtype)[off:] for x in (pa, pb, want_block))
                buf, out = poisoned(n, dtype, off if vector else 0)
                head = ((16 - a.data_ptr() % 16) % 16) // ES[dtype]
                if vector:
                    exp = expected_stream_launch(op, dtype, n, head, override)
                else:
                    exp = (f"stream_scalar<{capi.DTYPES[dtype]},{capi.OPS[op]}>", -(-n // 256), 256)
                cases.append((op, dtype, n, a, b if binary else None, out, buf, off if vector else 0, s, want, exp))
    torch.cuda.synchronize()

    def run_plan():
        for op, dtype, n, a, b, out, _, _, s, _, _ in cases:
            rc = lib.b200va_stream(capi.OPS[op], capi.DTYPES[dtype], a.data_ptr(), b.data_ptr() if b is not None else None,
                                   out.data_ptr(), n, s, torch.cuda.current_stream().cuda_stream)
            assert rc == capi.OK, (op, dtype, n, rc)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp, run_plan, ("stream_",))
    assert len(got) == len(cases), (len(got), len(cases))
    for g, (op, dtype, n, _, _, out, buf, off, _, want, exp) in zip(got, cases):
        what = f"{op} {dtype} n={n} under {env}"
        assert g == exp, (what, g, exp)
        assert_matches(out, want, dtype, what, nan_class=op != "copy")
        assert_guards(buf, GUARD + off, n, what)
        print(json.dumps(list(g)))


def test_stream_geometry_override_forms(tmp_path):
    """Each override in a process of its own (the library reads it once): its kernels, grids and blocks are the
    override's plan, and an override the library does not accept gives the table's.  Over all runs the launched
    stream kernels are the tune library's 112."""
    torch.cuda.empty_cache()
    launched = set()
    for ov in STREAM_OVERRIDES:
        d = tmp_path / ov.replace(",", "_")
        d.mkdir()
        code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; "
                "import test_gpu_tune_matrix as m; import pathlib; m.stream_child(pathlib.Path(sys.argv[3]))")
        p = subprocess.run([sys.executable, "-c", code, os.path.join(ROOT, "tests"), ROOT, str(d)], cwd=ROOT,
                           env=dict(os.environ, B200VA_STREAM_GEOMETRY=ov), capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, f"B200VA_STREAM_GEOMETRY={ov}:\n{p.stdout[-3000:]}\n{p.stderr[-6000:]}"
        launched |= {json.loads(line)[0] for line in p.stdout.splitlines() if line.startswith("[")}
    shipped = sass_kernels("tune", "stream_")
    assert len(shipped) == 112 and launched == shipped, (sorted(shipped - launched)[:8], sorted(launched - shipped)[:8])
