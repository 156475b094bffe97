"""b200va_convert_sr_f32 and b200va_quantize_fp8_sr_f32 on the GPU, every byte against oracle/sr_exact.py (NaN
matches NaN as a class).  Outputs are poisoned beforehand and guard elements on both sides must keep the poison.

- Sizes around the group (8 to a 2-byte destination, 16 to FP8) at every element offset of A and C, with first even,
  odd and above 2^32: the vector body with every head, the mixed-phase edge path, both parities of the bits.
- Dense sweeps: every bf16 high half with several low halves; every f16 value with fractional offsets; the FP8
  values, midpoints and saturation band at several k.
- Both sides of the HBM class edge, and n = 2^32 + 4099 with first near 2^40 (windows against the oracle, the rest
  against a second call over the upper part).
- Two calls over [0, m) and [m, n) equal one call; a repeated call and a replayed graph give the same bytes, another
  seed changes some inexact elements; the amax equals b200va_quantize_fp8's on the same input.
- Every rejected argument returns its code and writes nothing.
- A stream op -> SR -> dequantize chain on one stream without a host sync, and an SR tail reading the end of X behind
  the 2^28 K2d writer of test_gpu_pdl_chains.py.
- A profiler trace of the planned kernel, grid and block.
This module's name sorts after test_gpu_parity.py and test_gpu_stream.py, whose traces lose kernels behind a module
with profiler traces that runs before them (DESIGN.md section 3).
"""
import math

import numpy as np
import pytest

from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import sr_exact as S
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import (ES, GUARD, INT, LO, POISON, TORCH, M, _chains, _run, assert_guards, assert_matches,
                             expected_cast_launch, kernels_after_marker, poisoned, tiled, to_dev)
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DESTS = S.DESTS
FP8 = ("e4m3", "e5m2")
G = {"f16": 8, "bf16": 8, "e4m3": 16, "e5m2": 16}
SEED = 0x5EED
PERIOD = 199_999
CHUNK = 1 << 22


# ------------------------------------------------------------------------------------------- helpers
def oracle_sr(a: np.ndarray, dst: str, seed: int, first: int, k: int = 0) -> np.ndarray:
    """The contract's bit patterns, in chunks so that large n stays within host memory."""
    a = np.ascontiguousarray(a, np.float32)
    out = np.empty(a.size, np.uint8 if dst in FP8 else np.uint16)
    for lo in range(0, a.size, CHUNK):
        x = a[lo:lo + CHUNK]
        out[lo:lo + CHUNK] = S.round_sr(x, dst, S.random_words(seed, first + lo, x.size), k)
    return out


def sr(a, dst, out, seed=SEED, first=0, k=0, **kw):
    if dst in FP8:
        return va.quantize_fp8_sr(a, TORCH[dst], seed=seed, offset=first, scale_exp=k, out=out, **kw)
    assert k == 0
    return va.convert_sr(a, TORCH[dst], seed=seed, offset=first, out=out, **kw)


def check(a_host, a_dev, dst, seed, first, k=0, off_c=0, what=""):
    n = a_host.size
    buf, out = poisoned(n, dst, off_c)
    sr(a_dev, dst, out, seed, first, k)
    torch.cuda.synchronize()
    assert_matches(out, to_dev(oracle_sr(a_host, dst, seed, first, k), dst), dst, what)
    assert_guards(buf, GUARD + off_c, n, what)


def random_f32(n, rng):
    return V.random_bits("f32", n, rng)


def k_of(dst):
    return 3 if dst in FP8 else 0


# ------------------------------------------------------------------------------------------- element offsets
@pytest.mark.parametrize("dst", DESTS)
def test_sizes_around_the_group_at_every_offset(dst):
    sizes = sorted({0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 33, 47, 4099, 70_001})
    rng = np.random.default_rng([DESTS.index(dst), 1])
    total = max(sizes) + 4
    host = random_f32(total, rng)
    k = k_of(dst)
    abuf = torch.empty(GUARD + total + GUARD, dtype=torch.float32, device="cuda")
    abuf[GUARD:GUARD + total] = to_dev(host, "f32")
    for first in (0, 1, (1 << 32) + 5):
        for oa in range(4):
            want_all = oracle_sr(host[oa:oa + max(sizes)], dst, SEED, first, k)
            for oc in range(16 // ES[dst]):
                for n in sizes:
                    a, what = abuf[GUARD + oa:GUARD + oa + n], f"{dst} n={n} first={first} offsets A {oa} C {oc}"
                    buf, out = poisoned(n, dst, oc)
                    sr(a, dst, out, SEED, first, k)
                    torch.cuda.synchronize()
                    assert_matches(out, to_dev(want_all[:n], dst), dst, what)
                    assert_guards(buf, GUARD + oc, n, what)


# ------------------------------------------------------------------------------------------- dense sweeps
def test_every_bf16_high_half_with_several_low_halves():
    hi = np.arange(1 << 16, dtype=np.uint32) << 16
    rng = np.random.default_rng(2)
    lows = [0, 1, 0x7FFF, 0x8000, 0x8001, 0xFFFF, int(rng.integers(1, 0xFFFF))]
    a = np.concatenate([hi | np.uint32(lo) for lo in lows]).view(np.float32)
    for seed, first in ((1, 0), (2, 7), (SEED, (1 << 40) + 1)):
        for off_c in (0, 3):
            check(a, to_dev(a, "f32"), "bf16", seed, first, 0, off_c, f"bf16 sweep seed {seed} first {first} C {off_c}")


def test_every_f16_value_with_fractional_offsets():
    with np.errstate(invalid="ignore"):
        x = X.widen(np.arange(1 << 16, dtype=np.uint16), "f16").astype(np.float32)
    base = x.view(np.uint32)
    offs = [0, 1, 1 << 12, (1 << 13) - 1, 0x1555]
    a = np.concatenate([base + np.uint32(o) for o in offs]).view(np.float32)   # between the f16 value and the next
    for seed, first in ((1, 0), (3, 1)):
        for off_c in (0, 5):
            check(a, to_dev(a, "f32"), "f16", seed, first, 0, off_c, f"f16 sweep seed {seed} first {first} C {off_c}")


@pytest.mark.parametrize("fmt", FP8)
def test_fp8_values_midpoints_and_saturation_band(fmt):
    v, m = F.values(fmt), F.midpoints(fmt)
    top = F.MAX_FINITE[fmt]
    rng = np.random.default_rng(F.FORMATS8.index(fmt))
    band = np.concatenate([top * (1 + rng.random(200) * 0.2), [top, m[-1], 2 * top, 1e30, np.inf]])
    between = (v[:-1, None] + (v[1:] - v[:-1])[:, None] * rng.random((v.size - 1, 7))).ravel()
    x = np.concatenate([v, m, between, band])
    x = np.concatenate([x, -x, [np.nan, 0.0, -0.0]])
    for k in (-126, -8, 0, 5, 126):
        with np.errstate(all="ignore"):
            a = np.ldexp(x, -k).astype(np.float32)                  # products a 2^k, past f32's range where k < 0
        for first in (0, 1):
            check(a, to_dev(a, "f32"), fmt, SEED + k, first, k, first, f"{fmt} k={k} first {first}")


# ------------------------------------------------------------------------------------------- size classes
@pytest.mark.parametrize("dst", DESTS)
def test_both_sides_of_the_hbm_edge(dst):
    """n = h - 1 and h at aligned pointers, then h + 37 with A and C one element past a 16-byte boundary; h = 2^25,
    where the f32 source reaches the HBM class."""
    h = 1 << 25
    big = h + 37
    block = random_f32(PERIOD, np.random.default_rng([9, DESTS.index(dst)]))
    host = np.tile(block, -(-(big + 1) // PERIOD))[:big + 1]
    a = tiled(block, big + 1, "f32")
    k = k_of(dst)
    first = 12345
    want = to_dev(oracle_sr(host, dst, SEED, first, k), dst)          # element i of A has the global index first + i
    for n, off in ((h - 1, 0), (h, 0), (big, 1)):
        what = f"{dst} n={n} offset {off}"
        buf, out = poisoned(n, dst, off)
        sr(a[off:off + n], dst, out, SEED, first + off, k)
        torch.cuda.synchronize()
        assert_matches(out, want[off:off + n], dst, what)
        assert_guards(buf, GUARD + off, n, what)
        del buf, out


@pytest.mark.parametrize("dst", ["bf16", "e5m2"])
def test_beyond_32_bit_offsets_with_first_near_2_40(dst):
    """n = 2^32 + 4099 with first = 2^40 - 3: windows around element 2^31 (byte 2^32 of a 2-byte C), 2^32 and the end
    against the oracle; all of it against a call over [m, n) with first + m and a call over [0, m)."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 4 * n + 3 * ES[dst] * n + (4 << 30):
        pytest.skip("needs ~45 GiB of free device memory")
    first = (1 << 40) - 3
    k = k_of(dst)
    block = random_f32(PERIOD, np.random.default_rng(31))
    a = tiled(block, n, "f32")
    c = torch.empty(n * ES[dst], dtype=torch.uint8, device="cuda").view(TORCH[dst])
    sr(a, dst, c, SEED, first, k)
    for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - 8192):
        x = np.tile(block, 2 * (8192 // PERIOD + 2))
        start = lo % PERIOD
        win = x[start:start + 8192]
        assert_matches(c[lo:lo + 8192], to_dev(oracle_sr(win, dst, SEED, first + lo, k), dst), dst, f"window at {lo}")
    m = (1 << 32) - 77
    parts = torch.empty_like(c)
    sr(a[:m], dst, parts[:m], SEED, first, k)
    sr(a[m:], dst, parts[m:], SEED, first + m, k)
    torch.cuda.synchronize()
    assert_matches(parts, c, dst, "two calls against one, n = 2^32 + 4099")


# ------------------------------------------------------------------------------------------- reproducibility
@pytest.mark.parametrize("dst", DESTS)
def test_two_calls_equal_one_call(dst):
    n = 300_007
    host = random_f32(n, np.random.default_rng([5, DESTS.index(dst)]))
    a = to_dev(host, "f32")
    k = k_of(dst)
    for first in (0, 3, (1 << 64) - 1000, (1 << 64) - 1003):        # groups of 16 and of 8 across 2^64
        whole = torch.empty(n * ES[dst], dtype=torch.uint8, device="cuda").view(TORCH[dst])
        sr(a, dst, whole, SEED, first, k)
        assert_matches(whole, to_dev(oracle_sr(host, dst, SEED, first, k), dst), dst, f"{dst} first {first}")
        for m in (1, 5, G[dst], 1001, n - 3):
            parts = torch.empty_like(whole)
            sr(a[:m], dst, parts[:m], SEED, first, k)
            sr(a[m:], dst, parts[m:], SEED, (first + m) % (1 << 64), k)
            torch.cuda.synchronize()
            assert_matches(parts, whole, dst, f"{dst} first {first} split at {m}")


def test_repeats_and_graph_replays_give_the_same_bytes_and_another_seed_differs():
    n = 100_003
    rng = np.random.default_rng(7)
    host = (rng.standard_normal(n) * 300).astype(np.float32)
    a = to_dev(host, "f32")
    outs = {d: poisoned(n, d, 1) for d in DESTS}
    amax = torch.zeros(1, dtype=torch.float64, device="cuda")
    wants = {d: to_dev(oracle_sr(host, d, SEED, 11, k_of(d)), d) for d in DESTS}
    for d in DESTS:
        for _ in range(2):
            sr(a, d, outs[d][1], SEED, 11, k_of(d))
            torch.cuda.synchronize()
            assert_matches(outs[d][1], wants[d], d, f"{d} repeated")
        other = torch.empty_like(outs[d][1])
        sr(a, d, other, SEED + 1, 11, k_of(d))
        torch.cuda.synchronize()
        differ = other.view(INT[d]) != wants[d].view(INT[d])
        assert 0 < int(differ.sum()) < n, (d, int(differ.sum()))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            amax.zero_()
            for d in DESTS:
                sr(a, d, outs[d][1], SEED, 11, k_of(d), **({"amax": amax} if d == "e4m3" else {}))
    torch.cuda.synchronize()
    for r in range(2):
        for d in DESTS:
            outs[d][0].view(torch.uint8).fill_(POISON)
        amax.fill_(1e300)
        g.replay()
        torch.cuda.synchronize()
        for d in DESTS:
            assert_matches(outs[d][1], wants[d], d, f"{d} graph replay {r}")
            assert_guards(outs[d][0], GUARD + 1, n, f"{d} graph replay {r}")
        assert float(amax.item()) == F.amax(host, "f32")


def test_amax_equals_quantize_fp8s():
    rng = np.random.default_rng(8)
    finite = (rng.standard_normal(300_007) * 50).astype(np.float32)
    edges = X.edge_values("f32", 300_007, 3)
    with_nan = finite.copy()
    with_nan[123_457] = np.nan
    for name, x in (("finite", finite), ("value classes", edges), ("one NaN", with_nan),
                    ("-0", np.array([-0.0, -0.0], np.float32))):
        a = to_dev(x, "f32")
        for fmt in FP8:
            m_sr, m_rn = (torch.zeros(1, dtype=torch.float64, device="cuda") for _ in range(2))
            q = torch.empty(x.size, dtype=TORCH[fmt], device="cuda")
            va.quantize_fp8_sr(a, TORCH[fmt], seed=1, scale_exp=4, amax=m_sr, out=q)
            va.quantize_fp8(a, TORCH[fmt], scale_exp=4, amax=m_rn, out=torch.empty_like(q))
            torch.cuda.synchronize()
            got, want = float(m_sr.item()), float(m_rn.item())
            assert (math.isnan(got) and math.isnan(want)) or \
                np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (name, fmt, got, want)
            assert_matches(q, to_dev(oracle_sr(x, fmt, 1, 0, 4), fmt), fmt, f"{name} {fmt}")


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A, n = buf.data_ptr() + 4096, 1000
    C_, M_ = A + 16384, A + 32768
    F16, BF16 = capi.DTYPES["f16"], capi.DTYPES["bf16"]
    E4, E5 = capi.F8_E4M3, capi.F8_E5M2
    conv = [
        ((A, 0, C_, n), capi.ERR_VARIANT), ((A, 1, C_, n), capi.ERR_VARIANT), ((A, 4, C_, n), capi.ERR_VARIANT),
        ((A, -1, C_, n), capi.ERR_VARIANT),
        ((None, BF16, C_, n), capi.ERR_INVALID), ((A, F16, None, n), capi.ERR_INVALID),
        ((A, BF16, C_, (1 << 40) + 1), capi.ERR_INVALID),
        ((A + 2, F16, C_, n), capi.ERR_ALIGN), ((A, BF16, C_ + 1, n), capi.ERR_ALIGN),
        ((A, F16, A, n), capi.ERR_OVERLAP), ((A, BF16, A + 4 * n - 2, n), capi.ERR_OVERLAP),
        ((A + 8, F16, A - 2 * n + 10, n), capi.ERR_OVERLAP),
    ]
    quant = [
        ((A, 2, C_, n, 0, M_), capi.ERR_VARIANT), ((A, -1, C_, n, 0, M_), capi.ERR_VARIANT),
        ((A, E4, C_, n, 127, M_), capi.ERR_INVALID), ((A, E5, C_, n, -127, M_), capi.ERR_INVALID),
        ((None, E4, C_, n, 0, M_), capi.ERR_INVALID), ((A, E5, None, n, 0, M_), capi.ERR_INVALID),
        ((A, E4, C_, (1 << 40) + 1, 0, M_), capi.ERR_INVALID),
        ((A + 2, E4, C_, n, 0, M_), capi.ERR_ALIGN), ((A, E4, C_, n, 0, M_ + 4), capi.ERR_ALIGN),
        ((A, E4, A, n, 0, M_), capi.ERR_OVERLAP), ((A, E5, A + 4 * n - 1, n, 0, M_), capi.ERR_OVERLAP),
        ((A, E4, C_, n, 0, A + 8), capi.ERR_OVERLAP), ((A, E4, C_, n, 0, C_ + n - 8), capi.ERR_OVERLAP),
    ]
    for args, code in conv:
        assert L.b200va_convert_sr_f32(*args, 1, 0, None) == code, (args, code)
    for args, code in quant:
        assert L.b200va_quantize_fp8_sr_f32(*args[:5], 1, 0, args[5], None) == code, (args, code)
    assert L.b200va_convert_sr_f32(None, F16, None, 0, 1, 0, None) == capi.OK
    assert L.b200va_quantize_fp8_sr_f32(A, E4, C_, 0, 0, 1, 0, M_, None) == capi.OK
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == POISON).all(), "a rejected or empty call wrote to device memory"
    with pytest.raises(TypeError):
        va.convert_sr(torch.zeros(8, dtype=torch.float64, device="cuda"), "bf16", seed=1)
    with pytest.raises(TypeError):
        va.quantize_fp8_sr(torch.zeros(8, dtype=torch.float16, device="cuda"), "e4m3", seed=1)
    with pytest.raises(TypeError):
        va.convert_sr(torch.zeros(8, dtype=torch.float32, device="cuda"), "f64", seed=1)


# ------------------------------------------------------------------------------------------- stream order
def test_stream_op_sr_dequantize_chain_on_one_stream():
    """Rounds on one stream without a host sync: b = s a (b200va_stream), q = SR(b) to E4M3 with amax and
    c = dequantize(q); h = SR(b) to bf16 and d = h / 2 (b200va_stream); a different s and first per round, ten rounds
    at an L2-resident size and three in the HBM class."""
    st = torch.cuda.Stream()
    period = 49_999
    a0 = (np.random.default_rng(10).standard_normal(period) * 8).astype(np.float32)
    k = 4
    for n, rounds in (((1 << 20) + 5, 10), ((1 << 25) + 5, 3)):
        scalars = [1.0 + r / 8 for r in range(rounds)]
        host = np.tile(a0, -(-n // period))[:n]
        a = tiled(a0, n, "f32")
        b = torch.empty_like(a)
        q = torch.empty(n, dtype=torch.float8_e4m3fn, device="cuda")
        h = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        cs = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in scalars]
        ds = [torch.empty(n, dtype=torch.bfloat16, device="cuda") for _ in scalars]
        ms = torch.zeros(len(scalars), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        for r, s in enumerate(scalars):
            va.stream("scale", a, None, b, scalar=s, stream=st)
            va.quantize_fp8_sr(b, torch.float8_e4m3fn, seed=SEED, offset=r, scale_exp=k, amax=ms[r:r + 1], out=q, stream=st)
            va.dequantize_fp8(q, torch.float32, scale_exp=k, out=cs[r], stream=st)
            va.convert_sr(b, torch.bfloat16, seed=SEED, offset=r, out=h, stream=st)
            va.stream("scale", h, None, ds[r], scalar=0.5, stream=st)
        st.synchronize()
        for r, s in enumerate(scalars):
            hb = X.stream("scale", "f32", host, None, s)
            c_want = F.dequantize(oracle_sr(hb, "e4m3", SEED, r, k), "e4m3", "f32", k)
            d_want = X.stream("scale", "bf16", oracle_sr(hb, "bf16", SEED, r), None, 0.5)
            assert_matches(cs[r], to_dev(c_want, "f32"), "f32", f"n={n} round {r}: dequantize(SR(b))")
            assert_matches(ds[r], to_dev(d_want, "bf16"), "bf16", f"n={n} round {r}: SR(b) / 2")
            assert float(ms[r].item()) == F.amax(hb, "f32"), (n, r)
        del a, b, q, h, cs, ds


def test_sr_tail_reads_what_the_writer_wrote(env):
    """test_gpu_pdl_chains.py's chains (the 2^28 K2d writer of X, then 0-3 middle launches) with an SR quantize of
    the end of X, with amax, as the tail; then the same with an SR convert to bf16."""
    middles, chains = _chains(env)
    q = torch.empty(M + 1, dtype=torch.float8_e4m3fn, device="cuda")[1:]
    h = torch.empty(M + 1, dtype=torch.bfloat16, device="cuda")[1:]
    m = torch.zeros(1, dtype=torch.float64, device="cuda")
    want_q = oracle_sr(env["ref_window"], "e4m3", SEED, LO, 2)
    want_h = oracle_sr(env["ref_window"], "bf16", SEED, LO)
    want_amax = F.amax(env["ref_window"], "f32")

    def tail_q(w):
        m.zero_()
        va.quantize_fp8_sr(w, torch.float8_e4m3fn, seed=SEED, offset=LO, scale_exp=2, amax=m, out=q)

    def tail_h(w):
        va.convert_sr(w, torch.bfloat16, seed=SEED, offset=LO, out=h)

    failures = []
    for names in chains:
        q.view(torch.uint8).fill_(POISON)
        _run(env, middles, names, tail_q)
        bad = np.flatnonzero(q.view(torch.uint8).cpu().numpy() != want_q)
        amax = float(m.item())
        if bad.size or amax != want_amax:
            failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> SR quantize: {bad.size} bytes differ, "
                            f"amax {amax!r} want {want_amax!r}")
        h.view(torch.uint8).fill_(POISON)
        _run(env, middles, names, tail_h)
        bad = np.flatnonzero(h.view(torch.int16).cpu().numpy().view(np.uint16) != want_h)
        if bad.size:
            failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> SR convert: {bad.size} elements differ")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------- trace
def test_trace_shows_the_planned_kernel(tmp_path):
    """Per destination: n = 1000, the HBM class, n = 1001 in mixed phase and an odd n with a head.  Under the
    profiler the kernels after the marker are exactly the planned ones with their grid and block."""
    h = 1 << 25
    src = torch.zeros(h + 64, dtype=torch.float32, device="cuda")
    outs = {d: torch.zeros((h + 64) * ES[d], dtype=torch.uint8, device="cuda").view(TORCH[d]) for d in DESTS}
    plan, want = [], []
    for d in DESTS:
        for n, oa, oc in ((1000, 0, 0), (h, 0, 0), (1001, 0, 1), (4099, 1, 1)):
            a, c = src[oa:oa + n], outs[d][oc:oc + n]
            plan.append((d, a, c))
            want.append(expected_cast_launch("sr_cast_vec", 4, ES[d], n, a.data_ptr(), c.data_ptr()))
    amax = torch.zeros(1, dtype=torch.float64, device="cuda")

    def run_plan():
        for d, a, c in plan:
            sr(a, d, c, SEED, 0, k_of(d), **({"amax": amax} if d in FP8 else {}))
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("sr_cast_vec",))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w, p in zip(got, want, plan):
        assert g == w, (p[0], g, w)
