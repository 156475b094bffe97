"""b200va_quantize_mxfp8 and b200va_dequantize_mxfp8 on the GPU: every byte of C and of the scales S against
oracle/mxfp8_exact.py (NaN matches NaN as a class in C; S is compared exactly).  C and S are poisoned beforehand and
guard bytes on both sides of each must keep the poison.

- Every (type, format, block, rule) at ragged n around the block, the group of 16 and the tile edges.
- Every element offset of A and C within 16 bytes, with S at odd addresses: the vector body (both on a 16-byte
  boundary) and the edge path give the same bytes for the same values, and both match the oracle.
- The named sets of `mxfp8_exact.named_blocks`; all 65536 f16 and bf16 patterns, in order and permuted so that blocks
  mix magnitudes.
- Both sides of the HBM class per type and direction and a ragged, misaligned n in it; f16 -> E4M3 -> f16 at
  n = 2^32 + 4099.
- Dequantize of all 256 patterns under the scale bytes 0, 1, 126, 127, 128, 254 and 255 into every type; quantize ->
  dequantize; a change in one block leaves every other block's bytes alone.
- Every rejected argument writes nothing.
- A stream op -> quantize -> dequantize -> stream op chain on one stream without a host sync; a captured graph
  replayed; a quantize tail reading the end of X behind the 2^28 K2d writer of test_gpu_pdl_chains.py.
- A profiler trace of the planned kernels, grids and blocks.
This module's name sorts after test_gpu_typecast_fp8.py: a module with profiler traces that runs before the parity
and stream modules makes their traces lose kernels (DESIGN.md section 3).
"""
import numpy as np
import pytest

from conftest import has_gpu
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import mxfp8_exact as MX
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import (DT_CODE, ES, F8_CODE, GUARD, LO, POISON, TORCH, M, _chains, _run, assert_guards,
                             assert_matches, expected_mx_launch, hbm_n, kernels_after_marker, poisoned, tiled, to_dev)
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

DTYPES = V.DTYPES
FMTS = F.FORMATS8
COMBOS = [(t, f, b, r) for t in DTYPES for f in FMTS for b in MX.BLOCKS for r in MX.RULES]
PERIOD = 128 * 1563                       # a whole number of blocks, so a repeated period repeats its reference
SCALE_BYTES = (0, 1, 126, 127, 128, 254, 255)


# ------------------------------------------------------------------------------------------- helpers
def quantize(a, fmt, block, rule, out, scales, **kw):
    return va.quantize_mxfp8(a, TORCH[fmt], block=block, scale_rule=rule, out=out, scales=scales, **kw)


def dequantize(q, scales, dst, block, out, **kw):
    return va.dequantize_mxfp8(q, scales, TORCH[dst], block=block, out=out, **kw)


def check_quant(src, fmt, block, rule, a_host, a_dev, off_c=0, off_s=0, what=""):
    """Quantize a_dev into poisoned C and S at the given offsets; compare both with the reference of a_host.  Returns
    (q, s) as uint8 device tensors."""
    n = a_host.size
    bq, q = poisoned(n, fmt, off_c)
    bs, s = poisoned(MX.scale_count(n, block), "u8", off_s)
    quantize(a_dev, fmt, block, rule, q, s)
    torch.cuda.synchronize()
    wq, ws = MX.quantize(a_host, src, fmt, block, rule)
    assert_matches(q, to_dev(wq, fmt), fmt, what)
    assert_matches(s, to_dev(ws, "u8"), "u8", what, nan_class=False)
    assert_guards(bq, GUARD + off_c, n, what)
    assert_guards(bs, GUARD + off_s, s.numel(), what + " (scales)")
    return q.view(torch.uint8), s


def check_dequant(fmt, dst, block, bits, scales, q_dev, s_dev, off_c=0, what=""):
    n = bits.size
    buf, out = poisoned(n, dst, off_c)
    dequantize(q_dev, s_dev, dst, block, out)
    torch.cuda.synchronize()
    assert_matches(out, to_dev(MX.dequantize(bits, scales, fmt, dst, block), dst), dst, what)
    assert_guards(buf, GUARD + off_c, n, what)


def random_fp8(n, rng):
    return rng.integers(0, 256, n, dtype=np.uint16).astype(np.uint8)


def random_scales(count, rng):
    """Scale bytes around 127 (so f16 results stay in range), with the extremes and 0xFF at every 17th block."""
    s = rng.integers(110, 145, count).astype(np.uint8)
    s[::17] = np.resize(np.array(SCALE_BYTES, np.uint8), s[::17].size)
    return s


def at_offset(x_dev, off, torch_dtype):
    """A copy of x_dev `off` elements past a 16-byte boundary."""
    buf = torch.empty(x_dev.numel() + 16, dtype=torch_dtype, device="cuda")
    base = (-buf.data_ptr() % 16) // buf.element_size()
    v = buf[base + off:base + off + x_dev.numel()]
    v.view(torch.uint8).copy_(x_dev.view(torch.uint8))
    return v


# ------------------------------------------------------------------------------------------- sizes and offsets
@pytest.mark.parametrize("t,fmt,block,rule", COMBOS)
def test_ragged_sizes_around_block_group_and_tile_edges(t, fmt, block, rule):
    sizes = sorted({0, 1, 15, 16, 17, block - 1, block, block + 1, 2 * block + 5, 4096 - 1, 4096, 4096 + 17,
                    4096 + block + 1, 8192 - block, 8192 + 33, 70_001})
    rng = np.random.default_rng([DT_CODE[t], F8_CODE[fmt], block, rule == "ocp"])
    host = np.concatenate([V.random_bits(t, 40_000, rng), X.finite(t, 40_000, rng, 3.0)])
    rng.shuffle(host)
    a = to_dev(host, t)
    bits, sc = random_fp8(max(sizes), rng), random_scales(MX.scale_count(max(sizes), block), rng)
    for n in sizes:
        check_quant(t, fmt, block, rule, host[:n], a[:n], 0, 0, f"quantize {t}->{fmt} block {block} {rule} n={n}")
        if rule == "ocp":
            nb = MX.scale_count(n, block)
            check_dequant(fmt, t, block, bits[:n], sc[:nb], to_dev(bits[:n], fmt), to_dev(sc[:nb], "u8"), 0,
                          f"dequantize {fmt}->{t} block {block} n={n}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("t", DTYPES)
def test_every_offset_gives_the_bytes_of_offset_zero(t, fmt):
    """The same values at every element offset of A and of C within 16 bytes and S at offsets 0..3: only (0, 0) takes
    the vector body; every other placement must give its bytes, which are the oracle's."""
    rng = np.random.default_rng([3, DT_CODE[t], F8_CODE[fmt]])
    for block, rule, n in ((32, "ocp", 4099), (128, "nosat", 1157), (64, "ocp", 33)):
        host = np.concatenate([V.random_bits(t, n // 2, rng), X.finite(t, n - n // 2, rng, 2.0)])
        rng.shuffle(host)
        a0 = to_dev(host, t)
        what = f"quantize {t}->{fmt} block {block} {rule} n={n}"
        q0, s0 = check_quant(t, fmt, block, rule, host, a0, 0, 0, what)
        for oa in range(16 // ES[t]):
            a = at_offset(a0, oa, TORCH[t])
            for oc in range(16):
                q, s = check_quant(t, fmt, block, rule, host, a, oc, (oa + oc) % 4, f"{what} offsets A {oa} C {oc}")
                assert torch.equal(q, q0) and torch.equal(s, s0), f"{what} offsets A {oa} C {oc}: not the bytes of offset 0"
        bits, sc = random_fp8(n, rng), random_scales(MX.scale_count(n, block), rng)
        want = to_dev(MX.dequantize(bits, sc, fmt, t, block), t)
        q0 = to_dev(bits, fmt)
        for oa in range(16):
            q = at_offset(q0, oa, TORCH[fmt])
            s = at_offset(to_dev(sc, "u8"), 1 + oa % 3, torch.uint8)
            for oc in range(16 // ES[t]):
                what = f"dequantize {fmt}->{t} block {block} n={n} offsets A {oa} C {oc}"
                buf, out = poisoned(n, t, oc)
                dequantize(q, s, t, block, out)
                torch.cuda.synchronize()
                assert_matches(out, want, t, what)
                assert_guards(buf, GUARD + oc, n, what)


# ------------------------------------------------------------------------------------------- named and exhaustive
@pytest.mark.parametrize("t,fmt,block,rule", COMBOS)
def test_named_sets(t, fmt, block, rule):
    sets = MX.named_blocks(t, fmt, block)
    host = np.concatenate(list(sets.values()))
    a = to_dev(host, t)
    q, s = check_quant(t, fmt, block, rule, host, a, 0, 0, f"{t}->{fmt} block {block} {rule} named sets")
    assert not bool((s == 0xFF).any())
    q1, s1 = check_quant(t, fmt, block, rule, host, at_offset(a, 1, TORCH[t]), 3, 1, f"{t}->{fmt} block {block} {rule} named sets, edge path")
    assert torch.equal(q, q1) and torch.equal(s, s1)
    # back into the source type: the FP8 values scaled back, rounded once
    qh, sh = q.cpu().numpy(), s.cpu().numpy()
    check_dequant(fmt, t, block, qh, sh, q.view(TORCH[fmt]), s, 0, f"{fmt}->{t} block {block} named sets back")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("src", ["f16", "bf16"])
def test_every_16_bit_pattern(src, fmt):
    """In order (blocks of neighbouring magnitudes, NaN-only and inf blocks included) and permuted (blocks that mix
    every magnitude with NaNs and infinities)."""
    x = np.arange(1 << 16, dtype=np.uint16)
    for name, host in (("in order", x), ("permuted", np.random.default_rng(7).permutation(x))):
        a = to_dev(host, src)
        for block in MX.BLOCKS:
            for rule in MX.RULES:
                check_quant(src, fmt, block, rule, host, a, 0, 0, f"{src}->{fmt} all patterns {name}, block {block} {rule}")
        check_quant(src, fmt, 32, "ocp", host, a, 1, 1, f"{src}->{fmt} all patterns {name}, C offset 1")


@pytest.mark.parametrize("dst", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
def test_every_fp8_pattern_under_the_extreme_scale_bytes(fmt, dst):
    """7168 elements: every pattern meets every one of the scale bytes (256 / block and 7 are coprime)."""
    bits = np.tile(np.arange(256, dtype=np.uint8), 28)
    q = to_dev(bits, fmt)
    for block in MX.BLOCKS:
        sc = np.resize(np.array(SCALE_BYTES, np.uint8), bits.size // block)
        s = to_dev(sc, "u8")
        for off_c in (0, 1):
            check_dequant(fmt, dst, block, bits, sc, q, s, off_c, f"{fmt}->{dst} all patterns, block {block}, C offset {off_c}")
    sc = np.full(bits.size // 32, 0xFF, np.uint8)
    out = dequantize(q, to_dev(sc, "u8"), dst, 32, None)
    assert bool(torch.isnan(out).all())


@pytest.mark.parametrize("fmt", FMTS)
def test_round_trip_and_unrelated_blocks(fmt):
    rng = np.random.default_rng(F8_CODE[fmt] + 11)
    finite = np.flatnonzero(np.isfinite(F.DECODE[fmt])).astype(np.uint8)
    for block in MX.BLOCKS:
        nb = 300
        # FP8 values times one power of two per block come back exactly (NOSAT never saturates them)
        a = np.ldexp(F.DECODE[fmt][rng.choice(finite, nb * block)], np.repeat(rng.integers(-90, 90, nb), block))
        for src in ("f64", "f32"):
            host = a.astype(X.STORAGE[src])
            q, s = va.quantize_mxfp8(to_dev(host, src), TORCH[fmt], block=block, scale_rule="nosat")
            back = va.dequantize_mxfp8(q, s, TORCH[src], block=block)
            torch.cuda.synchronize()
            assert_matches(back, to_dev(host, src), src, f"round trip {src} {fmt} block {block}", nan_class=False)
        # a change in one block changes that block's bytes and scale only
        host = X.finite("bf16", nb * block + 7, rng, 2.0)
        other = host.copy()
        k = 137
        other[k * block + 5] = V.round_f64(np.array([-6.0e4]), "bf16")[0]
        (q0, s0), (q1, s1) = (check_quant("bf16", fmt, block, "ocp", h, to_dev(h, "bf16"), 0, 0, "unrelated blocks") for h in (host, other))
        keep = torch.ones(q0.numel(), dtype=torch.bool, device="cuda")
        keep[k * block:(k + 1) * block] = False
        assert torch.equal(q0[keep], q1[keep]) and not torch.equal(q0[~keep], q1[~keep])
        assert torch.equal(torch.cat([s0[:k], s0[k + 1:]]), torch.cat([s1[:k], s1[k + 1:]])) and int(s1[k]) > int(s0[k])


# ------------------------------------------------------------------------------------------- size classes
def _periodic_quant_want(host, t, fmt, block, rule, off, n):
    """The reference of quantizing tiled(host)[off:off + n]: the period's reference from its element `off` on,
    repeated, with the short last block computed from the elements it really holds."""
    rolled = np.roll(host, -off)
    wq, ws = MX.quantize(rolled, t, fmt, block, rule)
    q = tiled(wq, n, fmt).view(torch.uint8).clone()
    s = to_dev(ws, "u8")
    nb = MX.scale_count(n, block)
    s = s.repeat(-(-nb // s.numel()))[:nb].clone()
    tail = n - n % block
    if tail < n:
        tq, ts = MX.quantize(rolled[np.arange(tail, n) % host.size], t, fmt, block, rule)
        q[tail:] = to_dev(tq, "u8")
        s[-1] = int(ts[0])
    return q.view(TORCH[fmt]), s


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("t", DTYPES)
@pytest.mark.parametrize("kind", ["q", "d"])
def test_both_sides_of_the_hbm_edge(kind, t, fmt):
    """n = h - 1 and h at aligned pointers (h - 1 ends in a short block), then h + 37 with A and C one element past a
    16-byte boundary (the edge path at full size)."""
    h = hbm_n(ES[t])
    big = h + 37
    block, rule = (32, "ocp") if fmt == "e4m3" else (128, "nosat")
    rng = np.random.default_rng([9, DT_CODE[t], F8_CODE[fmt], kind == "q"])
    if kind == "q":
        host = np.concatenate([V.random_bits(t, PERIOD // 2, rng), X.finite(t, PERIOD // 2, rng, 2.0)])
        a = tiled(host, big + 1, t)
    else:
        host, sc = random_fp8(PERIOD, rng), random_scales(PERIOD // block, rng)
        a = tiled(host, big + 1, fmt)
    for n, off in ((h - 1, 0), (h, 0), (big, 1)):
        what = f"{kind} {t} {fmt} block {block} n={n} offset {off}"
        nb = MX.scale_count(n, block)
        if kind == "q":
            bq, q = poisoned(n, fmt, off)
            bs, s = poisoned(nb, "u8", off)
            quantize(a[off:off + n], fmt, block, rule, q, s)
            torch.cuda.synchronize()
            wq, ws = _periodic_quant_want(host, t, fmt, block, rule, off, n)
            assert_matches(q, wq, fmt, what)
            assert_matches(s, ws, "u8", what, nan_class=False)
            assert_guards(bq, GUARD + off, n, what)
            assert_guards(bs, GUARD + off, nb, what + " (scales)")
            del bq, q, wq
        else:
            # the view starts at element `off` of the period; its blocks start there too, with the period's scales
            rolled = np.roll(host, -off)
            want = tiled(MX.dequantize(rolled, sc, fmt, t, block), n, t)
            s = to_dev(sc, "u8")
            s = s.repeat(-(-nb // s.numel()))[:nb].contiguous()
            buf, out = poisoned(n, t, off)
            dequantize(a[off:off + n], s, t, block, out)
            torch.cuda.synchronize()
            assert_matches(out, want, t, what)
            assert_guards(buf, GUARD + off, n, what)
            del buf, out, want


def test_f16_e4m3_f16_beyond_32_bit_offsets():
    """n = 2^32 + 4099, block 32: element 2^32 needs a 64-bit index, and so does its block's scale."""
    n = (1 << 32) + 4099
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * 2 * n + 2 * n + (5 << 30):
        pytest.skip("needs ~29 GiB of free device memory")
    rng = np.random.default_rng(31)
    host = np.concatenate([V.random_bits("f16", PERIOD // 2, rng), X.finite("f16", PERIOD // 2, rng, 2.0)])
    a = tiled(host, n, "f16")
    q = torch.empty(n, dtype=torch.uint8, device="cuda")
    q.fill_(POISON)
    bs, s = poisoned(MX.scale_count(n, 32), "u8")
    quantize(a, "e4m3", 32, "ocp", q.view(torch.float8_e4m3fn), s)
    del a
    wq, ws = _periodic_quant_want(host, "f16", "e4m3", 32, "ocp", 0, n)
    assert_matches(q.view(torch.float8_e4m3fn), wq, "e4m3", "quantize, n = 2^32 + 4099")
    assert_matches(s, ws, "u8", "quantize, n = 2^32 + 4099", nan_class=False)
    assert_guards(bs, GUARD, s.numel(), "scales")
    del wq
    c = torch.empty(n, dtype=torch.float16, device="cuda")
    c.view(torch.uint8).fill_(POISON)
    dequantize(q.view(torch.float8_e4m3fn), s, "f16", 32, c)
    hq, hs = MX.quantize(host, "f16", "e4m3", 32, "ocp")
    want = tiled(MX.dequantize(hq, hs, "e4m3", "f16", 32), n - n % 32, "f16")
    for lo in ((1 << 31) - 4096, (1 << 32) - 4096, n - n % 32 - 8192):
        assert_matches(c[lo:lo + 8192], want[lo:lo + 8192], "f16", f"window at {lo}")
    assert_matches(c[:n - n % 32], want, "f16", "dequantize, n = 2^32 + 4099")
    tail = np.arange(n - n % 32, n) % host.size
    tq, ts = MX.quantize(host[tail], "f16", "e4m3", 32, "ocp")
    assert_matches(c[n - n % 32:], to_dev(MX.dequantize(tq, ts, "e4m3", "f16", 32), "f16"), "f16", "the short last block")


# ------------------------------------------------------------------------------------------- arguments
def test_rejected_arguments_return_their_code_and_write_nothing():
    L = capi.lib
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A, n = buf.data_ptr() + 4096, 1000
    C_, S_ = A + 16384, A + 32768 + 1                    # an output and scale bytes (odd address) away from A
    F32, F64, F16, BF16 = 0, 1, 2, 3
    E4, E5 = capi.F8_E4M3, capi.F8_E5M2
    q = [   # (src, A, fp8, C, S, n, block, rule)
        ((4, A, E4, C_, S_, n, 32, 0), capi.ERR_VARIANT), ((-1, A, E4, C_, S_, n, 32, 0), capi.ERR_VARIANT),
        ((F32, A, 2, C_, S_, n, 32, 0), capi.ERR_VARIANT), ((F32, A, -1, C_, S_, n, 32, 0), capi.ERR_VARIANT),
        ((F32, A, E4, C_, S_, n, 32, 2), capi.ERR_VARIANT), ((F32, A, E4, C_, S_, n, 32, -1), capi.ERR_VARIANT),
        ((F32, A, E4, C_, S_, n, 16, 0), capi.ERR_INVALID), ((F32, A, E4, C_, S_, n, 0, 0), capi.ERR_INVALID),
        ((F32, A, E4, C_, S_, n, 48, 0), capi.ERR_INVALID), ((F32, A, E4, C_, S_, n, 256, 1), capi.ERR_INVALID),
        ((F32, None, E4, C_, S_, n, 32, 0), capi.ERR_INVALID), ((F32, A, E5, None, S_, n, 32, 0), capi.ERR_INVALID),
        ((F32, A, E5, C_, None, n, 32, 0), capi.ERR_INVALID), ((F32, A, E4, C_, S_, (1 << 40) + 1, 128, 0), capi.ERR_INVALID),
        ((F32, A + 2, E4, C_, S_, n, 32, 0), capi.ERR_ALIGN), ((F64, A + 4, E4, C_, S_, n, 64, 0), capi.ERR_ALIGN),
        ((F16, A + 1, E5, C_, S_, n, 32, 1), capi.ERR_ALIGN),
        ((F32, A, E4, A, S_, n, 32, 0), capi.ERR_OVERLAP), ((F32, A, E4, A + 4 * n - 1, S_, n, 32, 0), capi.ERR_OVERLAP),
        ((BF16, A + 8, E4, A, S_, n, 32, 0), capi.ERR_OVERLAP),
        ((F32, A, E4, C_, A + 4 * n - 1, n, 32, 0), capi.ERR_OVERLAP), ((F32, A, E4, C_, A - 31, n, 32, 0), capi.ERR_OVERLAP),
        ((F32, A, E4, C_, C_ + n - 1, n, 128, 0), capi.ERR_OVERLAP), ((F64, A, E5, C_, C_ - 7, n, 128, 1), capi.ERR_OVERLAP),
    ]
    d = [   # (fp8, A, S, dst, C, n, block)
        ((E4, A, S_, 4, C_, n, 32), capi.ERR_VARIANT), ((2, A, S_, F32, C_, n, 32), capi.ERR_VARIANT),
        ((E5, A, S_, F16, C_, n, 33), capi.ERR_INVALID), ((E5, A, S_, F16, C_, n, -32), capi.ERR_INVALID),
        ((E4, None, S_, F32, C_, n, 32), capi.ERR_INVALID), ((E4, A, S_, F32, None, n, 32), capi.ERR_INVALID),
        ((E4, A, None, F32, C_, n, 32), capi.ERR_INVALID), ((E4, A, S_, F32, C_, (1 << 40) + 1, 32), capi.ERR_INVALID),
        ((E4, A, S_, F32, C_ + 2, n, 32), capi.ERR_ALIGN), ((E5, A, S_, F64, C_ + 4, n, 64), capi.ERR_ALIGN),
        ((E4, A, S_, BF16, C_ + 1, n, 128), capi.ERR_ALIGN),
        ((E4, A, S_, F32, A, n, 32), capi.ERR_OVERLAP), ((E4, A, S_, F16, A - 2 * n + 2, n, 32), capi.ERR_OVERLAP),
        ((E4, A, A + n - 1, F32, C_, n, 32), capi.ERR_OVERLAP), ((E5, A, C_ + 8 * n - 1, F64, C_, n, 64), capi.ERR_OVERLAP),
    ]
    for args, code in q:
        assert L.b200va_quantize_mxfp8(*args, None) == code, (args, code)
    for args, code in d:
        assert L.b200va_dequantize_mxfp8(*args, None) == code, (args, code)
    assert L.b200va_quantize_mxfp8(F32, None, E4, None, None, 0, 32, 0, None) == capi.OK       # n = 0: nothing to do
    assert L.b200va_quantize_mxfp8(F32, A, E4, C_, S_, 0, 64, 1, None) == capi.OK
    assert L.b200va_dequantize_mxfp8(E5, None, None, F64, None, 0, 128, None) == capi.OK
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == POISON).all(), "a rejected or empty call wrote to device memory"
    # right behind each other: no overlap, and the call runs
    assert L.b200va_quantize_mxfp8(F32, A, E4, A + 4 * n, A + 5 * n, n, 32, 0, None) == capi.OK
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        va.quantize_mxfp8(buf[:64].view(torch.float16), "e4m3", block=16)
    with pytest.raises(TypeError):
        va.quantize_mxfp8(buf[:256].view(torch.float16), "e4m3", scales=torch.empty(3, dtype=torch.uint8, device="cuda"))


# ------------------------------------------------------------------------------------------- stream order
def test_stream_op_quantize_dequantize_stream_op_on_one_stream():
    """Ten rounds on one stream without a host sync: b = s a (b200va_stream), (q, S) = quantize(b), c = dequantize(q, S),
    d_r = c / 2 (b200va_stream); a different s per round, at an L2-resident size and in the HBM class of the type."""
    st = torch.cuda.Stream()
    for src, fmt, dst, block, rule in (("f32", "e4m3", "f32", 32, "ocp"), ("bf16", "e5m2", "f16", 128, "nosat"),
                                       ("f64", "e4m3", "bf16", 64, "ocp")):
        period = 128 * 391
        a0 = X.finite(src, period, np.random.default_rng(DT_CODE[src]), 8.0)
        scalars = [1.0 + r / 8 for r in range(10)]
        wants = []
        for s in scalars:
            qh, sh = MX.quantize(X.stream("scale", src, a0, None, s), src, fmt, block, rule)
            wants.append(X.stream("scale", dst, MX.dequantize(qh, sh, fmt, dst, block), None, 0.5))
        for n in (21 * period, -(-(hbm_n(ES[src]) + 5) // period) * period):
            a = tiled(a0, n, src)
            b = torch.empty_like(a)
            q = torch.empty(n, dtype=TORCH[fmt], device="cuda")
            sc = torch.empty(n // block, dtype=torch.uint8, device="cuda")
            c = torch.empty(n, dtype=TORCH[dst], device="cuda")
            ds = [torch.empty_like(c) for _ in scalars]
            torch.cuda.synchronize()
            for s, d in zip(scalars, ds):
                va.stream("scale", a, None, b, scalar=s, stream=st)
                quantize(b, fmt, block, rule, q, sc, stream=st)
                dequantize(q, sc, dst, block, c, stream=st)
                va.stream("scale", c, None, d, scalar=0.5, stream=st)
            st.synchronize()
            for r, (d, w) in enumerate(zip(ds, wants)):
                assert_matches(d, tiled(w, n, dst), dst, f"{src}->{fmt}->{dst} n={n} round {r}")
            del a, b, q, sc, c, ds


def test_captured_graph_replays():
    cases = []
    for src, fmt, dst, block, rule in (("f32", "e5m2", "f64", 32, "nosat"), ("f64", "e4m3", "f16", 64, "ocp"),
                                       ("bf16", "e4m3", "f32", 128, "ocp")):
        x = V.random_bits(src, 100_003, np.random.default_rng(DT_CODE[src] + 40))
        bq, q = poisoned(x.size, fmt, 16)
        bs, s = poisoned(MX.scale_count(x.size, block), "u8", 1)
        bc, c = poisoned(x.size, dst, 16 // ES[dst])
        cases.append((src, fmt, dst, block, rule, x, to_dev(x, src), bq, q, bs, s, bc, c))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for src, fmt, dst, block, rule, _, a, _, q, _, s, _, c in cases:
                quantize(a, fmt, block, rule, q, s)
                dequantize(q, s, dst, block, c)
    torch.cuda.synchronize()
    for r in range(2):
        for case in cases:
            case[7].view(torch.uint8).fill_(POISON)
            case[9].fill_(POISON)
            case[11].view(torch.uint8).fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        for src, fmt, dst, block, rule, x, _, bq, q, bs, s, bc, c in cases:
            what = f"{src}->{fmt}->{dst} block {block} replay {r}"
            wq, ws = MX.quantize(x, src, fmt, block, rule)
            assert_matches(q, to_dev(wq, fmt), fmt, what)
            assert_matches(s, to_dev(ws, "u8"), "u8", what, nan_class=False)
            assert_matches(c, to_dev(MX.dequantize(wq, ws, fmt, dst, block), dst), dst, what)
            assert_guards(bq, GUARD + 16, x.size, what)
            assert_guards(bs, GUARD + 1, s.numel(), what)
            assert_guards(bc, GUARD + 16 // ES[dst], x.size, what)


def test_quantize_tail_reads_what_the_writer_wrote(env):
    """test_gpu_pdl_chains.py's chains (the 2^28 K2d writer of X, then 0-3 middle launches) with a block-scaled
    quantize of the end of X as the tail: its bytes and its scales against the exact window."""
    middles, chains = _chains(env)
    q = torch.empty(M + 1, dtype=torch.float8_e4m3fn, device="cuda")[1:]
    s = torch.empty(MX.scale_count(M, 32), dtype=torch.uint8, device="cuda")
    wq, ws = MX.quantize(env["ref_window"], "f32", "e4m3", 32, "ocp")
    failures = []
    for names in chains:
        q.view(torch.uint8).fill_(POISON)
        s.fill_(POISON)
        _run(env, middles, names, lambda w: quantize(w, "e4m3", 32, "ocp", q, s))
        bad = np.flatnonzero(q.view(torch.uint8).cpu().numpy() != wq)
        bad_s = np.flatnonzero(s.cpu().numpy() != ws)
        if bad.size or bad_s.size:
            failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> quantize: {bad.size} bytes and {bad_s.size} scales differ")
    assert not failures, "\n".join(failures)
    assert LO + M < env["X"].numel()


# ------------------------------------------------------------------------------------------- trace
def test_trace_shows_the_planned_kernels(tmp_path):
    """Per type, direction and block: n = 1000 and the HBM class on the vector body, n = 4099 on the edge path.  Under
    the profiler the kernels after the marker are exactly the planned ones with their grid and block."""
    nmax = max(hbm_n(ES[t]) for t in DTYPES) + 64
    wide = {t: torch.zeros(nmax, dtype=TORCH[t], device="cuda") for t in DTYPES}
    narrow = torch.zeros(nmax, dtype=torch.uint8, device="cuda")
    scales = torch.full((nmax // 32 + 2,), 127, dtype=torch.uint8, device="cuda")
    plan, want = [], []
    for kind in ("q", "d"):
        for t in DTYPES:
            for block in MX.BLOCKS:
                for n, off in ((1000, 0), (hbm_n(ES[t]), 0), (4099, 1)):
                    fmt = FMTS[(n + block) % 2]
                    w, f8 = wide[t][off:off + n], narrow[off:off + n].view(TORCH[fmt])
                    plan.append((kind, t, fmt, block, w, f8, scales[1:1 + MX.scale_count(n, block)]))
                    want.append(expected_mx_launch(kind, ES[t], n, block, off == 0))

    def run_plan():
        for kind, t, fmt, block, w, f8, s in plan:
            if kind == "q":
                quantize(w, fmt, block, "ocp", f8, s)
            else:
                dequantize(f8, s, t, block, w)
        torch.cuda.synchronize()

    got = kernels_after_marker(tmp_path, run_plan, ("mx_",))
    assert len(got) == len(want), (len(got), len(want), got[:8])
    for g, w, p in zip(got, want, plan):
        assert g == w, (p[:4], g, w)
