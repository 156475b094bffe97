"""CPU checks of tests/fp8_rowwise_exact.py, the row-wise scales against torch's scaled_mm checks, and the SASS of the
block-scaled quantize kernel that carries b200va_quantize_fp8_rowwise's three launches.

- The reference's maxima, k, scale bits and bytes against a Fraction restatement of the rule, on random bit patterns
  and on edge rows: every f64 binade edge, 1.75 2^e +- 1 ulp, zero, NaN/inf-only and subnormal rows, and both clamps.
- A row's scale is the largest of its 1x128 block scales (tests/fp8_block_exact.py); the workspace holds exactly the
  1x128 block scales of both sides.
- S.view(-1, 1) and St.view(1, -1) pass scaled_mm's RowWise checks (torch.nn.functional.scaled_mm and
  torch._scaled_mm) for the three products of a linear layer, and a mis-shaped scale is rejected.
- mx_quant_vec holds the row-wise bodies' traffic and still no local memory.
"""
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

import fp8_block_exact as BE
import fp8_rowwise_exact as RE
import sass
from oracle import convert_exact as V
from oracle import fp8_exact as F
from oracle import stream_exact as X
from oracle.stream_exact import widen

from k8s_gpu_hpa_b200 import capi


# ------------------------------------------------------------------------------------------- the rule, restated
def k_fraction(m: Fraction, fmt: str) -> int:
    """clamp(K(m), -126, 126): K(m) the largest k with m 2^k <= max finite, K(0) = +inf."""
    if m == 0:
        return 126
    top = Fraction(F.MAX_FINITE[fmt])
    k = 126
    while k > -126 and m * Fraction(2) ** k > top:
        k -= 1
    return k


def restated(x: np.ndarray, fmt: str):
    """(C, k) of the f64 matrix x with one scale per row, by Fractions: the row maximum over the finite elements, k,
    and each element rounded to nearest (ties to even) on the FP8 grid, saturating."""
    rows, cols = x.shape
    ks = []
    c = np.zeros((rows, cols), np.uint8)
    for r in range(rows):
        fin = [Fraction(abs(float(v))) for v in x[r] if np.isfinite(v)]
        k = k_fraction(max(fin, default=Fraction(0)), fmt)
        ks.append(k)
        for j in range(cols):
            v = float(x[r, j])
            if not np.isfinite(v):
                y = v
            else:
                y = np.copysign(F.nearest_fraction(Fraction(v) * Fraction(2) ** k, fmt), v)
            c[r, j] = F.round_fp8(np.array([y]), fmt)[0]
    return c, np.array(ks)


def edge_rows():
    """Rows of 8 f64 values whose maximum sits at a binade edge, 1.75 2^e +- 1 ulp, or makes k clamp."""
    rows = []
    for e in range(-1074, 1024, 7):
        for m in (2.0 ** e, 1.75 * 2.0 ** e if e > -1073 else 2.0 ** e):
            for v in (m, np.nextafter(m, 0.0), np.nextafter(m, np.inf)):
                if np.isfinite(v) and v > 0:
                    rows.append([v, -v / 3, v / 1024, 0.0, -0.0, v / 7, -v, v * 2.0 ** -60])
    rows.append([0.0] * 8)
    rows.append([np.nan, np.inf, -np.inf, np.nan, 0.0, -0.0, np.inf, np.nan])
    rows.append([5e-324, -5e-324, 2.0 ** -1040, 0.0, 1e-310, -2e-310, 3e-320, 0.0])      # subnormal
    rows.append([1.7e308, -1e300, 1.0, 0.0, 2.0 ** 1000, 1e-300, -3.0, 5.0])            # k clamps at -126
    rows.append([2.0 ** -1000, -2.0 ** -1001, 0.0, 2.0 ** -1020, 0.0, 0.0, 0.0, 0.0])     # k clamps at 126
    return np.array(rows)


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_reference_matches_the_restatement_on_edge_rows(fmt):
    x = edge_rows()
    c, s, ct, st = RE.quantize(x.ravel(), "f64", fmt, *x.shape)
    want_c, k = restated(x, fmt)
    assert np.array_equal(c, want_c)
    assert np.array_equal(s.view(np.int32), ((127 - k) << 23).astype(np.int32))
    want_ct, kt = restated(np.ascontiguousarray(x.T), fmt)
    assert np.array_equal(ct, want_ct)
    assert np.array_equal(st.view(np.int32), ((127 - kt) << 23).astype(np.int32))
    assert k.min() == -126 and k.max() == 126


@pytest.mark.parametrize("fmt", F.FORMATS8)
@pytest.mark.parametrize("src", ("f32", "f64", "f16", "bf16"))
def test_reference_matches_the_restatement_on_random_bits(src, fmt):
    rng = np.random.default_rng([17, len(src), len(fmt)])
    rows, cols = 6, 40
    host = V.random_bits(src, rows * cols, rng)
    c, s, ct, st = RE.quantize(host, src, fmt, rows, cols)
    x = widen(host, src).reshape(rows, cols)
    want_c, k = restated(x, fmt)
    want_ct, kt = restated(np.ascontiguousarray(x.T), fmt)
    assert np.array_equal(c, want_c) and np.array_equal(ct, want_ct)
    assert np.array_equal(s, RE.scales(k)) and np.array_equal(st, RE.scales(kt))


def test_row_scale_is_the_largest_block_scale():
    rng = np.random.default_rng(23)
    for rows, cols in ((3, 700), (130, 257), (1, 1), (129, 128)):
        x = X.finite("f32", rows * cols, rng, 6.0).reshape(rows, cols)
        x[rng.integers(0, rows, 5), rng.integers(0, cols, 5)] = 0.0
        for fmt in F.FORMATS8:
            _, s, _, st = RE.quantize(x.ravel(), "f32", fmt, rows, cols)
            _, bs, _, bst = BE.quantize(x.ravel(), "f32", fmt, "1x128", rows, cols)
            nb, nbt = -(-cols // 128), -(-rows // 128)
            assert np.array_equal(s, bs.reshape(nb, rows).max(axis=0))
            assert np.array_equal(st, bst.reshape(nbt, cols).max(axis=0))


def test_workspace_is_the_block_scales_of_both_sides():
    for rows, cols in ((0, 5), (5, 0), (1, 1), (128, 128), (129, 513), (1000, 130), (4096, 65536), (16384, 16384)):
        want = 4 * (BE.scale_count(rows, cols, "1x128") + BE.scale_count(cols, rows, "1x128"))
        assert RE.workspace_bytes(rows, cols) == want
        assert capi.lib.b200va_fp8_rowwise_workspace(rows, cols) == want


# ------------------------------------------------------------------------------------------- scaled_mm's checks
def _fp8(*shape):
    return torch.empty(*shape, dtype=torch.float8_e4m3fn, device="meta")


def _f32(n):
    return torch.empty(n, dtype=torch.float32, device="meta")


def _products(Mt, K, N):
    """The three products of a linear layer Y = X W^T (X: Mt x K, W: N x K) as (a, b, scale_a, scale_b), from each
    tensor's (C, S, Ct, St) shapes."""
    X_ = (_fp8(Mt, K), _f32(Mt), _fp8(K, Mt), _f32(K))
    W_ = (_fp8(N, K), _f32(N), _fp8(K, N), _f32(K))
    dY = (_fp8(Mt, N), _f32(Mt), _fp8(N, Mt), _f32(N))
    return {"forward": (X_[0], W_[0].t(), X_[1].view(-1, 1), W_[1].view(1, -1), (Mt, N)),
            "data gradient": (dY[0], W_[2].t(), dY[1].view(-1, 1), W_[3].view(1, -1), (Mt, K)),
            "weight gradient": (dY[2], X_[2].t(), dY[3].view(-1, 1), X_[3].view(1, -1), (N, K))}


@pytest.mark.parametrize("product", ["forward", "data gradient", "weight gradient"])
def test_scales_pass_scaled_mm_rowwise_checks(product):
    F_ = torch.nn.functional
    RW = F_.ScalingType.RowWise
    a, b, sa, sb, shape = _products(256, 512, 384)[product]
    out = F_.scaled_mm(a, b, sa, RW, sb, RW, output_dtype=torch.bfloat16)
    assert tuple(out.shape) == shape
    out = torch._scaled_mm(a, b, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
    assert tuple(out.shape) == shape
    # torch._scaled_mm checks both scales' shapes; F.scaled_mm checks their element counts
    for bad_a, bad_b in ((sa.view(1, -1), sb), (sa, sb.view(-1, 1)), (sa[:-1], sb), (sa, sb[:, :-1])):
        with pytest.raises(Exception):
            torch._scaled_mm(a, b, scale_a=bad_a, scale_b=bad_b, out_dtype=torch.bfloat16)
    for bad_a, bad_b in ((sa[:-1], sb), (sa, sb[:, :-1])):
        with pytest.raises(Exception):
            F_.scaled_mm(a, b, bad_a, RW, bad_b, RW, output_dtype=torch.bfloat16)


# ------------------------------------------------------------------------------------------- SASS
@pytest.mark.parametrize("path", ["production", "tune"])
def test_rowwise_bodies_in_the_sass(path):
    fns = {fn: b for fn, b in sass.functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH).items()
           if re.match(r"_ZN6b200va\d+mx_", fn)}
    quant = {fn: b for fn, b in fns.items() if "mx_quant_vec" in fn}
    assert len(quant) == 3
    for fn, body in fns.items():
        assert not re.search(r"\b(LDL|STL)\b", body), fn
    for fn, body in quant.items():
        ops = sass.opcodes(body)
        # the reduction's and the cast's f32 scale loads, the tile's byte scatter and its 16-byte Ct rows
        assert "LDG.E" in ops and "STS.U8" in ops and "LDS.128" in ops and "STG.E.NA.128" in ops, fn
        assert "BAR.SYNC" in ops or "BAR.SYNC.DEFER_BLOCKING" in ops, fn
        assert not any(o.startswith(("ATOM", "RED")) for o in ops), fn
