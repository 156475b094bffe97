"""CPU checks of tests/fp8_block_exact.py, the blockwise scale layout against torch's scaled_mm checks, and the SASS
of the block-scaled kernels that carry b200va_quantize_fp8_blockwise and b200va_dequantize_fp8_blockwise.

- k is the negated, clamped B200VA_MX_SCALE_NOSAT exponent and quantize_fp8_auto's margin-0 k at every f64 binade
  edge; with k unclamped no finite element saturates.
- fp8_blockwise_scale_layout's shape and stride pass torch.nn.functional.scaled_mm's meta checks for the (1x128,
  1x128), (1x128, 128x128) and (128x128, 1x128) pairs, and a row-major view is rejected.
- mx_quant_vec holds the tile's shared-memory traffic, barrier and f32 scale stores; no mx_ kernel spills; the
  library keeps its function count (tests/test_kernel_inventory.py).
"""
import re

import numpy as np
import pytest
import torch

import fp8_auto_exact as AE
import fp8_block_exact as BE
import sass
from oracle import fp8_exact as F
from oracle import mxfp8_exact as MX

from k8s_gpu_hpa_b200 import capi, vector_add as va


def edges():
    for e in range(-1074, 1024):
        for m in (2.0 ** e, 1.75 * 2.0 ** e if e > -1073 else 2.0 ** e):
            for v in (m, np.nextafter(m, 0.0), np.nextafter(m, np.inf)):
                if np.isfinite(v) and v > 0:
                    yield float(v)


@pytest.mark.parametrize("fmt", F.FORMATS8)
def test_k_is_the_negated_nosat_exponent_and_the_auto_k(fmt):
    vs = np.array(list(edges()))
    k = BE.exponents(vs, fmt)
    blocks = MX.blocks_with_maximum(vs, "f64", 32)
    e = MX.block_exponents(blocks, "f64", fmt, 32, "nosat")
    assert (k == np.clip(-e, -126, 126)).all()
    assert all(int(k[i]) == AE.auto_scale_exp(float(v), fmt, 0) for i, v in enumerate(vs))
    assert BE.exponents(np.array([0.0]), fmt).tolist() == [126]
    free = (k > -126) & (k < 126)
    assert (np.ldexp(vs[free], k[free]) <= F.MAX_FINITE[fmt]).all()
    assert (np.ldexp(vs[free], k[free] + 1) > F.MAX_FINITE[fmt]).all()


def test_scale_counts_match_the_library():
    for rows, cols in ((0, 5), (5, 0), (1, 1), (128, 128), (129, 513), (1000, 130), (4096, 65536)):
        for kind in BE.KINDS:
            assert capi.lib.b200va_fp8_blockwise_scales(rows, cols, capi.FP8_BLOCK[kind]) == BE.scale_count(rows, cols, kind)
            if rows and cols:
                assert va.fp8_blockwise_scale_layout(rows, cols, kind)[0] == BE.scale_count(rows, cols, kind)
    assert capi.lib.b200va_fp8_blockwise_scales(128, 128, 2) == 0


def _meta_scales(rows, cols, kind, row_major=False):
    numel, shape, stride = va.fp8_blockwise_scale_layout(rows, cols, kind)
    if row_major:
        stride = (shape[1], 1)
    return torch.empty(numel, dtype=torch.float32, device="meta").as_strided(shape, stride)


@pytest.mark.parametrize("pair", [("1x128", "1x128"), ("1x128", "128x128"), ("128x128", "1x128")])
def test_layout_passes_scaled_mm_checks(pair):
    F_ = torch.nn.functional
    S = F_.ScalingType
    rec = {"1x128": S.BlockWise1x128, "128x128": S.BlockWise128x128}
    M, K, N = 256, 512, 384
    a = torch.empty(M, K, dtype=torch.float8_e4m3fn, device="meta")
    b_t = torch.empty(N, K, dtype=torch.float8_e4m3fn, device="meta")          # the K-major second operand
    sa, sb = _meta_scales(M, K, pair[0]), _meta_scales(N, K, pair[1])
    out = F_.scaled_mm(a, b_t.t(), sa, rec[pair[0]], sb, rec[pair[1]], output_dtype=torch.bfloat16)
    assert tuple(out.shape) == (M, N)
    with pytest.raises(Exception):
        F_.scaled_mm(a, b_t.t(), _meta_scales(M, K, pair[0], row_major=True), rec[pair[0]],
                     _meta_scales(N, K, pair[1], row_major=True), rec[pair[1]], output_dtype=torch.bfloat16)


@pytest.mark.parametrize("path", ["production", "tune"])
def test_blockwise_bodies_in_the_sass(path):
    fns = {fn: b for fn, b in sass.functions(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH).items()
           if re.match(r"_ZN6b200va\d+mx_", fn)}
    quant = {fn: b for fn, b in fns.items() if "mx_quant_vec" in fn}
    assert len(quant) == 3
    for fn, body in fns.items():
        assert not re.search(r"\b(LDL|STL)\b", body), fn
    for fn, body in quant.items():
        assert "BAR.SYNC" in body and "STS.U8" in body and "LDS.128" in body and "STG.E.NA.128" in body, fn
        assert re.search(r"\bSTG\.E\b(?!\.)", body) or "STG.E " in body, fn          # the f32 scale stores
