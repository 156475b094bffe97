"""The SASS of b200va_quantize_fp8_transpose's kernels in both libraries (no GPU needed).

The four fp8_quant_vec<SRC> kernels carry the transposed body beside the 1-D quantize and the amax pass, so each must
now hold the shared-memory tile (byte stores, 16-byte loads, a barrier) and still the 1-D path's rounding, 16-byte
loads and no-allocate 16-byte stores, one atomic for all of its bodies, and no local memory.  The production library
keeps its 199 functions.
"""
import re

import pytest

import sass
from k8s_gpu_hpa_b200 import capi


def _quant_kernels(path: str) -> dict[str, str]:
    return {fn: body for fn, body in sass.functions(path).items() if re.match(r"_ZN6b200va\d+fp8_quant_vec", fn)}


@pytest.mark.parametrize("path", ["production", "tune"])
def test_quant_kernels_carry_the_tile_and_keep_the_1d_path(path):
    quant = _quant_kernels(capi.LIB_PATH if path == "production" else capi.TUNE_LIB_PATH)
    assert len(quant) == 4, sorted(quant)
    for fn, body in quant.items():
        ops = sass.opcodes(body)
        assert "STS.U8" in ops and "LDS.128" in ops, fn
        assert ops.count("BAR.SYNC.DEFER_BLOCKING") >= 2, fn            # the tile's, beside cta_amax's
        for f8 in ("E4M3", "E5M2"):
            assert f"F2FP.SATFINITE.{f8}.F32" in body, (fn, f8)
        assert "LDG.E.128" in ops and "STG.E.NA.128" in ops, fn
        assert sum(o.startswith(("ATOMG", "RED")) for o in ops) == 1, fn
        assert not re.search(r"\b(LDL|STL)\b", body), fn


def test_the_production_library_keeps_199_functions():
    assert len(sass.functions(capi.LIB_PATH)) == 199
