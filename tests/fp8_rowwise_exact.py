"""Exact reference of b200va_quantize_fp8_rowwise and b200va_dequantize_fp8_rowwise (include/b200va.h), built on
oracle/fp8_exact.py (the rounding), tests/fp8_auto_exact.py (the scale exponent K) and tests/fp8_block_exact.py
(the finite maxima): numpy only.

  maxima      the largest finite |a| of each row (for C) and each column (for Ct), widened exactly
  k           auto_scale_exp(m, fmt, 0): clamp(K(m), -126, 126), K(0) = +inf; the scale is the f32 2^-k
  bytes       fp8_exact.round_fp8(a 2^k) with the element's row k (C) or column k (Ct)
  dequantize  q s formed exactly in f64 (q has at most 4 significant bits) and rounded once to the destination
"""
from __future__ import annotations

import numpy as np

from oracle import fp8_exact as F
from oracle.convert_exact import round_f64
from oracle.stream_exact import widen

import fp8_block_exact as BE


def workspace_bytes(rows: int, cols: int) -> int:
    """The 1x128 block scales of both sides, 4 bytes each."""
    return 4 * (BE.scale_count(rows, cols, "1x128") + BE.scale_count(cols, rows, "1x128"))


def row_maxima(x: np.ndarray) -> np.ndarray:
    """The finite maximum of each row of the f64 matrix x."""
    return np.where(np.isfinite(x), np.abs(x), 0.0).max(axis=1, initial=0.0)


def scales(k: np.ndarray) -> np.ndarray:
    """The f32 scales 2^-k."""
    return np.ldexp(np.float32(1), -np.asarray(k)).astype(np.float32)


def _quantize_rows(x: np.ndarray, fmt: str):
    """(bytes, k per row) of the f64 matrix x quantized with one scale per row."""
    k = BE.exponents(row_maxima(x), fmt)
    with np.errstate(all="ignore"):
        return F.round_fp8(np.ldexp(x, k[:, None]).ravel(), fmt).reshape(x.shape), k


def quantize(a: np.ndarray, src: str, fmt: str, rows: int, cols: int):
    """(C, S, Ct, St) of b200va_quantize_fp8_rowwise: uint8 [rows, cols], f32 [rows], uint8 [cols, rows], f32 [cols]."""
    x = widen(np.ascontiguousarray(a).ravel(), src).reshape(rows, cols)
    c, k = _quantize_rows(x, fmt)
    ct, kt = _quantize_rows(np.ascontiguousarray(x.T), fmt)
    return c, scales(k), ct, scales(kt)


def dequantize(q: np.ndarray, s: np.ndarray, fmt: str, dst: str, rows: int, cols: int) -> np.ndarray:
    """b200va_dequantize_fp8_rowwise in dst storage: q S[r] exact in f64, one rounding."""
    v = F.DECODE[fmt][np.asarray(q, np.uint8).reshape(rows, cols)]
    with np.errstate(all="ignore"):
        x = (v * np.asarray(s, np.float32).astype(np.float64)[:, None]).ravel()
    return x if dst == "f64" else round_f64(x, dst)
