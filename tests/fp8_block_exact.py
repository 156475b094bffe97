"""Exact reference of b200va_quantize_fp8_blockwise and b200va_dequantize_fp8_blockwise (include/b200va.h), built on
oracle/fp8_exact.py (the rounding) and tests/fp8_auto_exact.py (the scale exponent K): numpy only.

  block maxima  the largest finite |a| of each block, widened exactly (NaN and +-inf do not take part)
  k             auto_scale_exp(m, fmt, 0): clamp(K(m), -126, 126), K(0) = +inf; the scale is the f32 2^-k
  bytes         fp8_exact.round_fp8(a 2^k) with each element's block k
  layouts       1x128: S[b rows + i]; 128x128: S[p L4 + q]; the padding entries are left as they were
  dequantize    q s formed exactly in f64 (q has at most 4 significant bits) and rounded once to the destination
"""
from __future__ import annotations

import numpy as np

from oracle import fp8_exact as F
from oracle.convert_exact import round_f64
from oracle.stream_exact import widen

import fp8_auto_exact as AE

KINDS = ("1x128", "128x128")
B = 128


def scale_count(rows: int, cols: int, kind: str) -> int:
    if rows == 0 or cols == 0:
        return 0
    nkb_c = -(-cols // B)
    return rows * nkb_c if kind == "1x128" else -(-rows // B) * (-(-nkb_c // 4) * 4)


def block_maxima(x: np.ndarray, rb: int, cb: int) -> np.ndarray:
    """The finite maxima of the rb x cb blocks of the f64 matrix x (short at the edges): [ceil(R/rb), ceil(C/cb)]."""
    R, C = x.shape
    m = np.where(np.isfinite(x), np.abs(x), 0.0)
    pr, pc = -(-R // rb) * rb, -(-C // cb) * cb
    p = np.zeros((pr, pc))
    p[:R, :C] = m
    return p.reshape(pr // rb, rb, pc // cb, cb).max(axis=(1, 3))


def exponents(m: np.ndarray, fmt: str) -> np.ndarray:
    return np.vectorize(lambda v: AE.auto_scale_exp(float(v), fmt, 0), otypes=[np.int64])(m) if m.size else \
        np.zeros(m.shape, np.int64)


def _quantize_operand(x: np.ndarray, fmt: str, kind: str):
    """(bytes, k per block [nbr, nbc]) of the rows x cols f64 matrix x quantized row-wise in kind's blocks."""
    rb = 1 if kind == "1x128" else B
    k = exponents(block_maxima(x, rb, B), fmt)
    kk = np.repeat(np.repeat(k, rb, axis=0), B, axis=1)[:x.shape[0], :x.shape[1]]
    with np.errstate(all="ignore"):
        return F.round_fp8(np.ldexp(x, kk).ravel(), fmt).reshape(x.shape), k


def scales_layout(k: np.ndarray, rows: int, cols: int, kind: str, base: np.ndarray | None = None) -> np.ndarray:
    """The f32 scales 2^-k of the blocks k ([nbr, nbc]) stored in kind's layout over base (untouched padding)."""
    n = scale_count(rows, cols, kind)
    out = np.zeros(n, np.float32) if base is None else base.copy()
    s = np.ldexp(np.float32(1), -k).astype(np.float32)
    if kind == "1x128":
        out[:] = s.T.ravel()                                  # S[b rows + i]
    else:
        l4 = n // s.shape[0]
        v = out.reshape(s.shape[0], l4)
        v[:, :s.shape[1]] = s                                 # S[p L4 + q]
    return out


def quantize(a: np.ndarray, src: str, fmt: str, kind: str, rows: int, cols: int, s_base=None, st_base=None):
    """(C, S, Ct, St) of b200va_quantize_fp8_blockwise: uint8 [rows, cols], f32 scales, uint8 [cols, rows], f32."""
    x = widen(np.ascontiguousarray(a).ravel(), src).reshape(rows, cols)
    c, k = _quantize_operand(x, fmt, kind)
    ct, kt = _quantize_operand(np.ascontiguousarray(x.T), fmt, kind)
    return (c, scales_layout(k, rows, cols, kind, s_base), ct, scales_layout(kt, cols, rows, kind, st_base))


def scale_per_element(s: np.ndarray, rows: int, cols: int, kind: str) -> np.ndarray:
    """The f32 scale of each element of a rows x cols operand, read from kind's layout."""
    i, j = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    if kind == "1x128":
        idx = (j // B) * rows + i
    else:
        idx = (i // B) * (scale_count(rows, cols, kind) // -(-rows // B)) + j // B
    return s[idx]


def dequantize(q: np.ndarray, s: np.ndarray, fmt: str, dst: str, kind: str, rows: int, cols: int) -> np.ndarray:
    """b200va_dequantize_fp8_blockwise in dst storage: q s exact in f64, one rounding."""
    v = F.DECODE[fmt][np.asarray(q, np.uint8).reshape(rows, cols)]
    with np.errstate(all="ignore"):
        x = (v * scale_per_element(s, rows, cols, kind).astype(np.float64)).ravel()
    return x if dst == "f64" else round_f64(x, dst)
