"""Host-side plumbing over the C ABI for tests and bench.py: torch owns device memory and
streams, libb200va.so does the work.  Every function here ends in a C-ABI call on raw
pointers; nothing computes ``a + b`` in Python/torch (no fallback path).

Names follow the reference's process (SURVEY.md section 8(a)):
  a2 ``fill_rand_host`` / ``fill_ctr``     a4/a5 ``add``      a1 ``add_loop``
  a3+a4+a6 ``Stager`` / ``add_host``      a6 ``verify`` / ``verify_host``
whose only reference anchor is the call site ``cuda-test-deployment.yaml:18-19``.
"""
from __future__ import annotations

import ctypes as C
import subprocess

import numpy as np

from . import capi
from .capi import K_AUTO, VARIANTS, Tune, check, lib


def _torch():
    import torch
    return torch


def _variant(v) -> int:
    return VARIANTS[v] if isinstance(v, str) else int(v)


def _dev_ptr(t, name: str) -> int:
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    return t.data_ptr()


def _f32_operands(ref: str, **operands) -> tuple[int, ...]:
    """The device pointers of the operands, in order, each checked by _dev_ptr and all checked to have the length of
    operand `ref` and to lie on its device, before the caller makes any C-ABI call (a shorter operand would be read or
    written past its end)."""
    ptrs = tuple(_dev_ptr(t, name) for name, t in operands.items())
    r = operands[ref]
    for name, t in operands.items():
        if t.numel() != r.numel():
            raise ValueError(f"{name} differs from {ref} in length ({t.numel()} elements, {ref} has {r.numel()})")
        if t.device != r.device:
            raise ValueError(f"{name} is on {t.device}, {ref} on {r.device}")
    return ptrs


def _stream_ptr(stream) -> int:
    torch = _torch()
    if stream is None:
        stream = torch.cuda.current_stream()
    return stream.cuda_stream


def add(a, b, out=None, *, variant=K_AUTO, tune: Tune | None = None, stream=None, inputs_stable: bool = False,
        cold: bool = False, full_matrix: bool = False):
    """C = A + B on the current CUDA stream (asynchronous). ``out`` may be ``a`` or ``b``.
    ``inputs_stable``: b200va_add_f32_ex with B200VA_F_INPUTS_STABLE (the previous launch on the
    stream does not write a or b); ``cold``: B200VA_F_COLD (operands not in L2).  ``full_matrix``: send an explicit ``tune`` to
    libb200va_tune.so, which carries every geometry (the production library refuses the
    ones AUTO never picks with ERR_VARIANT)."""
    torch = _torch()
    if out is None:
        out = torch.empty_like(a)
    pa, pb, pc = _f32_operands("a", a=a, b=b, out=out)
    with torch.cuda.device(a.device):
        if tune is not None:
            h = capi.tune_lib() if full_matrix else lib
            check(h.b200va_add_f32_tuned(pa, pb, pc, a.numel(), C.byref(tune), _stream_ptr(stream)), "b200va_add_f32_tuned")
        elif inputs_stable or cold:
            flags = (capi.F_INPUTS_STABLE if inputs_stable else 0) | (capi.F_COLD if cold else 0)
            check(lib.b200va_add_f32_ex(pa, pb, pc, a.numel(), _variant(variant), flags, _stream_ptr(stream)), "b200va_add_f32_ex")
        else:
            check(lib.b200va_add_f32(pa, pb, pc, a.numel(), _variant(variant), _stream_ptr(stream)), "b200va_add_f32")
    return out


def add_loop(a, b, out, iters: int, *, graph_batch: int = 0, variant=K_AUTO, stream=None):
    """The launch loop in-process: ``iters`` launches (CUDA-graph batched if graph_batch>1)."""
    torch = _torch()
    pa, pb, pc = _f32_operands("a", a=a, b=b, out=out)
    with torch.cuda.device(a.device):
        check(lib.b200va_add_f32_loop(pa, pb, pc, a.numel(), _variant(variant), iters, graph_batch,
                                      _stream_ptr(stream)), "b200va_add_f32_loop")
    return out


class Loop:
    """The persistent launch loop (a1): ``graph_batch`` launches captured once into a CUDA graph,
    ``run(iters)`` replays it asynchronously on the current stream (b200va_loop_*)."""

    def __init__(self, a, b, out, *, graph_batch: int = 50, variant=K_AUTO):
        torch = _torch()
        self._h = C.c_void_p()
        pa, pb, pc = _f32_operands("a", a=a, b=b, out=out)
        self._keep = (a, b, out)
        self._device = a.device
        with torch.cuda.device(a.device):
            check(lib.b200va_loop_create(C.byref(self._h), pa, pb, pc, a.numel(), _variant(variant), graph_batch),
                  "b200va_loop_create")

    def run(self, iters: int, *, stream=None) -> None:
        torch = _torch()
        with torch.cuda.device(self._device):
            check(lib.b200va_loop_run(self._h, iters, _stream_ptr(stream)), "b200va_loop_run")

    def close(self) -> None:
        """Destroy the graph; the stream must have drained."""
        if self._h:
            lib.b200va_loop_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        _torch().cuda.synchronize(self._device)
        self.close()


_FLOAT = {"f32": "float32", "f64": "float64", "f16": "float16", "bf16": "bfloat16"}
_FP8 = {"e4m3": "float8_e4m3fn", "e5m2": "float8_e5m2"}


def _resolve(dtype, names: dict, codes: dict, what: str):
    """(torch dtype, ABI code) of a dtype given as a torch dtype or by its short name in ``names``."""
    torch = _torch()
    dtypes = {getattr(torch, v): k for k, v in names.items()}
    if isinstance(dtype, str):
        if dtype not in names:
            raise TypeError(f"{what} must be one of {sorted(names)}, got {dtype!r}")
        dtype = getattr(torch, names[dtype])
    if dtype not in dtypes:
        raise TypeError(f"{what} must be one of {'/'.join(names.values())}, got {dtype}")
    return dtype, codes[dtypes[dtype]]


def _float_dtype(dtype):
    """(torch dtype, B200VA_DT_* code) of f32/f64/f16/bf16 given as a torch dtype or "f32"/"f64"/"f16"/"bf16"."""
    return _resolve(dtype, _FLOAT, capi.DTYPES, "dtype")


def _fp8_format(fmt):
    """(torch dtype, B200VA_F8_* code) of an FP8 format given as a torch dtype or "e4m3" / "e5m2"."""
    return _resolve(fmt, _FP8, capi.F8, "fmt")


def _operand(t, name: str, resolve=_float_dtype) -> int:
    """The ABI code of a contiguous CUDA tensor whose dtype ``resolve`` accepts (default f32/f64/f16/bf16)."""
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda or not t.is_contiguous():
        raise TypeError(f"{name} must be a contiguous CUDA tensor")
    return resolve(t.dtype)[1]


def _like(t, dtype, a, name: str):
    """``t``, checked to be a contiguous tensor of ``dtype`` with a's length on a's device."""
    torch = _torch()
    if (not isinstance(t, torch.Tensor) or t.dtype != dtype or t.numel() != a.numel() or t.device != a.device
            or not t.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous tensor of {dtype} with a's length on a's device")
    return t


def _out(out, dtype, a):
    """``out`` checked by _like, or a new tensor of ``dtype`` shaped like a on a's device."""
    return _torch().empty(a.shape, dtype=dtype, device=a.device) if out is None else _like(out, dtype, a, "out")


def stream(op: str, a, b=None, out=None, *, scalar: float = 0.0, stream=None):
    """STREAM-style op (copy | scale | add | triad) on CUDA tensors of f32/f64/f16/bf16
    through b200va_stream.  Asynchronous on the current stream."""
    code = _operand(a, "a")
    if b is not None:
        _like(b, a.dtype, a, "b")
    out = _out(out, a.dtype, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_stream(capi.OPS[op], code, a.data_ptr(), b.data_ptr() if b is not None else None,
                                out.data_ptr(), a.numel(), float(scalar), _stream_ptr(stream)), "b200va_stream")
    return out


def convert(a, dtype, out=None, *, stream=None):
    """``a`` rounded once to ``dtype`` (torch.float32/float64/float16/bfloat16, or "f32"/"f64"/"f16"/"bf16")
    through b200va_convert: round-to-nearest-even, no FTZ, overflow to inf; the same dtype is a bit copy.
    ``out``: a contiguous CUDA tensor of ``dtype`` with a's length on a's device (it may be ``a`` itself when
    both element sizes are equal), else a new one.  Asynchronous on the current stream."""
    src = _operand(a, "a")
    dtype, dst = _float_dtype(dtype)
    out = _out(out, dtype, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_convert(src, a.data_ptr(), dst, out.data_ptr(), a.numel(), _stream_ptr(stream)), "b200va_convert")
    return out


def _one_element(t, dtype, a, name: str):
    """``t`` checked to be a one-element tensor of ``dtype`` on a's device."""
    torch = _torch()
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.numel() != 1 or t.device != a.device:
        raise TypeError(f"{name} must be a one-element {dtype} tensor on a's device")
    return t


def _amax(amax, a):
    """``amax``: None, or checked to be a one-element float64 tensor on a's device."""
    return amax if amax is None else _one_element(amax, _torch().float64, a, "amax")


def _matrix(a) -> tuple[int, int, int]:
    """(ABI code, rows, cols) of a contiguous 2-D CUDA tensor of f32/f64/f16/bf16."""
    code = _operand(a, "a")
    if a.dim() != 2:
        raise TypeError(f"a must be a 2-D tensor, got {a.dim()} dimensions")
    return code, a.shape[0], a.shape[1]


def _out_shaped(out, dtype, shape, a, name: str):
    """``out`` checked to be a contiguous tensor of ``dtype`` and ``shape`` on a's device, or a new one."""
    torch = _torch()
    if out is None:
        return torch.empty(shape, dtype=dtype, device=a.device)
    if (not isinstance(out, torch.Tensor) or out.dtype != dtype or tuple(out.shape) != tuple(shape)
            or out.device != a.device or not out.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous {dtype} tensor of shape {list(shape)} on a's device")
    return out


def _quantize(a, fmt, k: int, amax, out, stream, *, transpose=False, out_t=None, auto=False, scale_exp=None):
    """The four per-tensor quantize wrappers: ``a`` of any shape, or with ``transpose`` the 2-D ``a`` whose transposed
    bytes go to ``out_t``.  ``k`` is the host's scale exponent, or with ``auto`` the margin of one chosen on the device
    and written to ``scale_exp`` (a new one when None), a None ``amax`` then being a zeroed one made on the call's
    stream.  Returns out, then out_t when transposing, then scale_exp when auto."""
    torch = _torch()
    if transpose:
        src, rows, cols = _matrix(a)
    else:
        src = _operand(a, "a")
    dtype, code = _fp8_format(fmt)
    if transpose:
        out = _out_shaped(out, dtype, (rows, cols), a, "out")
        out_t = _out_shaped(out_t, dtype, (cols, rows), a, "out_t")
    else:
        out = _out(out, dtype, a)
    _amax(amax, a)
    if auto:
        scale_exp = (torch.empty(1, dtype=torch.int32, device=a.device) if scale_exp is None
                     else _one_element(scale_exp, torch.int32, a, "scale_exp"))
    name = "b200va_quantize_fp8" + "_transpose" * transpose + "_auto" * auto
    shape = (out_t.data_ptr(), rows, cols) if transpose else (a.numel(),)
    with torch.cuda.device(a.device):
        st = stream if stream is not None else torch.cuda.current_stream()
        if auto and amax is None:
            with torch.cuda.stream(st):
                amax = torch.zeros(1, dtype=torch.float64, device=a.device)
        scale = (int(k), amax.data_ptr() if amax is not None else None) + ((scale_exp.data_ptr(),) if auto else ())
        check(getattr(lib, name)(src, a.data_ptr(), code, out.data_ptr(), *shape, *scale, st.cuda_stream), name)
    outs = (out, out_t) if transpose else (out,)
    return outs + (scale_exp,) if auto else outs


def _dequantize(q, name: str, dtype, out, stream, *, k: int = 0, auto=False, scale_exp=None):
    """The two per-tensor dequantize wrappers: FP8 ``q`` (the argument ``name``) by the host's scale exponent ``k``,
    or with ``auto`` by the one the device reads from ``scale_exp``."""
    torch = _torch()
    code = _operand(q, name, _fp8_format)
    dtype, dst = _float_dtype(dtype)
    if auto:
        _one_element(scale_exp, torch.int32, q, "scale_exp")
    out = _out(out, dtype, q)
    fn = "b200va_dequantize_fp8_auto" if auto else "b200va_dequantize_fp8"
    with torch.cuda.device(q.device):
        check(getattr(lib, fn)(code, q.data_ptr(), dst, out.data_ptr(), q.numel(),
                               scale_exp.data_ptr() if auto else int(k), _stream_ptr(stream)), fn)
    return out


def quantize_fp8(a, fmt, *, scale_exp: int = 0, amax=None, out=None, stream=None):
    """``a`` (f32/f64/f16/bf16) times 2^scale_exp, rounded once to FP8 (b200va_quantize_fp8): round-to-nearest-even,
    saturating at +-max finite (448 for E4M3, 57344 for E5M2), inf included; NaN stays NaN.  ``fmt``:
    torch.float8_e4m3fn / torch.float8_e5m2 or "e4m3" / "e5m2".  ``amax``: a one-element float64 CUDA tensor that
    max-accumulates max |a| (unscaled; NaN if any element is); set it to 0 before the first call.  ``out``: a
    contiguous CUDA tensor of the FP8 dtype with a's length on a's device, else a new one.  Asynchronous on the
    current stream."""
    return _quantize(a, fmt, scale_exp, amax, out, stream)[0]


def dequantize_fp8(a, dtype, *, scale_exp: int = 0, out=None, stream=None):
    """FP8 ``a`` (torch.float8_e4m3fn / float8_e5m2) times 2^-scale_exp, rounded once to ``dtype``
    (torch.float32/float64/float16/bfloat16, or "f32"/"f64"/"f16"/"bf16") by b200va_dequantize_fp8: round-to-nearest-
    even, no FTZ, overflow to inf.  ``out``: a contiguous CUDA tensor of ``dtype`` with a's length on a's device, else
    a new one.  Asynchronous on the current stream."""
    return _dequantize(a, "a", dtype, out, stream, k=scale_exp)


def quantize_fp8_auto(a, fmt, *, margin: int = 0, amax=None, scale_exp=None, out=None, stream=None):
    """``a`` (f32/f64/f16/bf16) quantized to FP8 with a power-of-two scale 2^k chosen on the device from the amax
    (b200va_quantize_fp8_auto): an amax pass max-accumulates the largest finite |a| into ``amax``, then k is the
    largest exponent with amax 2^k <= max finite (448 for E4M3, 57344 for E5M2), less ``margin`` (0..126), clamped to
    [-126, 126], and a[i] 2^k is rounded once by quantize_fp8's rules.  With margin >= 0, only +-inf saturates.
    ``amax``: a one-element float64 CUDA tensor, the caller's running max; None makes a zeroed one on the stream
    (current scaling).  ``scale_exp``: a one-element int32 CUDA tensor that receives k, else a new one.  ``out``: as
    in quantize_fp8.  Returns (out, scale_exp) without a host sync; torch.exp2(-scale_exp.float()) is the per-tensor
    dequantization scale a tensor-wise torch._scaled_mm takes.  Asynchronous on the current stream."""
    return _quantize(a, fmt, margin, amax, out, stream, auto=True, scale_exp=scale_exp)


def dequantize_fp8_auto(q, scale_exp, dtype, *, out=None, stream=None):
    """FP8 ``q`` times 2^-k, k the one-element int32 CUDA tensor ``scale_exp`` that quantize_fp8_auto wrote, rounded
    once to ``dtype`` by dequantize_fp8's rules (b200va_dequantize_fp8_auto); k is read on the device, and one outside
    [-126, 126] makes every element NaN.  ``out``: as in dequantize_fp8.  Asynchronous on the current stream."""
    return _dequantize(q, "q", dtype, out, stream, auto=True, scale_exp=scale_exp)


def quantize_fp8_transpose(a, fmt, *, scale_exp: int = 0, amax=None, out=None, out_t=None, stream=None):
    """The 2-D ``a`` (rows x cols, contiguous, f32/f64/f16/bf16) quantized to FP8 as quantize_fp8 does, and the
    transpose of the result, in one pass over a (b200va_quantize_fp8_transpose).  ``out`` ([rows, cols]) gets the bytes
    quantize_fp8 writes for a, ``out_t`` ([cols, rows]) their transpose, both contiguous in the FP8 dtype on a's device
    (new ones when None).  ``amax``: as in quantize_fp8.  Returns (out, out_t).  rows and cols multiples of 16 with
    16-byte aligned operands take the tiled path; any other shape gives the same bytes, slowly.

    On an H100 an FP8 GEMM takes both operands K-major, so the backward products of a linear layer use out_t as is:
    the weight gradient dW = dY^T X is ``torch._scaled_mm(dy_t, x_t.t(), scale_a, scale_b)`` with
    ``dy_t = quantize_fp8_transpose(dy, ...)[1]`` and ``x_t = quantize_fp8_transpose(x, ...)[1]``: x_t.t() is the
    column-major mat2 it requires, with no copy.  Asynchronous on the current stream."""
    return _quantize(a, fmt, scale_exp, amax, out, stream, transpose=True, out_t=out_t)


def quantize_fp8_transpose_auto(a, fmt, *, margin: int = 0, amax=None, scale_exp=None, out=None, out_t=None,
                                stream=None):
    """quantize_fp8_auto of the 2-D ``a`` with the transpose of the result (b200va_quantize_fp8_transpose_auto): the
    amax pass, then one quantize-transpose with the k chosen on the device.  ``amax``, ``scale_exp`` and ``margin`` as
    in quantize_fp8_auto, ``out`` and ``out_t`` as in quantize_fp8_transpose.  Returns (out, out_t, scale_exp) without
    a host sync; torch.exp2(-scale_exp.float()) is the scale torch._scaled_mm takes for out or out_t.t().
    Asynchronous on the current stream."""
    return _quantize(a, fmt, margin, amax, out, stream, transpose=True, out_t=out_t, auto=True, scale_exp=scale_exp)


_U64 = (1 << 64) - 1


def _sr_source(a) -> None:
    """The stochastically rounding casts take float32 sources only."""
    torch = _torch()
    if not isinstance(a, torch.Tensor) or a.dtype != torch.float32:
        raise TypeError(f"a must be a float32 tensor, got {getattr(a, 'dtype', type(a).__name__)}")
    _operand(a, "a")


def convert_sr(a, dtype, *, seed: int, offset: int = 0, out=None, stream=None):
    """float32 ``a`` rounded stochastically to ``dtype`` (torch.float16 / torch.bfloat16, or "f16" / "bf16") by
    b200va_convert_sr_f32: each element rounds to one of its two neighbours, up with probability equal to its
    position between them, past max finite to inf.  The random bits depend only on ``seed`` and the global index
    ``offset + i`` of element i (both taken mod 2^64), so a slice cast with offset equal to its start gives the same
    bytes as the matching slice of a whole-array call.  ``out``: a contiguous CUDA tensor of ``dtype`` with a's
    length on a's device, else a new one.  Asynchronous on the current stream."""
    _sr_source(a)
    dtype, dst = _float_dtype(dtype)
    if dst not in (capi.DTYPES["f16"], capi.DTYPES["bf16"]):
        raise TypeError(f"dtype must be float16 or bfloat16, got {dtype}")
    out = _out(out, dtype, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_convert_sr_f32(a.data_ptr(), dst, out.data_ptr(), a.numel(), int(seed) & _U64,
                                        int(offset) & _U64, _stream_ptr(stream)), "b200va_convert_sr_f32")
    return out


def quantize_fp8_sr(a, fmt, *, seed: int, offset: int = 0, scale_exp: int = 0, amax=None, out=None, stream=None):
    """float32 ``a`` times 2^scale_exp rounded stochastically to FP8 (b200va_quantize_fp8_sr_f32): the random bits and
    rounding of convert_sr, then saturation at +-max finite (448 for E4M3, 57344 for E5M2), inf included; NaN stays
    NaN.  ``fmt``: torch.float8_e4m3fn / torch.float8_e5m2 or "e4m3" / "e5m2".  ``amax``: as in quantize_fp8.
    ``out``: a contiguous CUDA tensor of the FP8 dtype with a's length on a's device, else a new one.  Asynchronous on
    the current stream."""
    _sr_source(a)
    dtype, code = _fp8_format(fmt)
    out = _out(out, dtype, a)
    _amax(amax, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_quantize_fp8_sr_f32(a.data_ptr(), code, out.data_ptr(), a.numel(), int(scale_exp),
                                             int(seed) & _U64, int(offset) & _U64,
                                             amax.data_ptr() if amax is not None else None, _stream_ptr(stream)),
              "b200va_quantize_fp8_sr_f32")
    return out


def _mx_scales(scales, a, block: int):
    """``scales`` checked to be a contiguous one-byte tensor (uint8, or float8_e8m0fnu where torch has it) of
    b200va_mxfp8_scale_bytes(n, block) elements on a's device, or a new uint8 one."""
    torch = _torch()
    if block not in capi.MX_BLOCKS:
        raise ValueError(f"block must be one of {capi.MX_BLOCKS}, got {block}")
    count = lib.b200va_mxfp8_scale_bytes(a.numel(), block)
    if scales is None:
        return torch.empty(count, dtype=torch.uint8, device=a.device)
    byte_dtypes = (torch.uint8,) + ((torch.float8_e8m0fnu,) if hasattr(torch, "float8_e8m0fnu") else ())
    if (not isinstance(scales, torch.Tensor) or scales.dtype not in byte_dtypes or scales.numel() != count
            or scales.device != a.device or not scales.is_contiguous()):
        raise TypeError(f"scales must be a contiguous uint8 (E8M0) tensor of {count} elements on a's device")
    return scales


def quantize_mxfp8(a, fmt, *, block: int = 32, scale_rule: str = "ocp", out=None, scales=None, stream=None):
    """``a`` (f32/f64/f16/bf16) quantized to block-scaled FP8 in one pass (b200va_quantize_mxfp8): every ``block``
    (32, 64 or 128) consecutive elements, counted from element 0, share one E8M0 scale 2^e chosen from the block's
    largest finite magnitude, and each element is a 2^-e rounded once to ``fmt`` (torch.float8_e4m3fn /
    torch.float8_e5m2 or "e4m3" / "e5m2") by quantize_fp8's rules.  ``scale_rule``: "ocp" (e = floor(log2 amax) -
    emax, the OCP MX rule) or "nosat" (the smallest e under which the block's finite values do not saturate).
    ``out``: a contiguous CUDA tensor of the FP8 dtype with a's length; ``scales``: a contiguous uint8 tensor of
    ceil(n / block) elements (value e + 127); new ones otherwise.  Returns (q, scales).  Asynchronous on the current
    stream."""
    src = _operand(a, "a")
    dtype, code = _fp8_format(fmt)
    if scale_rule not in capi.MX_SCALE:
        raise ValueError(f"scale_rule must be one of {sorted(capi.MX_SCALE)}, got {scale_rule!r}")
    scales = _mx_scales(scales, a, block)
    out = _out(out, dtype, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_quantize_mxfp8(src, a.data_ptr(), code, out.data_ptr(), scales.data_ptr(), a.numel(), block,
                                        capi.MX_SCALE[scale_rule], _stream_ptr(stream)), "b200va_quantize_mxfp8")
    return out, scales


def dequantize_mxfp8(q, scales, dtype, *, block: int = 32, out=None, stream=None):
    """Block-scaled FP8 ``q`` (torch.float8_e4m3fn / float8_e5m2) with its E8M0 ``scales`` (uint8, one per ``block``
    elements) back to ``dtype`` (torch.float32/float64/float16/bfloat16, or "f32"/"f64"/"f16"/"bf16") by
    b200va_dequantize_mxfp8: q[i] 2^(scales[i // block] - 127) rounded once (round-to-nearest-even, no FTZ, overflow
    to inf); a scale byte 0xFF makes its block NaN.  ``out``: a contiguous CUDA tensor of ``dtype`` with q's length
    on q's device, else a new one.  Asynchronous on the current stream."""
    code = _operand(q, "q", _fp8_format)
    dtype, dst = _float_dtype(dtype)
    if scales is None:
        raise TypeError("scales must be given")
    scales = _mx_scales(scales, q, block)
    out = _out(out, dtype, q)
    with _torch().cuda.device(q.device):
        check(lib.b200va_dequantize_mxfp8(code, q.data_ptr(), scales.data_ptr(), dst, out.data_ptr(), q.numel(), block,
                                          _stream_ptr(stream)), "b200va_dequantize_mxfp8")
    return out


def fp8_blockwise_scale_layout(rows: int, cols: int, block: str) -> tuple[int, tuple[int, int], tuple[int, int]]:
    """(numel, shape, stride) of the f32 scales of a rows x cols operand quantized in ``block`` ("1x128" or
    "128x128") blocks: the storage b200va_quantize_fp8_blockwise writes, and the as_strided view of it that
    torch.nn.functional.scaled_mm takes (MN-major).  1x128: S[b * rows + i], an [rows, ceil(cols/128)] view with strides
    [1, rows].  128x128: S[p * L4 + q], an [L4, ceil(rows/128)] view with strides [1, L4], L4 = ceil(ceil(cols/128) / 4)
    4 (the entries q >= ceil(cols/128) are padding).  The transposed operand's layout is this with rows and cols
    swapped."""
    if block not in capi.FP8_BLOCK:
        raise ValueError(f"block must be one of {sorted(capi.FP8_BLOCK)}, got {block!r}")
    nkb_r, nkb_c = -(-rows // 128), -(-cols // 128)
    if block == "1x128":
        return rows * nkb_c, (rows, nkb_c), (1, max(rows, 1))
    l4 = -(-nkb_c // 4) * 4
    return nkb_r * l4, (l4, nkb_r), (1, l4)


def _blockwise_scales(scales, rows: int, cols: int, block: str, dev, name: str):
    """``scales`` checked to be a float32 tensor on ``dev`` whose storage holds the layout's count from its storage
    offset, viewed in the layout; or a new one."""
    torch = _torch()
    numel, shape, stride = fp8_blockwise_scale_layout(rows, cols, block)
    if scales is None:
        return torch.empty(numel, dtype=torch.float32, device=dev).as_strided(shape, stride)
    if (not isinstance(scales, torch.Tensor) or scales.dtype != torch.float32 or scales.device != dev
            or scales.untyped_storage().nbytes() // 4 - scales.storage_offset() < numel):
        raise TypeError(f"{name} must be a float32 tensor on {dev} with storage for {numel} scales")
    return scales.as_strided(shape, stride)


def quantize_fp8_blockwise(a, fmt, *, block: str = "1x128", rowwise: bool = True, columnwise: bool = True, out=None,
                           scales=None, out_t=None, scales_t=None, stream=None):
    """The 2-D ``a`` (rows x cols, contiguous, f32/f64/f16/bf16) quantized to FP8 with one f32 power-of-two scale per
    block (b200va_quantize_fp8_blockwise), the operands of an H100 blockwise-scaled FP8 GEMM.  ``block``: "1x128"
    (activations, gradients) or "128x128" (weights).  Per block, k is the largest exponent with amax 2^k <= max finite
    (amax over the finite elements), clamped to [-126, 126]; the scale is 2^-k and each element a 2^k rounded once by
    quantize_fp8's rules.  ``rowwise``: ``out`` ([rows, cols]) and ``scales`` in A's blocks; ``columnwise``: ``out_t``
    ([cols, rows]) and ``scales_t`` in the blocks of A^T (for 1x128, 128 x 1 blocks of a along its columns); both in
    one pass over a.  Returns (out, scales, out_t, scales_t), None for a side not asked for; each scale tensor is the
    view fp8_blockwise_scale_layout gives, so ``out`` with ``scales`` and ``out_t.t()`` with ``scales_t`` go to
    torch.nn.functional.scaled_mm as they are.  Asynchronous on the current stream."""
    torch = _torch()
    src, rows, cols = _matrix(a)
    dtype, code = _fp8_format(fmt)
    if block not in capi.FP8_BLOCK:
        raise ValueError(f"block must be one of {sorted(capi.FP8_BLOCK)}, got {block!r}")
    if not rowwise and not columnwise:
        raise ValueError("at least one of rowwise and columnwise must be set")
    if rowwise:
        out = _out_shaped(out, dtype, (rows, cols), a, "out")
        scales = _blockwise_scales(scales, rows, cols, block, a.device, "scales")
    else:
        out = scales = None
    if columnwise:
        out_t = _out_shaped(out_t, dtype, (cols, rows), a, "out_t")
        scales_t = _blockwise_scales(scales_t, cols, rows, block, a.device, "scales_t")
    else:
        out_t = scales_t = None
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    with torch.cuda.device(a.device):
        check(lib.b200va_quantize_fp8_blockwise(src, a.data_ptr(), code, capi.FP8_BLOCK[block], rows, cols, ptr(out),
                                                ptr(scales), ptr(out_t), ptr(scales_t), _stream_ptr(stream)),
              "b200va_quantize_fp8_blockwise")
    return out, scales, out_t, scales_t


def dequantize_fp8_blockwise(q, scales, dtype, *, block: str, out=None, stream=None):
    """The 2-D FP8 ``q`` (rows x cols, torch.float8_e4m3fn / float8_e5m2) with its f32 block ``scales`` (the view
    quantize_fp8_blockwise returns, or any float32 tensor whose storage holds the layout) back to ``dtype``
    (b200va_dequantize_fp8_blockwise): q s rounded once, s the scale of q's block, any f32 (not only a power of two).
    For ``out_t`` pass ``scales_t``.  ``out``: a contiguous [rows, cols] tensor of ``dtype`` on q's device, else a new
    one.  Asynchronous on the current stream."""
    torch = _torch()
    code = _operand(q, "q", _fp8_format)
    if q.dim() != 2:
        raise TypeError(f"q must be a 2-D tensor, got {q.dim()} dimensions")
    rows, cols = q.shape
    dtype, dst = _float_dtype(dtype)
    if scales is None:
        raise TypeError("scales must be given")
    scales = _blockwise_scales(scales, rows, cols, block, q.device, "scales")
    out = _out_shaped(out, dtype, (rows, cols), q, "out")
    with torch.cuda.device(q.device):
        check(lib.b200va_dequantize_fp8_blockwise(code, q.data_ptr(), scales.data_ptr(), capi.FP8_BLOCK[block], dst,
                                                  out.data_ptr(), rows, cols, _stream_ptr(stream)),
              "b200va_dequantize_fp8_blockwise")
    return out


def _f32_vector(t, n: int, dev, name: str):
    """``t`` checked to be a contiguous float32 tensor of n elements on ``dev``, viewed 1-D; or a new one."""
    torch = _torch()
    if t is None:
        return torch.empty(n, dtype=torch.float32, device=dev)
    if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.numel() != n or t.device != dev
            or not t.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous float32 tensor of {n} elements on {dev}")
    return t.view(n)


def quantize_fp8_rowwise(a, fmt, *, rowwise: bool = True, columnwise: bool = True, out=None, scales=None, out_t=None,
                         scales_t=None, workspace=None, stream=None):
    """The 2-D ``a`` (rows x cols, contiguous, f32/f64/f16/bf16) quantized to FP8 with one f32 power-of-two scale per
    row (b200va_quantize_fp8_rowwise), the operands of an H100 row-wise scaled FP8 GEMM.  Per row, k is the largest
    exponent with amax 2^k <= max finite (amax over the row's finite elements), clamped to [-126, 126]; the scale is
    2^-k and each element a 2^k rounded once by quantize_fp8's rules.  ``rowwise``: ``out`` ([rows, cols]) and
    ``scales`` ([rows]); ``columnwise``: ``out_t`` ([cols, rows], A^T's rows) and ``scales_t`` ([cols], one per column
    of a).  Returns (out, scales, out_t, scales_t), None for a side not asked for.  The scales are 1-D float32, so for a
    linear layer Y = X W^T, with torch.nn.functional.scaled_mm and ScalingType.RowWise (or torch._scaled_mm):

        Y  = scaled_mm(C_X,  C_W.t(),   scale_a=S_X.view(-1, 1),   scale_b=S_W.view(1, -1))
        dX = scaled_mm(C_dY, Ct_W.t(),  scale_a=S_dY.view(-1, 1),  scale_b=St_W.view(1, -1))
        dW = scaled_mm(Ct_dY, Ct_X.t(), scale_a=St_dY.view(-1, 1), scale_b=St_X.view(1, -1))

    where (C_T, S_T, Ct_T, St_T) is this call's result for tensor T, both sides asked for.  ``workspace``: a contiguous
    CUDA tensor of at least b200va_fp8_rowwise_workspace(rows, cols) bytes, else one is taken from the torch allocator
    on the call's stream.  Three launches, asynchronous on the current stream."""
    torch = _torch()
    src, rows, cols = _matrix(a)
    dtype, code = _fp8_format(fmt)
    if not rowwise and not columnwise:
        raise ValueError("at least one of rowwise and columnwise must be set")
    if rowwise:
        out = _out_shaped(out, dtype, (rows, cols), a, "out")
        scales = _f32_vector(scales, rows, a.device, "scales")
    else:
        out = scales = None
    if columnwise:
        out_t = _out_shaped(out_t, dtype, (cols, rows), a, "out_t")
        scales_t = _f32_vector(scales_t, cols, a.device, "scales_t")
    else:
        out_t = scales_t = None
    need = lib.b200va_fp8_rowwise_workspace(rows, cols)
    if workspace is not None and (not isinstance(workspace, torch.Tensor) or workspace.device != a.device
                                  or not workspace.is_contiguous()):
        raise TypeError("workspace must be a contiguous tensor on a's device")
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    with torch.cuda.device(a.device):
        if workspace is None:
            # allocated on the stream the call runs on, so the allocator reuses it only after that stream's work
            with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
                workspace = torch.empty(max(need, 4), dtype=torch.uint8, device=a.device)
        check(lib.b200va_quantize_fp8_rowwise(src, a.data_ptr(), code, rows, cols, ptr(out), ptr(scales), ptr(out_t),
                                              ptr(scales_t), workspace.data_ptr(),
                                              workspace.numel() * workspace.element_size(), _stream_ptr(stream)),
              "b200va_quantize_fp8_rowwise")
    return out, scales, out_t, scales_t


def dequantize_fp8_rowwise(q, scales, dtype, *, out=None, stream=None):
    """The 2-D FP8 ``q`` (rows x cols, torch.float8_e4m3fn / float8_e5m2) with one f32 scale per row (``scales``,
    rows elements) back to ``dtype`` (b200va_dequantize_fp8_rowwise): q s rounded once, s any f32 (not only a power of
    two).  For ``out_t`` pass ``scales_t``.  ``out``: a contiguous [rows, cols] tensor of ``dtype`` on q's device, else a
    new one.  Asynchronous on the current stream."""
    torch = _torch()
    code = _operand(q, "q", _fp8_format)
    if q.dim() != 2:
        raise TypeError(f"q must be a 2-D tensor, got {q.dim()} dimensions")
    rows, cols = q.shape
    dtype, dst = _float_dtype(dtype)
    if scales is None:
        raise TypeError("scales must be given")
    scales = _f32_vector(scales, rows, q.device, "scales")
    out = _out_shaped(out, dtype, (rows, cols), q, "out")
    with torch.cuda.device(q.device):
        check(lib.b200va_dequantize_fp8_rowwise(code, q.data_ptr(), scales.data_ptr(), dst, out.data_ptr(), rows, cols,
                                                _stream_ptr(stream)), "b200va_dequantize_fp8_rowwise")
    return out


def dot(a, b, *, out=None, workspace=None, stream=None):
    """The reproducible dot product of two equal-length contiguous CUDA tensors of one of f32/f64/f16/bf16
    (b200va_dot): a 0-d float64 CUDA tensor, written asynchronously on the current stream.  The bits
    depend on the values and the length only.  ``out``: a float64 CUDA tensor of at least one element to
    write the result into (its first element); ``workspace``: a CUDA tensor of at least
    b200va_dot_workspace_bytes(n) bytes, else one is taken from the torch allocator for this call."""
    torch = _torch()
    code = _operand(a, "a")
    _like(b, a.dtype, a, "b")
    n = a.numel()
    need = lib.b200va_dot_workspace_bytes(n)
    if out is None:
        out = torch.empty((), dtype=torch.float64, device=a.device)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float64 or out.device != a.device
          or out.numel() < 1 or not out.is_contiguous()):
        raise TypeError("out must be a contiguous float64 tensor on a's device")
    if workspace is not None and (not isinstance(workspace, torch.Tensor) or workspace.device != a.device
                                  or not workspace.is_contiguous()):
        raise TypeError("workspace must be a contiguous tensor on a's device")
    with torch.cuda.device(a.device):
        if workspace is None:
            # allocated on the stream the call runs on, so the allocator reuses it only after that stream's work
            with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
                workspace = torch.empty(max(need, 8), dtype=torch.uint8, device=a.device)
        check(lib.b200va_dot(code, a.data_ptr(), b.data_ptr(), n, out.data_ptr(),
                             workspace.data_ptr(), workspace.numel() * workspace.element_size(), _stream_ptr(stream)),
              "b200va_dot")
    return out


def probe(kind: str, a, b, c, *, stream=None):
    """Ceiling probe (b200va_probe_f32): 'read2' loads a and b, 'fill' stores c, 'copy' c = a.  c is clobbered.
    The operands the kind uses are checked like add's (float32, contiguous, c's length on c's device); the others
    are ignored."""
    torch = _torch()
    code = capi.PROBES[kind]
    used = {"a": a, "b": b} if kind == "read2" else {"a": a} if kind == "copy" else {}
    *_, pc = _f32_operands("c", **used, c=c)
    pa, pb = (used[k].data_ptr() if k in used else None for k in ("a", "b"))
    with torch.cuda.device(c.device):
        check(lib.b200va_probe_f32(code, pa, pb, pc, c.numel(), _stream_ptr(stream)), "b200va_probe_f32")


def fill_ctr(out, seed: int, first: int = 0, *, stream=None):
    """Counter generator on the device: out[i] = ctr(seed, first + i)."""
    torch = _torch()
    with torch.cuda.device(out.device):
        check(lib.b200va_fill_ctr_f32(_dev_ptr(out, "out"), out.numel(), seed, first, _stream_ptr(stream)),
              "b200va_fill_ctr_f32")
    return out


def fill_ctr_host(n: int, seed: int, first: int = 0) -> np.ndarray:
    x = np.empty(n, dtype=np.float32)
    check(lib.b200va_host_fill_ctr_f32(x.ctypes.data, n, seed, first), "b200va_host_fill_ctr_f32")
    return x


def fill_rand_host(n: int) -> tuple[np.ndarray, np.ndarray]:
    """The sample's input recipe (interleaved, never-seeded rand())."""
    a, b = np.empty(n, dtype=np.float32), np.empty(n, dtype=np.float32)
    check(lib.b200va_host_fill_rand_f32(a.ctypes.data, b.ctypes.data, n), "b200va_host_fill_rand_f32")
    return a, b


def verify(a, b, c, *, stream=None) -> tuple[int, int]:
    """Device-side bitwise check; returns (mismatch count, first bad index or -1). Synchronises."""
    torch = _torch()
    pa, pb, pc = _f32_operands("a", a=a, b=b, c=c)
    res = torch.empty(2, dtype=torch.int64, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.b200va_verify_f32(pa, pb, pc, a.numel(), res.data_ptr(), _stream_ptr(stream)), "b200va_verify_f32")
    bad, first = (int(v) & 0xFFFFFFFFFFFFFFFF for v in res.tolist())
    return bad, (-1 if bad == 0 else first)


def digest(x, *, stream=None) -> tuple[int, int]:
    """(sum of uint32 bit patterns mod 2^64, xor of them) computed in HBM. Synchronises."""
    torch = _torch()
    res = torch.empty(2, dtype=torch.int64, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.b200va_digest_f32(_dev_ptr(x, "x"), x.numel(), res.data_ptr(), _stream_ptr(stream)),
              "b200va_digest_f32")
    s, xo = (int(v) & 0xFFFFFFFFFFFFFFFF for v in res.tolist())
    return s, xo


def verify_host(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> int:
    """The sample's self-check made strict (bitwise). Returns -1 or the first bad index."""
    bad = C.c_size_t(0)
    rc = lib.b200va_host_verify_f32(a.ctypes.data, b.ctypes.data, c.ctypes.data, a.size, C.byref(bad))
    if rc == capi.OK:
        return -1
    if rc == capi.ERR_VERIFY:
        return bad.value
    check(rc, "b200va_host_verify_f32")
    return -1


def _host_ptr(x, name: str) -> int:
    torch = _torch()
    if isinstance(x, np.ndarray):
        if x.dtype != np.float32 or not x.flags.c_contiguous:
            raise TypeError(f"{name} must be a C-contiguous float32 array")
        return x.ctypes.data
    if isinstance(x, torch.Tensor) and not x.is_cuda and x.dtype == torch.float32 and x.is_contiguous():
        return x.data_ptr()
    raise TypeError(f"{name} must be a float32 numpy array or CPU tensor")


class PinnedBuffer:
    """Pinned, GPU-local-NUMA host memory from b200va_host_alloc, viewed as a float32 numpy
    array (``.array``).  The memory lives until ``free()`` / garbage collection."""

    def __init__(self, n: int, write_combined: bool = False):
        self._p = C.c_void_p()
        self.n = n
        check(lib.b200va_host_alloc_ex(C.byref(self._p), max(1, n) * 4, 1 if write_combined else 0), "b200va_host_alloc_ex")
        self.array = np.ctypeslib.as_array(C.cast(self._p, C.POINTER(C.c_float)), shape=(n,))

    @property
    def numa_node(self) -> int:
        """NUMA node of the first page (-1 if unknown)."""
        return int(lib.b200va_host_node_of(self._p)) if self._p else -1

    def free(self):
        if self._p:
            self.array = None
            lib.b200va_host_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Stager:
    """Host-buffer path (a3 + a4 + a6-copy): H2D, add and D2H pipelined in chunks."""

    def __init__(self, device: int = 0, chunk_elems: int = 0, depth: int = 0):
        self._h = C.c_void_p()
        check(lib.b200va_stager_create(C.byref(self._h), device, chunk_elems, depth), "b200va_stager_create")

    def add(self, a, b, out, *, variant=K_AUTO, zero_copy: bool = False, mode: int | None = None) -> float:
        """Synchronous; returns the device-timed milliseconds of the whole pipeline.
        mode: -1 auto (default), 0 slot streams, 1 zero-copy kernel, 2 lanes (one stream per
        direction), 3 pageable arrays through a pinned bounce ring, 4 register-once."""
        n = a.size if isinstance(a, np.ndarray) else a.numel()
        if mode is None:
            mode = capi.STAGE_ZEROCOPY if zero_copy else capi.STAGE_AUTO
        check(lib.b200va_stager_add_f32(self._h, _host_ptr(a, "a"), _host_ptr(b, "b"), _host_ptr(out, "out"), n,
                                        _variant(variant), mode), "b200va_stager_add_f32")
        ms = C.c_float()
        check(lib.b200va_stager_last_ms(self._h, C.byref(ms)), "b200va_stager_last_ms")
        return ms.value

    @property
    def last_mode(self) -> int:
        """The pipeline the last ``add`` actually ran (after AUTO / fallbacks)."""
        m = C.c_int(-2)
        check(lib.b200va_stager_last_mode(self._h, C.byref(m)), "b200va_stager_last_mode")
        return m.value

    def release_host(self) -> None:
        """Unregister the host arrays the register-once path page-locked."""
        check(lib.b200va_stager_release_host(self._h), "b200va_stager_release_host")

    def close(self):
        if self._h:
            lib.b200va_stager_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def add_host(a: np.ndarray, b: np.ndarray, out: np.ndarray | None = None, *, device: int = 0, variant=K_AUTO):
    """One ``./vectorAdd`` worth of work on host arrays: alloc, H2D, add, D2H, free."""
    if out is None:
        out = np.empty_like(a)
    check(lib.b200va_add_f32_host(_host_ptr(a, "a"), _host_ptr(b, "b"), _host_ptr(out, "out"), a.size, device,
                                  _variant(variant)), "b200va_add_f32_host")
    return out


def run_cli(*args: str, timeout: float = 600.0) -> subprocess.CompletedProcess:
    """Run the drop-in ``vectorAdd`` executable (the outer boundary)."""
    return subprocess.run([capi.CLI_PATH, *args], capture_output=True, text=True, timeout=timeout)
