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
    if a.numel() != b.numel():
        raise ValueError("a and b differ in length")
    if out is None:
        out = torch.empty_like(a)
    if out.numel() != a.numel():
        raise ValueError("out differs in length")
    pa, pb, pc = _dev_ptr(a, "a"), _dev_ptr(b, "b"), _dev_ptr(out, "out")
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
    pa, pb, pc = _dev_ptr(a, "a"), _dev_ptr(b, "b"), _dev_ptr(out, "out")
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
        self._keep = (a, b, out)
        self._device = a.device
        with torch.cuda.device(a.device):
            check(lib.b200va_loop_create(C.byref(self._h), _dev_ptr(a, "a"), _dev_ptr(b, "b"), _dev_ptr(out, "out"), a.numel(),
                                         _variant(variant), graph_batch), "b200va_loop_create")

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


def quantize_fp8(a, fmt, *, scale_exp: int = 0, amax=None, out=None, stream=None):
    """``a`` (f32/f64/f16/bf16) times 2^scale_exp, rounded once to FP8 (b200va_quantize_fp8): round-to-nearest-even,
    saturating at +-max finite (448 for E4M3, 57344 for E5M2), inf included; NaN stays NaN.  ``fmt``:
    torch.float8_e4m3fn / torch.float8_e5m2 or "e4m3" / "e5m2".  ``amax``: a one-element float64 CUDA tensor that
    max-accumulates max |a| (unscaled; NaN if any element is); set it to 0 before the first call.  ``out``: a
    contiguous CUDA tensor of the FP8 dtype with a's length on a's device, else a new one.  Asynchronous on the
    current stream."""
    torch = _torch()
    src = _operand(a, "a")
    dtype, code = _fp8_format(fmt)
    out = _out(out, dtype, a)
    if amax is not None and (not isinstance(amax, torch.Tensor) or amax.dtype != torch.float64 or amax.numel() != 1
                             or amax.device != a.device):
        raise TypeError("amax must be a one-element float64 tensor on a's device")
    with torch.cuda.device(a.device):
        check(lib.b200va_quantize_fp8(src, a.data_ptr(), code, out.data_ptr(), a.numel(), int(scale_exp),
                                      amax.data_ptr() if amax is not None else None, _stream_ptr(stream)),
              "b200va_quantize_fp8")
    return out


def dequantize_fp8(a, dtype, *, scale_exp: int = 0, out=None, stream=None):
    """FP8 ``a`` (torch.float8_e4m3fn / float8_e5m2) times 2^-scale_exp, rounded once to ``dtype``
    (torch.float32/float64/float16/bfloat16, or "f32"/"f64"/"f16"/"bf16") by b200va_dequantize_fp8: round-to-nearest-
    even, no FTZ, overflow to inf.  ``out``: a contiguous CUDA tensor of ``dtype`` with a's length on a's device, else
    a new one.  Asynchronous on the current stream."""
    code = _operand(a, "a", _fp8_format)
    dtype, dst = _float_dtype(dtype)
    out = _out(out, dtype, a)
    with _torch().cuda.device(a.device):
        check(lib.b200va_dequantize_fp8(code, a.data_ptr(), dst, out.data_ptr(), a.numel(), int(scale_exp),
                                        _stream_ptr(stream)), "b200va_dequantize_fp8")
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
    """Ceiling probe (b200va_probe_f32): 'read2' loads a and b, 'fill' stores c, 'copy' c = a.  c is clobbered."""
    torch = _torch()
    with torch.cuda.device(c.device):
        check(lib.b200va_probe_f32(capi.PROBES[kind], a.data_ptr() if a is not None else None, b.data_ptr() if b is not None else None,
                                   _dev_ptr(c, "c"), c.numel(), _stream_ptr(stream)), "b200va_probe_f32")


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
    res = torch.empty(2, dtype=torch.int64, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.b200va_verify_f32(_dev_ptr(a, "a"), _dev_ptr(b, "b"), _dev_ptr(c, "c"), a.numel(),
                                    res.data_ptr(), _stream_ptr(stream)), "b200va_verify_f32")
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
