"""The order of the per-tensor FP8 casts' argument checks, when a call breaks more than one rule.

b200va_quantize_fp8, b200va_dequantize_fp8, their _auto forms, b200va_quantize_fp8_transpose and its _auto form, and
b200va_quantize_fp8_sr_f32 check their arguments in one order (include/b200va.h):
  1. the dtype and format codes (B200VA_ERR_VARIANT);
  2. k, or the margin, out of range, and for _auto a NULL d_amax or d_scale_exp (B200VA_ERR_INVALID);
  3. A and C as b200va_convert checks them: NULL, then alignment, then n > 2^40, then C meeting A;
  4. d_amax alignment, then d_amax meeting A or C;
  5. d_scale_exp alignment, then d_scale_exp meeting A, C or d_amax;
  6. Ct NULL, then Ct meeting another operand.
Per entry point, cases() lists single faults in that order, one or two per argument.  Each single fault must return
its code, and each pair of faults on different arguments the code of the one listed first.  No rejected call may
write: every pointer lies inside one poisoned allocation, which must keep its poison after every call.  n is small
except in the n > 2^40 fault.  The other rejected-argument tables (test_gpu_typecast_fp8*.py,
test_gpu_round_stochastic.py) cover each rule on its own.
"""
import itertools

import pytest

from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import POISON
    from k8s_gpu_hpa_b200 import capi

VARIANT, INVALID, ALIGN, OVERLAP = "VARIANT", "INVALID", "ALIGN", "OVERLAP"       # B200VA_ERR_*
F32, E4, N, R, COLS = 0, 0, 1000, 16, 64
HUGE = (1 << 40) + 1


def cases(A, C, T, M, S):
    """(entry point, arguments without the stream, faults) per entry point: A, C, Ct, d_amax and d_scale_exp sit at
    A, C, T, M and S, apart from one another.  A fault is (argument name, values, code); values replace the named
    arguments.  Faults come in check order."""
    quant = [("C", (None,), INVALID), ("A", (A + 2,), ALIGN), ("n", (HUGE,), INVALID), ("C", (A + 8,), OVERLAP)]
    amax = [("amax", (M + 4,), ALIGN), ("amax", (A + 8,), OVERLAP)]
    scale = [("scale", (S + 2,), ALIGN), ("scale", (M,), OVERLAP)]
    dequant = [("A", (None,), INVALID), ("C", (C + 2,), ALIGN), ("n", (HUGE,), INVALID), ("C", (A + 4,), OVERLAP)]
    shape = [("C", (None,), INVALID), ("A", (A + 2,), ALIGN), ("shape", (1 << 20, (1 << 20) + 16), INVALID),
             ("shape", (1 << 32, 1 << 32), INVALID), ("C", (A + 8,), OVERLAP)]
    ct = [("Ct", (None,), INVALID), ("Ct", (C + 16,), OVERLAP)]
    codes = [("src", (4,), VARIANT), ("fmt", (2,), VARIANT)]
    host_k = [("k", (127,), INVALID)]
    auto_k = [("k", (127,), INVALID), ("amax", (None,), INVALID), ("scale", (None,), INVALID)]
    return [
        ("b200va_quantize_fp8", dict(src=F32, A=A, fmt=E4, C=C, n=N, k=0, amax=M),
         codes + host_k + quant + amax),
        ("b200va_dequantize_fp8", dict(fmt=E4, A=A, dst=F32, C=C, n=N, k=0),
         [("dst", (4,), VARIANT), ("fmt", (2,), VARIANT), ("k", (-127,), INVALID)] + dequant),
        ("b200va_quantize_fp8_auto", dict(src=F32, A=A, fmt=E4, C=C, n=N, k=0, amax=M, scale=S),
         codes + auto_k + quant + amax + scale),
        ("b200va_dequantize_fp8_auto", dict(fmt=E4, A=A, dst=F32, C=C, n=N, scale=S),
         [("dst", (4,), VARIANT), ("fmt", (2,), VARIANT), ("scale", (None,), INVALID)] + dequant
         + [("scale", (S + 1,), ALIGN), ("scale", (A + 4,), OVERLAP)]),
        ("b200va_quantize_fp8_transpose", dict(src=F32, A=A, fmt=E4, C=C, Ct=T, shape=(R, COLS), k=0, amax=M),
         codes + host_k + shape + amax + ct),
        ("b200va_quantize_fp8_transpose_auto",
         dict(src=F32, A=A, fmt=E4, C=C, Ct=T, shape=(R, COLS), k=0, amax=M, scale=S),
         codes + auto_k + shape + amax + scale + ct),
        ("b200va_quantize_fp8_sr_f32", dict(A=A, fmt=E4, C=C, n=N, k=0, seed=1, first=0, amax=M),
         [("fmt", (2,), VARIANT)] + host_k + quant + amax),
    ]


def arguments(base, *faults):
    """The positional arguments of base with the faults applied (the shape slot holds rows and cols)."""
    args = dict(base)
    for name, values, _ in faults:
        args[name] = values if name == "shape" else values[0]
    return [v for name, x in args.items() for v in (x if name == "shape" else (x,))]


def calls(A, C, T, M, S):
    """(entry point, arguments, expected code, what) of every single fault and every pair of faults on different
    arguments."""
    out = []
    for fn, base, faults in cases(A, C, T, M, S):
        for f in faults:
            out.append((fn, arguments(base, f), f[2], f"{f[0]}={f[1]}"))
        for f, g in itertools.combinations(faults, 2):
            if f[0] != g[0]:
                out.append((fn, arguments(base, f, g), f[2], f"{f[0]}={f[1]} before {g[0]}={g[1]}"))
    return out


def test_the_first_broken_rule_decides_the_code_and_nothing_is_written():
    buf = torch.empty(1 << 17, dtype=torch.uint8, device="cuda")
    buf.fill_(POISON)
    torch.cuda.synchronize()
    A = buf.data_ptr() + 4096
    C, T, M, S = A + 16384, A + 32768, A + 49152, A + 49168
    failures = []
    for fn, args, code, what in calls(A, C, T, M, S):
        got = getattr(capi.lib, fn)(*args, None)
        if got != getattr(capi, "ERR_" + code):
            failures.append(f"{fn} {what}: {got}, want {code}")
        assert bool((buf == POISON).all()), f"{fn} {what} wrote to device memory"
    assert not failures, "\n".join(failures[:40])
    # the arguments without a fault are accepted, so every code above comes from its fault
    for fn, base, _ in cases(A, C, T, M, S):
        assert getattr(capi.lib, fn)(*arguments(base), None) == capi.OK, fn
    torch.cuda.synchronize()
