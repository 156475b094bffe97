"""Rate of the cast kernels by family, next to the f32 COPY and READ2 ceiling probes, in one process.

    python tools/cast_rate.py [--family convert|fp8|fp8t|fp8b|fp8r|mxfp8|sr|all] [--log2n 28] [--calls 20] [--rounds 3]
                              [--shape ROWSxCOLS]

Per round, every op of the chosen families is timed at n elements with CUDA events around `calls` back-to-back calls
(after two warm-up calls), then b200va_probe_f32 COPY (8 n bytes) and READ2 (8 n read) at the same n.  The families
and the algorithmic bytes of one call:
  convert  every ordered pair of distinct types of f32, f64, f16, bf16: n * (sizeof SRC + sizeof DST);
  fp8      per type and format (E4M3, E5M2): quantize without amax, quantize with amax, dequantize back:
           n * (sizeof T + 1); then the per-tensor scale taken from the amax, two ways: the two-pass recipe,
           b200va_quantize_fp8 with amax into a scratch output (the pass that finds the scale) followed by the real
           b200va_quantize_fp8, 2 n * (sizeof T + 1) bytes as it runs here (without the host read of the amax that
           a caller needs between the two); and b200va_quantize_fp8_auto, its amax pass and the quantize with the
           k chosen on the device, n * (2 sizeof T + 1).  "us" is the time of the whole recipe, "TB/s" counts what
           it moves; neither resets the amax between calls (a running max).  Last, b200va_dequantize_fp8_auto with
           the device k, n * (sizeof T + 1).
  fp8t     the quantize-transpose at 8192 x 8192, 16384 x 16384, 4096 x 32768 and 32768 x 4096 (not at n) from each
           type to E4M3, and to E5M2 at 8192 x 8192, next to: b200va_quantize_fp8 alone (the floor: read A, write
           C), the same followed by torch's transpose of the FP8 result into a preallocated tensor, the _auto form,
           and b200va_quantize_fp8_auto followed by torch's transpose.  Every entry counts n * (sizeof T + 2) bytes,
           what the fused call moves, so the rates compare times.
  fp8b     the blockwise quantize at FP8T_SHAPES (or --shape) from each type to E4M3, and to E5M2 at 8192 x 8192:
           1x128 with both sides, row-wise only and column-wise only, and 128x128 with Ct; beside them at the same
           shape the quantize-transpose (the same bytes less the scales), quantize_mxfp8 at block 128 on the flattened
           A (the yardstick of the row-wise-only case), and the torch-eager recipe for both 1x128 sides (view as
           blocks, amax, exp2 of the scale exponent, multiply, .to(float8); .t().contiguous() and the same again).
           Each entry counts n (sizeof T + outputs) + 4 (scale floats) bytes for what it writes.
  fp8r     the row-wise quantize at FP8R_SHAPES (or --shape) from each type to E4M3: both sides, row-wise only and
           column-wise only, and the dequantize of C; beside them at the same shape quantize_fp8_transpose_auto (the
           same bytes as both sides: A read twice, C and Ct written), quantize_fp8_auto (the same as row-wise only) and
           the torch-eager recipe for both sides (per-row amax, exp2 of floor(log2(max / amax)), multiply, .to(float8);
           .t().contiguous() and the same again).  Each entry counts n (sizeof T + outputs) + 4 (scale floats) bytes,
           A read once, so the rates compare times.
  mxfp8    per type and format, alternated in this order: quantize and dequantize at block 32 and at block 128,
           n * (sizeof T + 1 + 1 / block); the per-tensor recipes they compete with are in the fp8 family.
  sr       the stochastically rounding casts from f32, each beside its round-to-nearest counterpart: to f16 and bf16,
           and to E4M3 and E5M2 without and with amax, n * (4 + sizeof DST); then the torch-eager bf16 recipe (a random
           int32 tensor as large as the input, added to the f32 patterns, masked and cast in separate kernels), counted
           at the same n * 6 bytes.
The card's name, power limit and maximum SM clock are printed first (nvidia-smi), as they are part of every number.
One JSON line per measurement on stdout.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIZE = {"f32": 4, "f64": 8, "f16": 2, "bf16": 2}


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (s.strip() for s in out.stdout.splitlines()[0].split(","))
    return {"card": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, calls: int) -> float:
    """Seconds per call: CUDA events around `calls` back-to-back calls after two warm-up calls."""
    import torch

    fn()
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3 / calls


# Each family yields (op name, callable, algorithmic bytes per call); its operands live until the next one is asked for.
def convert_ops(torch, va, n, tdt, f8):
    for s in tdt:
        for d in tdt:
            if s == d:
                continue
            a = torch.randn(n, dtype=torch.float32, device="cuda").to(tdt[s])
            c = torch.empty(n, dtype=tdt[d], device="cuda")
            yield f"convert {s}->{d}", lambda: va.convert(a, tdt[d], c), n * (SIZE[s] + SIZE[d])
            del a, c


def fp8_ops(torch, va, n, tdt, f8):
    for s in tdt:
        a = torch.randn(n, dtype=torch.float32, device="cuda").to(tdt[s])
        amax = torch.zeros(1, dtype=torch.float64, device="cuda")
        for f in f8:
            q = torch.empty(n, dtype=f8[f], device="cuda")
            c = torch.empty(n, dtype=tdt[s], device="cuda")
            nbytes = n * (SIZE[s] + 1)
            yield f"quantize {s}->{f}", lambda: va.quantize_fp8(a, f8[f], out=q), nbytes
            yield f"quantize {s}->{f} amax", lambda: va.quantize_fp8(a, f8[f], amax=amax, out=q), nbytes
            yield f"dequantize {f}->{s}", lambda: va.dequantize_fp8(q, tdt[s], out=c), nbytes
            scratch = torch.empty(n, dtype=f8[f], device="cuda")
            k = torch.zeros(1, dtype=torch.int32, device="cuda")

            def two_pass():
                va.quantize_fp8(a, f8[f], amax=amax, out=scratch)
                va.quantize_fp8(a, f8[f], out=q)

            yield f"two-pass per-tensor quantize {s}->{f}", two_pass, 2 * n * (SIZE[s] + 1)
            yield (f"quantize_fp8_auto {s}->{f}", lambda: va.quantize_fp8_auto(a, f8[f], amax=amax, scale_exp=k, out=q),
                   n * (2 * SIZE[s] + 1))
            yield f"dequantize_fp8_auto {f}->{s}", lambda: va.dequantize_fp8_auto(q, k, tdt[s], out=c), nbytes
            del q, c, scratch, k
        del a, amax


FP8T_SHAPES = ((8192, 8192), (16384, 16384), (4096, 32768), (32768, 4096))


def fp8t_ops(torch, va, n, tdt, f8):
    """n is unused: the quantize-transpose family runs at FP8T_SHAPES."""
    for rows, cols in FP8T_SHAPES:
        m = rows * cols
        for s in tdt:
            a = torch.randn(rows, cols, dtype=torch.float32, device="cuda").to(tdt[s])
            amax = torch.zeros(1, dtype=torch.float64, device="cuda")
            k = torch.zeros(1, dtype=torch.int32, device="cuda")
            nbytes = m * (SIZE[s] + 2)
            for f in (("e4m3", "e5m2") if (rows, cols) == (8192, 8192) else ("e4m3",)):
                q = torch.empty(rows, cols, dtype=f8[f], device="cuda")
                qt = torch.empty(cols, rows, dtype=f8[f], device="cuda")
                tag = f"{s}->{f} {rows}x{cols}"

                def recipe1():
                    va.quantize_fp8(a, f8[f], out=q)
                    qt.copy_(q.t())

                def recipe1_auto():
                    va.quantize_fp8_auto(a, f8[f], amax=amax, scale_exp=k, out=q)
                    qt.copy_(q.t())

                yield f"quantize_fp8_transpose {tag}", lambda: va.quantize_fp8_transpose(a, f8[f], out=q, out_t=qt), nbytes
                yield f"quantize_fp8 alone {tag}", lambda: va.quantize_fp8(a, f8[f], out=q), nbytes
                yield f"quantize_fp8 + torch transpose {tag}", recipe1, nbytes
                yield (f"quantize_fp8_transpose_auto {tag}",
                       lambda: va.quantize_fp8_transpose_auto(a, f8[f], amax=amax, scale_exp=k, out=q, out_t=qt), nbytes)
                yield f"quantize_fp8_auto + torch transpose {tag}", recipe1_auto, nbytes
                del q, qt
            del a, amax, k


def fp8b_ops(torch, va, n, tdt, f8, shapes=FP8T_SHAPES):
    """n is unused: the blockwise family runs at FP8T_SHAPES (or the --shape given)."""
    for rows, cols in shapes:
        m = rows * cols
        ns, nst = m // 128, m // 128                                    # 1x128 scales of each side
        for s in tdt:
            a = torch.randn(rows, cols, dtype=torch.float32, device="cuda").to(tdt[s])
            for f in (("e4m3", "e5m2") if (rows, cols) == (8192, 8192) else ("e4m3",)):
                q = torch.empty(rows, cols, dtype=f8[f], device="cuda")
                qt = torch.empty(cols, rows, dtype=f8[f], device="cuda")
                sc = torch.empty(ns, dtype=torch.float32, device="cuda")
                sct = torch.empty(nst, dtype=torch.float32, device="cuda")
                s128 = torch.empty(va.fp8_blockwise_scale_layout(rows, cols, "128x128")[0], dtype=torch.float32, device="cuda")
                s128t = torch.empty(va.fp8_blockwise_scale_layout(cols, rows, "128x128")[0], dtype=torch.float32, device="cuda")
                e8 = torch.empty(ns, dtype=torch.uint8, device="cuda")
                top = 448.0 if f == "e4m3" else 57344.0
                tag = f"{s}->{f} {rows}x{cols}"

                def eager_side(x):
                    blocks = x.float().reshape(x.shape[0], -1, 128)
                    amax = blocks.abs().nan_to_num(0.0, 0.0, 0.0).amax(dim=2, keepdim=True)
                    k = torch.floor(torch.log2(top / amax)).clamp(-126, 126)
                    return (blocks * torch.exp2(k)).to(f8[f]).reshape(x.shape), torch.exp2(-k).squeeze(2).t().contiguous()

                def eager():
                    eager_side(a)
                    eager_side(a.t().contiguous())

                both = m * (SIZE[s] + 2) + 4 * (ns + nst)
                yield (f"fp8 blockwise 1x128 both {tag}",
                       lambda: va.quantize_fp8_blockwise(a, f8[f], out=q, scales=sc, out_t=qt, scales_t=sct), both)
                yield (f"fp8 blockwise 1x128 rowwise {tag}",
                       lambda: va.quantize_fp8_blockwise(a, f8[f], columnwise=False, out=q, scales=sc), m * (SIZE[s] + 1) + 4 * ns)
                yield (f"fp8 blockwise 1x128 columnwise {tag}",
                       lambda: va.quantize_fp8_blockwise(a, f8[f], rowwise=False, out_t=qt, scales_t=sct), m * (SIZE[s] + 1) + 4 * nst)
                yield (f"fp8 blockwise 128x128 both {tag}",
                       lambda: va.quantize_fp8_blockwise(a, f8[f], block="128x128", out=q, scales=s128, out_t=qt, scales_t=s128t),
                       m * (SIZE[s] + 2) + 4 * (s128.numel() + s128t.numel()))
                yield (f"quantize_fp8_transpose {tag}", lambda: va.quantize_fp8_transpose(a, f8[f], out=q, out_t=qt), both)
                yield (f"quantize_mxfp8 block 128 {tag}",
                       lambda: va.quantize_mxfp8(a.view(-1), f8[f], block=128, out=q.view(-1), scales=e8), m * (SIZE[s] + 1) + ns)
                yield f"torch eager 1x128 both {tag}", eager, both
                del q, qt, sc, sct, s128, s128t, e8
            del a


FP8R_SHAPES = ((16384, 16384), (32768, 4096), (4096, 14336))


def fp8r_ops(torch, va, n, tdt, f8, shapes=FP8R_SHAPES):
    """n is unused: the row-wise family runs at FP8R_SHAPES (or the --shape given)."""
    f = "e4m3"
    for rows, cols in shapes:
        m = rows * cols
        for s in tdt:
            a = torch.randn(rows, cols, dtype=torch.float32, device="cuda").to(tdt[s])
            q = torch.empty(rows, cols, dtype=f8[f], device="cuda")
            qt = torch.empty(cols, rows, dtype=f8[f], device="cuda")
            sc = torch.empty(rows, dtype=torch.float32, device="cuda")
            sct = torch.empty(cols, dtype=torch.float32, device="cuda")
            ws = torch.empty(va.lib.b200va_fp8_rowwise_workspace(rows, cols), dtype=torch.uint8, device="cuda")
            back = torch.empty(rows, cols, dtype=tdt[s], device="cuda")
            amax = torch.zeros(1, dtype=torch.float64, device="cuda")
            k = torch.zeros(1, dtype=torch.int32, device="cuda")
            tag = f"{s}->{f} {rows}x{cols}"

            def eager_side(x):
                amax_r = x.float().abs().nan_to_num(0.0, 0.0, 0.0).amax(dim=1, keepdim=True)
                kr = torch.floor(torch.log2(448.0 / amax_r)).clamp(-126, 126)
                return (x.float() * torch.exp2(kr)).to(f8[f]), torch.exp2(-kr).view(-1)

            def eager():
                eager_side(a)
                eager_side(a.t().contiguous())

            both = m * (SIZE[s] + 2) + 4 * (rows + cols)
            yield (f"fp8 rowwise both {tag}",
                   lambda: va.quantize_fp8_rowwise(a, f, out=q, scales=sc, out_t=qt, scales_t=sct, workspace=ws), both)
            yield (f"quantize_fp8_transpose_auto {tag}",
                   lambda: va.quantize_fp8_transpose_auto(a, f, amax=amax, scale_exp=k, out=q, out_t=qt), both)
            yield (f"fp8 rowwise rowwise {tag}",
                   lambda: va.quantize_fp8_rowwise(a, f, columnwise=False, out=q, scales=sc, workspace=ws),
                   m * (SIZE[s] + 1) + 4 * rows)
            yield (f"quantize_fp8_auto {tag}",
                   lambda: va.quantize_fp8_auto(a.view(-1), f, amax=amax, scale_exp=k, out=q.view(-1)), m * (SIZE[s] + 1))
            yield (f"fp8 rowwise columnwise {tag}",
                   lambda: va.quantize_fp8_rowwise(a, f, rowwise=False, out_t=qt, scales_t=sct, workspace=ws),
                   m * (SIZE[s] + 1) + 4 * cols)
            yield f"fp8 rowwise dequantize {tag}", lambda: va.dequantize_fp8_rowwise(q, sc, tdt[s], out=back), m * (SIZE[s] + 1)
            yield f"torch eager rowwise both {tag}", eager, both
            del a, q, qt, sc, sct, ws, back, amax, k


def mxfp8_ops(torch, va, n, tdt, f8):
    for s in tdt:
        a = torch.randn(n, dtype=torch.float32, device="cuda").to(tdt[s])
        c = torch.empty(n, dtype=tdt[s], device="cuda")
        for f in f8:
            q = torch.empty(n, dtype=f8[f], device="cuda")
            for block in (32, 128):
                sc = torch.empty(n // block, dtype=torch.uint8, device="cuda")
                nbytes = n * (SIZE[s] + 1) + n // block
                yield (f"mx quantize {s}->{f} block {block}",
                       lambda: va.quantize_mxfp8(a, f8[f], block=block, out=q, scales=sc), nbytes)
                yield (f"mx dequantize {f}->{s} block {block}",
                       lambda: va.dequantize_mxfp8(q, sc, tdt[s], block=block, out=c), nbytes)
                del sc
            del q
        del a, c


def sr_ops(torch, va, n, tdt, f8):
    a = torch.randn(n, dtype=torch.float32, device="cuda")
    amax = torch.zeros(1, dtype=torch.float64, device="cuda")
    for d in ("f16", "bf16"):
        c = torch.empty(n, dtype=tdt[d], device="cuda")
        nbytes = n * (4 + SIZE[d])
        yield f"sr convert f32->{d}", lambda: va.convert_sr(a, tdt[d], seed=1, out=c), nbytes
        yield f"convert f32->{d}", lambda: va.convert(a, tdt[d], c), nbytes
        del c
    for f in f8:
        q = torch.empty(n, dtype=f8[f], device="cuda")
        nbytes = n * 5
        yield f"sr quantize f32->{f}", lambda: va.quantize_fp8_sr(a, f8[f], seed=1, out=q), nbytes
        yield f"quantize f32->{f}", lambda: va.quantize_fp8(a, f8[f], out=q), nbytes
        yield f"sr quantize f32->{f} amax", lambda: va.quantize_fp8_sr(a, f8[f], seed=1, amax=amax, out=q), nbytes
        yield f"quantize f32->{f} amax", lambda: va.quantize_fp8(a, f8[f], amax=amax, out=q), nbytes
        del q
    c = torch.empty(n, dtype=torch.bfloat16, device="cuda")

    def eager():
        r = torch.randint(0, 1 << 16, (n,), dtype=torch.int32, device="cuda")
        c.copy_(((a.view(torch.int32) + r) & -65536).view(torch.float32))

    yield "torch-eager sr f32->bf16", eager, n * 6
    del a, amax, c


FAMILIES = {"convert": convert_ops, "fp8": fp8_ops, "fp8t": fp8t_ops, "fp8b": fp8b_ops, "fp8r": fp8r_ops, "mxfp8": mxfp8_ops,
            "sr": sr_ops}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--family", choices=[*FAMILIES, "all"], default="all")
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shape", default=None, help="ROWSxCOLS: run the fp8b and fp8r families at this shape only")
    args = ap.parse_args()

    import torch

    from k8s_gpu_hpa_b200 import vector_add as va

    if not torch.cuda.is_available():
        raise SystemExit("cast_rate.py needs a CUDA device")
    n = 1 << args.log2n
    print(json.dumps(card()), flush=True)
    tdt = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}
    f8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
    families = list(FAMILIES) if args.family == "all" else [args.family]

    def report(r, op, t, nbytes):
        print(json.dumps({"round": r, "op": op, "n": n, "us": round(t * 1e6, 1), "TB/s": round(nbytes / t / 1e12, 3)}),
              flush=True)

    for r in range(args.rounds):
        for family in families:
            ops = FAMILIES[family]
            if family in ("fp8b", "fp8r") and args.shape:
                shape = tuple(int(v) for v in args.shape.split("x"))
                ops = lambda *x, f=ops: f(*x, shapes=(shape,))  # noqa: E731
            for op, fn, nbytes in ops(torch, va, n, tdt, f8):
                report(r, op, timed(fn, args.calls), nbytes)
        x, y, z = (torch.ones(n, dtype=torch.float32, device="cuda") for _ in range(3))
        for kind, nbytes in (("copy", 8 * n), ("read2", 8 * n)):
            report(r, f"probe {kind}", timed(lambda: va.probe(kind, x, y, z), args.calls), nbytes)
        del x, y, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
