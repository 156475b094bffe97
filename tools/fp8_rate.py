"""Rate of b200va_quantize_fp8 and b200va_dequantize_fp8 per pair, next to the f32 COPY and READ2 ceiling probes, in one
process.

    python tools/fp8_rate.py [--log2n 28] [--calls 20] [--rounds 3]

Per round, each of the 16 pairs (quantize from f32, f64, f16, bf16 to E4M3 and E5M2 without amax, the same with
amax, and dequantize back into each type) is timed at n elements with CUDA events around `calls` back-to-back calls
(after two warm-up calls), then b200va_probe_f32 COPY and READ2 at the same n.  Algorithmic bytes per call are
n * (sizeof T + 1); COPY moves 8 n bytes and READ2 reads 8 n.  The card's name, power limit and maximum SM clock are
printed first (nvidia-smi), as they are part of every number.  One JSON line per measurement on stdout.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.convert_rate import SIZE, card, timed  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from k8s_gpu_hpa_b200 import vector_add as va

    if not torch.cuda.is_available():
        raise SystemExit("fp8_rate.py needs a CUDA device")
    n = 1 << args.log2n
    print(json.dumps(card()), flush=True)
    tdt = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}
    f8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}

    def report(r, op, t, nbytes):
        print(json.dumps({"round": r, "op": op, "n": n, "us": round(t * 1e6, 1), "TB/s": round(nbytes / t / 1e12, 3)}),
              flush=True)

    for r in range(args.rounds):
        for s in tdt:
            a = torch.randn(n, dtype=torch.float32, device="cuda").to(tdt[s])
            amax = torch.zeros(1, dtype=torch.float64, device="cuda")
            for f in f8:
                q = torch.empty(n, dtype=f8[f], device="cuda")
                c = torch.empty(n, dtype=tdt[s], device="cuda")
                nbytes = n * (SIZE[s] + 1)
                report(r, f"quantize {s}->{f}", timed(lambda: va.quantize_fp8(a, f8[f], out=q), args.calls), nbytes)
                report(r, f"quantize {s}->{f} amax",
                       timed(lambda: va.quantize_fp8(a, f8[f], amax=amax, out=q), args.calls), nbytes)
                report(r, f"dequantize {f}->{s}", timed(lambda: va.dequantize_fp8(q, tdt[s], out=c), args.calls), nbytes)
                del q, c
            del a, amax
        x, y, z = (torch.ones(n, dtype=torch.float32, device="cuda") for _ in range(3))
        for kind, nbytes in (("copy", 8 * n), ("read2", 8 * n)):
            report(r, f"probe {kind}", timed(lambda: va.probe(kind, x, y, z), args.calls), nbytes)
        del x, y, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
