"""Rate of b200va_convert per pair of types, next to the f32 COPY and READ2 ceiling probes, in one process.

    python tools/convert_rate.py [--log2n 28] [--calls 20] [--rounds 3]

Per round, every ordered pair of distinct types is timed at n elements with CUDA events around `calls` back-to-back
calls (after two warm-up calls), then b200va_probe_f32 COPY and READ2 at the same n.  Algorithmic bytes per
convert call are n * (sizeof SRC + sizeof DST); COPY moves 8 n bytes and READ2 reads 8 n.  The card's name, power
limit and maximum SM clock are printed first (nvidia-smi), as they are part of every number.  One JSON line per
measurement on stdout.
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


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from k8s_gpu_hpa_b200 import vector_add as va

    if not torch.cuda.is_available():
        raise SystemExit("convert_rate.py needs a CUDA device")
    n = 1 << args.log2n
    print(json.dumps(card()), flush=True)
    tdt = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}
    pairs = [(s, d) for s in tdt for d in tdt if s != d]
    for r in range(args.rounds):
        for s, d in pairs:
            a = torch.randn(n, dtype=torch.float32, device="cuda").to(tdt[s])
            c = torch.empty(n, dtype=tdt[d], device="cuda")
            t = timed(lambda: va.convert(a, tdt[d], c), args.calls)
            print(json.dumps({"round": r, "op": f"convert {s}->{d}", "n": n, "us": round(t * 1e6, 1),
                              "TB/s": round(n * (SIZE[s] + SIZE[d]) / t / 1e12, 3)}), flush=True)
            del a, c
        x, y, z = (torch.ones(n, dtype=torch.float32, device="cuda") for _ in range(3))
        for kind, nbytes in (("copy", 8 * n), ("read2", 8 * n)):
            t = timed(lambda: va.probe(kind, x, y, z), args.calls)
            print(json.dumps({"round": r, "op": f"probe {kind}", "n": n, "us": round(t * 1e6, 1),
                              "TB/s": round(nbytes / t / 1e12, 3)}), flush=True)
        del x, y, z
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
