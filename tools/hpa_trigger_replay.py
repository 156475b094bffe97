#!/usr/bin/env python
"""BASELINE.json configs[4] / SURVEY 8(f) row 1: sustained in-process launch loop at N = 2^24
driving GPU utilisation, replayed against the (unchanged) recording rule and HPA.

For each duty-cycle target the drop-in binary runs `--iters 5000`-launch blocks for a
wall-clock duration while sampling NVML utilisation (the local stand-in for
dcgm_gpu_utilization); the sampled trace is then fed through hpa_replay.Replay
(exporter 10 s collect, 1 s scrape, rule, HPA sync 15 s, target 5, 1..3 replicas).

    python tools/hpa_trigger_replay.py [seconds per target] > profiles/<round>/<name>_hpa_trigger_replay.jsonl

(run on an H100; tests/test_hpa_replay.py replays the committed recordings offline)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from k8s_gpu_hpa_b200 import hpa_replay as hr  # noqa: E402

CLI = os.path.join(ROOT, "k8s-gpu-hpa_b200", "vectorAdd")


def main():
    duration = float(sys.argv[1]) if len(sys.argv) > 1 else 20.0
    for target in (0, 60, 20, 8, 4, 2):
        cmd = [CLI, "--mode", "resident", "--n", "2^24", "--iters", "5000" if target == 0 else "50", "--graph", "50",
               "--duration", str(duration), "--nvml"]
        if target:
            cmd += ["--target-util", str(target), "--period-ms", "100"]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=duration * 3 + 120)
        if p.returncode != 0:
            print(json.dumps({"target_util": target, "error": p.stderr[-300:]}), flush=True)
            continue
        r = json.loads(p.stdout.strip().splitlines()[-1])
        trace = [(0.5 * i, float(u)) for i, u in enumerate(r["nvml_trace"][0]) if u >= 0]
        ev = hr.Replay().run({"cuda-test-0": trace, "cuda-test-1": trace, "cuda-test-2": trace}, duration)
        print(json.dumps({
            "target_util": target or "unthrottled (5000-launch blocks)", "duration_s": duration,
            "launches": r["launches_per_gpu"], "elements_per_s_while_busy": r["elements_per_s"],
            "algorithmic_GBps_while_busy": r["algorithmic_GBps"], "gpu_busy_frac_events": r["gpu_busy_frac"],
            "nvml_util_mean": r["nvml_util_mean"], "nvml_util_max": r["nvml_util_max"], "mismatches": r["mismatches"],
            "hpa_threshold": hr.HPA_TARGET, "steady_state_would_scale_up": hr.would_scale_up(r["nvml_util_mean"]),
            "replay_events_t_metric_replicas": ev}), flush=True)


if __name__ == "__main__":
    main()
