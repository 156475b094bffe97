"""Every entry point captured into the caller's own CUDA graph (torch.cuda.graph), the way training code runs the casts.

Two kinds of hidden library state meet a capture here.  The first dynamically scheduled add of a process (variant k2,
or a K1d tune) sets up the device's ticket ring; when that first call is made inside a capture, the setup must neither
break the capture nor leave a failure behind.  And a captured dynamically scheduled add keeps its ticket counter for
every replay of the graph, so the counter must be one that no direct launch is handed while the graph lives
(csrc/b200va_add.cu: sched_slot, capture_slot).

Every output is a poisoned arena with guards (gpu_helpers.poisoned), poisoned again before every replay, and compared
bit for bit -- NaN as a class where the op's contract says so -- with the exact references.  The inputs change between
replays, so a replay that reuses stale values is caught.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import GUARD, INT, POISON, assert_guards, assert_matches, k1d_tunes, poisoned, to_dev
    from k8s_gpu_hpa_b200 import capi, vector_add as va
    from oracle import convert_exact as V
    from oracle import dot_exact as D
    from oracle import fp8_exact as F
    from oracle import mxfp8_exact as M
    from oracle import sr_exact as S
    from oracle import stream_exact as X

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RING = 4096                     # ticket-counter slots per device for direct launches (kSchedSlots)
CAPTURE_SLOTS = 16384           # ticket counters per device for captured launches (kCaptureSlots)
ROUNDS = 4                      # three replays, then one direct call
NA = (3 << 20) + 5              # adds: more tiles than the persistent K2d / K1d grids hold CTAs, plus a ragged tail
NC = 3 * 65536 + 77             # casts, STREAM ops and the dot: several dot chunks, ragged in every vector width
CUDA_CAPTURE_UNSUPPORTED = -(1000 + 900)   # cudaErrorStreamCaptureUnsupported
ENTRIES = 22                    # what entries() builds


# ------------------------------------------------------------------------------------------- the entry points
def _values(rng, n):
    """f32 values at every scale FP8 and bf16 care about, with every 7th element a random bit pattern (NaN, inf,
    subnormals, zeros of both signs)."""
    x = (rng.standard_normal(n) * np.exp2(rng.integers(-14, 14, n))).astype(np.float32)
    x[::7] = V.random_bits("f32", x[::7].size, rng)
    return x


def _host_inputs(seed=1):
    """Round r's inputs of every entry point, on the host (numpy only: no library call)."""
    rng = np.random.default_rng(seed)
    h = []
    for r in range(ROUNDS):
        h.append({
            "a": oracle.fill_ctr(NA, 0x10 + r), "b": oracle.fill_ctr(NA, 0x20 + r),
            "x": _values(rng, NC), "y": (rng.standard_normal(NC) * 64).astype(np.float32),
            "q8": rng.integers(0, 256, NC, dtype=np.uint8), "mq": rng.integers(0, 256, NC, dtype=np.uint8),
            "ms": rng.integers(100, 156, -(-NC // 32), dtype=np.uint8),
        })
        h[-1]["ms"][::97] = 0xFF                                  # a NaN scale now and then
    return h


IN_FMT = {"a": "f32", "b": "f32", "x": "f32", "y": "f32", "q8": "e5m2", "mq": "e4m3", "ms": "u8"}
SEED, FIRST = 0x5EED, 12345


class Entry:
    """One entry point: its poisoned outputs {key: (fmt, n)}, its launch on the current stream and its exact result
    {key: host storage} for round r's inputs."""

    def __init__(self, name, outs, launch, want, nan_class=True):
        self.name, self.launch_fn, self.want, self.nan_class = name, launch, want, nan_class
        self.outs = {k: (fmt, n) + poisoned(n, fmt) for k, (fmt, n) in outs.items()}
        self.o = {k: v[3] for k, v in self.outs.items()}

    def launch(self, d):
        self.launch_fn(d, self.o)

    def poison(self):
        for _, _, buf, _ in self.outs.values():
            buf.view(torch.uint8).fill_(POISON)

    def check(self, h, what):
        want = self.want(h)
        for k, (fmt, n, buf, view) in self.outs.items():
            assert_matches(view, to_dev(np.ascontiguousarray(want[k]), fmt), fmt, f"{what}: {self.name} {k}",
                           nan_class=self.nan_class and fmt != "u8")
            assert_guards(buf, GUARD, n, f"{what}: {self.name} {k}")


def _amax(v):
    return np.array([v], np.float64)


def entries():
    """Every capturable entry point, the dynamically scheduled adds first.  Building them calls no library function."""
    k1d = k1d_tunes()[0]
    k4 = capi.Tune(kind=capi.K4_SCALAR_MLP, threads=256, unroll=8)
    add = lambda h: {"c": oracle.vadd(h["a"], h["b"])}
    e = [Entry("add k2", {"c": ("f32", NA)}, lambda d, o: va.add(d["a"], d["b"], o["c"], variant="k2"), add),
         Entry("add_tuned K1d", {"c": ("f32", NA)}, lambda d, o: va.add(d["a"], d["b"], o["c"], tune=k1d), add),
         Entry("add_tuned K4", {"c": ("f32", NA)}, lambda d, o: va.add(d["a"], d["b"], o["c"], tune=k4), add)]
    for v in ("auto", "k1", "k3"):
        e.append(Entry(f"add {v}", {"c": ("f32", NA)}, lambda d, o, v=v: va.add(d["a"], d["b"], o["c"], variant=v), add))
    for flags in ({"inputs_stable": True}, {"cold": True}, {"inputs_stable": True, "cold": True}):
        e.append(Entry(f"add_ex {'+'.join(flags)}", {"c": ("f32", NA)},
                       lambda d, o, f=flags: va.add(d["a"], d["b"], o["c"], **f), add))
    for op, s in (("copy", 0.0), ("scale", 3.0), ("add", 0.0), ("triad", -0.75)):
        e.append(Entry(f"stream {op}", {"c": ("f32", NC)},
                       lambda d, o, op=op, s=s: va.stream(op, d["x"], d["y"] if op in ("add", "triad") else None,
                                                          o["c"], scalar=s),
                       lambda h, op=op, s=s: {"c": X.stream(op, "f32", h["x"], h["y"] if op in ("add", "triad") else None, s)},
                       nan_class=op != "copy"))

    def quantize(d, o):
        o["m"].zero_()                                            # the amax is reset inside the graph
        va.quantize_fp8(d["x"], "e4m3", scale_exp=-2, amax=o["m"], out=o["q"])

    def quantize_sr(d, o):
        o["m"].zero_()
        va.quantize_fp8_sr(d["x"], "e5m2", seed=SEED, offset=FIRST, scale_exp=1, amax=o["m"], out=o["q"])

    def dot(d, o):
        va.dot(d["a"][:NC], d["b"][:NC], out=o["r"], workspace=d["ws"])

    e += [
        Entry("convert f32->bf16", {"c": ("bf16", NC)}, lambda d, o: va.convert(d["x"], "bf16", o["c"]),
              lambda h: {"c": V.convert(h["x"], "f32", "bf16")}),
        Entry("quantize_fp8 e4m3 + amax", {"q": ("e4m3", NC), "m": ("f64", 1)}, quantize,
              lambda h: {"q": F.quantize(h["x"], "f32", "e4m3", -2), "m": _amax(F.amax(h["x"], "f32"))}),
        Entry("dequantize_fp8 e5m2->f16", {"c": ("f16", NC)},
              lambda d, o: va.dequantize_fp8(d["q8"], "f16", scale_exp=3, out=o["c"]),
              lambda h: {"c": F.dequantize(h["q8"], "e5m2", "f16", 3)}),
        Entry("quantize_mxfp8 e4m3/32", {"q": ("e4m3", NC), "s": ("u8", -(-NC // 32))},
              lambda d, o: va.quantize_mxfp8(d["x"], "e4m3", block=32, out=o["q"], scales=o["s"]),
              lambda h: dict(zip("qs", M.quantize(h["x"], "f32", "e4m3", 32, "ocp")))),
        Entry("dequantize_mxfp8 e4m3/32->bf16", {"c": ("bf16", NC)},
              lambda d, o: va.dequantize_mxfp8(d["mq"], d["ms"], "bf16", block=32, out=o["c"]),
              lambda h: {"c": M.dequantize(h["mq"], h["ms"], "e4m3", "bf16", 32)}),
        Entry("convert_sr f32->bf16", {"c": ("bf16", NC)},
              lambda d, o: va.convert_sr(d["x"], "bf16", seed=SEED, offset=FIRST, out=o["c"]),
              lambda h: {"c": S.convert_sr(h["x"], "bf16", SEED, FIRST)}),
        Entry("quantize_fp8_sr e5m2 + amax", {"q": ("e5m2", NC), "m": ("f64", 1)}, quantize_sr,
              lambda h: {"q": S.quantize_fp8_sr(h["x"], "e5m2", SEED, FIRST, 1), "m": _amax(F.amax(h["x"], "f32"))}),
        Entry("dot f32", {"r": ("f64", 1)}, dot, lambda h: {"r": _amax(D.dot(h["a"][:NC], h["b"][:NC], "f32"))}),
        Entry("fill_ctr", {"c": ("f32", NC)}, lambda d, o: va.fill_ctr(o["c"], 0x33, 7),
              lambda h: {"c": oracle.fill_ctr(NC, 0x33, 7)}, nan_class=False),
    ]
    return e


class Inputs:
    """The device inputs of every entry point; load(r) copies round r's values in (torch only)."""

    def __init__(self, host):
        self.host = host
        self.d = {k: to_dev(v, IN_FMT[k]) for k, v in host[0].items()}
        self.d["ws"] = torch.empty(max(8, 8 * -(-NC // 65536)), dtype=torch.uint8, device="cuda")

    def load(self, r):
        for k, v in self.host[r].items():
            self.d[k].view(INT[IN_FMT[k]]).copy_(to_dev(v, IN_FMT[k]).view(INT[IN_FMT[k]]))


def _report(fn):
    try:
        fn()
        return "ok"
    except Exception as e:     # noqa: BLE001 -- reported to the parent test
        return f"{type(e).__name__}: {e}"[:400]


def cold_capture_child(mode, first):
    """The body of one cold process: torch makes its context, then the library's first call -- `first` -- and every
    other entry point are captured into one graph under capture_error_mode `mode`.  Three replays with new inputs and
    fresh poison, each checked; then one direct call of every entry point.  Prints a JSON report."""
    t0 = time.monotonic()
    torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    host = _host_inputs()
    inp = Inputs(host)
    es = entries()
    es.sort(key=lambda e: e.name != first)
    rep = {"mode": mode, "first": first, "capture": {}, "replay": {}, "direct": {}}
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()

    def capture():
        with torch.cuda.graph(g, capture_error_mode=mode):
            for e in es:
                rep["capture"][e.name] = _report(lambda e=e: e.launch(inp.d))

    rep["graph"] = _report(capture)
    torch.cuda.synchronize()
    for r in range(ROUNDS - 1):
        if rep["graph"] != "ok":
            break
        inp.load(r)
        for e in es:
            e.poison()
        g.replay()
        torch.cuda.synchronize()
        for e in es:
            res = _report(lambda e=e: e.check(host[r], f"replay {r}"))
            if res != "ok" or e.name not in rep["replay"]:
                rep["replay"][e.name] = res
    del g
    inp.load(ROUNDS - 1)
    for e in es:
        e.poison()
        rep["direct"][e.name] = _report(lambda e=e: e.launch(inp.d))
    torch.cuda.synchronize()
    for e in es:
        if rep["direct"][e.name] == "ok":
            rep["direct"][e.name] = _report(lambda e=e: e.check(host[ROUNDS - 1], "direct"))
    rep["seconds"] = round(time.monotonic() - t0, 1)
    print("REPORT " + json.dumps(rep))


@pytest.mark.parametrize("first", ["add k2", "add_tuned K1d"])
@pytest.mark.parametrize("mode", ["global", "thread_local", "relaxed"])
def test_first_library_call_of_a_process_inside_a_capture(mode, first):
    """One fresh process per (capture mode, first call): the first call of the library, a dynamically scheduled add
    that sets up the device's ticket ring, is made inside torch.cuda.graph, followed by every other capturable entry
    point.  The capture must succeed, its three replays must be right, and a direct call of each entry point after it
    must work: no failure may be left behind."""
    code = (f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_gpu_graph_capture as m; "
            f"m.cold_capture_child({mode!r}, {first!r})")
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("REPORT ")]
    assert p.returncode == 0 and lines, f"exit {p.returncode}\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    rep = json.loads(lines[-1][len("REPORT "):])
    print(f"{mode} / {first}: {rep['seconds']} s in the child")
    bad = {f"{stage} {k}": v for stage in ("capture", "replay", "direct") for k, v in rep[stage].items() if v != "ok"}
    assert rep["graph"] == "ok" and not bad, json.dumps({"graph": rep["graph"], "failed": bad}, indent=1)
    assert len(rep["replay"]) == len(rep["direct"]) == len(rep["capture"]) == ENTRIES


# ------------------------------------------------------------------------------------------- captured dynamic adds
def ctr_inputs(n):
    a = va.fill_ctr(torch.empty(n, dtype=torch.float32, device="cuda"), oracle.SEED_A)
    b = va.fill_ctr(torch.empty(n, dtype=torch.float32, device="cuda"), oracle.SEED_B)
    return a, b


def check_add(a, b, c, n, what, win=256):
    """verify, the oracle's digest, and the oracle element by element on windows at the head, middle and tail."""
    assert va.verify(a[:n], b[:n], c[:n]) == (0, -1), what
    assert va.digest(c[:n]) == oracle.ctr_vadd_digest(n), f"{what}: digest"
    for lo in (0, n // 2, n - win):
        want = oracle.vadd(oracle.fill_ctr(win, oracle.SEED_A, lo), oracle.fill_ctr(win, oracle.SEED_B, lo))
        assert np.array_equal(c[lo:lo + win].cpu().numpy().view(np.uint32), want.view(np.uint32)), f"{what} [{lo}:]"


def dyn_launch(form, a, b, c, stream=None):
    if form == "k2":
        va.add(a, b, c, variant="k2", stream=stream)
    else:
        va.add(a, b, c, tune=k1d_tunes()[0], stream=stream)


@pytest.mark.parametrize("beside", ["k2", "K1d"])
def test_captured_k2_next_to_the_direct_launch_that_gets_the_same_ring_position(beside):
    """A graph G holding one k2 add is captured; exactly 4095 direct dynamically scheduled launches follow, so a
    captured launch that had taken a ring slot would now share it with the next direct launch.  That launch -- k2, or
    a K1d, whose CTAs fit on the SMs beside G's persistent grid, so the two certainly run at once -- is released on
    stream Y together with G's replay on stream X, both behind one event.  Both outputs, then G replayed alone, then 64
    more direct launches, are verified."""
    n = (1 << 24) + 5
    a, b = ctr_inputs(n)
    cg, cy = torch.empty_like(a), torch.empty_like(a)
    small_a, small_b = a[:(1 << 16) + 3], b[:(1 << 16) + 3]
    small_c = torch.empty_like(small_a)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        va.add(a, b, cg, variant="k2")
    torch.cuda.synchronize()
    for i in range(RING - 1):
        dyn_launch("k2" if i % 2 else "K1d", small_a, small_b, small_c)
        if i % 512 == 511:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    check_add(small_a, small_b, small_c, small_a.numel(), "the last small direct launch")
    sx, sy, sz = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    cg.view(torch.int32).fill_(0x7F7F7F7F)
    cy.view(torch.int32).fill_(0x7F7F7F7F)
    torch.cuda.synchronize()
    go = torch.cuda.Event()
    with torch.cuda.stream(sz):
        torch.cuda._sleep(5_000_000)                  # a few milliseconds: both launches are queued before it ends
        go.record(sz)
    sx.wait_event(go)
    sy.wait_event(go)
    with torch.cuda.stream(sx):
        g.replay()
    dyn_launch(beside, a, b, cy, stream=sy)
    torch.cuda.synchronize()
    check_add(a, b, cg, n, "G's replay on X")
    check_add(a, b, cy, n, f"the direct {beside} launch on Y")
    cg.view(torch.int32).fill_(0x7F7F7F7F)
    g.replay()
    torch.cuda.synchronize()
    check_add(a, b, cg, n, "G replayed again, alone")
    m = 3 << 20
    for i in range(64):
        cy[:m].view(torch.int32).fill_(0x7F7F7F7F)
        dyn_launch("k2" if i % 2 else "K1d", a[:m], b[:m], cy[:m])
        assert va.verify(a[:m], b[:m], cy[:m]) == (0, -1), f"direct launch {i} after the replays"
    del g


def test_graph_of_4096_captured_dynamic_adds_next_to_4096_direct_launches():
    """A graph of 4096 captured k2 / K1d adds, each followed by its own poison fill before and a device verify after,
    replays on stream X while a second host thread issues 4096 + 64 direct k2 / K1d launches on stream Y, every one
    verified.  A captured launch that held a ring slot would hold all 4096 of them here."""
    n = (3 << 20) + 3
    a, b = ctr_inputs(n)
    outs = [torch.empty_like(a) for _ in range(4)]
    res = torch.empty((RING, 2), dtype=torch.int64, device="cuda")
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        for i in range(RING):
            c = outs[i % 4]
            c.view(torch.int32).fill_(0x7F7F7F7F)
            dyn_launch("k2" if i % 2 else "K1d", a, b, c)
            capi.check(capi.lib.b200va_verify_f32(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, res[i].data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream), "b200va_verify_f32")
    torch.cuda.synchronize()
    errors, done = [], threading.Event()
    launches = RING + 64

    def direct():
        try:
            sy = torch.cuda.Stream()
            ya, yb = ctr_inputs(n)
            yc = [torch.empty_like(ya) for _ in range(4)]
            yres = torch.empty((launches, 2), dtype=torch.int64, device="cuda")
            with torch.cuda.stream(sy):
                for i in range(launches):
                    c = yc[i % 4]
                    c.view(torch.int32).fill_(0x7F7F7F7F)
                    dyn_launch("k2" if i % 3 else "K1d", ya, yb, c)
                    capi.check(capi.lib.b200va_verify_f32(ya.data_ptr(), yb.data_ptr(), c.data_ptr(), n,
                                                          yres[i].data_ptr(), sy.cuda_stream), "b200va_verify_f32")
                    if i % 256 == 255:
                        sy.synchronize()
            sy.synchronize()
            bad = torch.nonzero(yres[:, 0] != 0)
            if bad.numel():
                errors.append(f"direct launch {int(bad[0])}: {int(yres[int(bad[0]), 0])} elements wrong "
                              f"({bad.numel()} launches)")
        except BaseException as e:      # noqa: BLE001 -- reported to the main thread
            errors.append(repr(e))
        finally:
            done.set()

    sx = torch.cuda.Stream()
    y = threading.Thread(target=direct)
    replays = 0
    y.start()
    try:
        with torch.cuda.stream(sx):
            while replays < 3 or (not done.is_set() and replays < 200):
                res.fill_(-1)
                g.replay()
                sx.synchronize()
                bad = torch.nonzero(res[:, 0] != 0)
                assert bad.numel() == 0, (f"replay {replays}: captured launch {int(bad[0])} has "
                                          f"{int(res[int(bad[0]), 0])} elements wrong ({bad.numel()} launches)")
                replays += 1
    finally:
        y.join()
    assert not errors, errors
    del g


def test_captured_counters_run_out_with_an_error_and_come_back():
    """The pool of captured-launch counters is finite: one captured dynamically scheduled launch more than it holds is
    refused with an error code (no counter is shared), the capture itself stays valid, and destroying the graphs
    returns every counter."""
    n = (1 << 16) + 3
    a, b = ctr_inputs(n)
    c = torch.empty_like(a)
    torch.cuda.synchronize()

    def capture(count, last=None):
        g, codes = torch.cuda.CUDAGraph(), []
        with torch.cuda.graph(g):
            for _ in range(count):
                codes.append(capi.lib.b200va_add_f32(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, capi.K2_TMA,
                                                     torch.cuda.current_stream().cuda_stream))
            if last:
                last()
        return g, codes

    # the graphs of earlier tests are destroyed, but the driver may release their counters a little later
    for attempt in range(20):
        g, codes = capture(CAPTURE_SLOTS + 1, lambda: va.add(a, b, c, variant="k1"))
        if codes[:-1] == [0] * CAPTURE_SLOTS or attempt == 19:
            break
        del g
        torch.cuda.synchronize()
        time.sleep(0.25)
    assert codes[:-1] == [0] * CAPTURE_SLOTS and codes[-1] == capi.ERR_NOMEM, \
        f"{codes.count(0)} captured, then {sorted(set(codes) - {0})}"
    c.fill_(-1.0)
    g.replay()                              # a launch that needs no counter was captured after the refusal
    torch.cuda.synchronize()
    check_add(a, b, c, n, "the replay of the full pool's graph")
    del g
    torch.cuda.synchronize()
    for attempt in range(20):               # the counters come back: the whole pool fits again
        g, codes = capture(CAPTURE_SLOTS)
        if codes == [0] * CAPTURE_SLOTS:
            break
        del g
        torch.cuda.synchronize()
        time.sleep(0.25)
    assert codes == [0] * CAPTURE_SLOTS, f"{codes.count(0)} of {CAPTURE_SLOTS} counters came back"
    print(f"the pool was whole again after {attempt} waits of 0.25 s")
    c.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    check_add(a, b, c, n, "the replay of the pool that came back")
    del g
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- chains in one graph
def test_dependent_chains_inside_one_captured_graph():
    """One captured graph across the programmatic edges between entry points: triad -> quantize_fp8 (amax) ->
    dequantize_fp8 -> convert -> dot; quantize_mxfp8 -> dequantize_mxfp8; an inputs_stable add behind the dot, which
    does not write its inputs.  Replayed with new inputs each time; every stage and the amax checked."""
    n = NC
    rng = np.random.default_rng(7)
    a, b = torch.empty(n, dtype=torch.float32, device="cuda"), torch.empty(n, dtype=torch.float32, device="cuda")
    bt, t = poisoned(n, "f32")
    bq, q = poisoned(n, "e4m3")
    bd, dq = poisoned(n, "f32")
    bh, h = poisoned(n, "bf16")
    br, r = poisoned(1, "f64")
    bm, m = poisoned(1, "f64")
    bmq, mq = poisoned(n, "e5m2")
    bms, ms = poisoned(-(-n // 64), "u8")
    bmd, md = poisoned(n, "f16")
    bc, c = poisoned(n, "f32")
    ws = torch.empty(8 * -(-n // 65536), dtype=torch.uint8, device="cuda")
    s = 1.5
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        va.stream("triad", a, b, t, scalar=s)
        m.zero_()
        va.quantize_fp8(t, "e4m3", scale_exp=-3, amax=m, out=q)
        va.dequantize_fp8(q, "f32", scale_exp=-3, out=dq)
        va.convert(dq, "bf16", h)
        va.dot(h, h, out=r, workspace=ws)
        va.quantize_mxfp8(t, "e5m2", block=64, scale_rule="nosat", out=mq, scales=ms)
        va.dequantize_mxfp8(mq, ms, "f16", block=64, out=md)
        va.add(a, b, c, inputs_stable=True)
    for rnd in range(3):
        ha = (rng.standard_normal(n) * np.exp2(rng.integers(-6, 12, n))).astype(np.float32)
        hb = (rng.standard_normal(n) * 8).astype(np.float32)
        a.copy_(torch.from_numpy(ha))
        b.copy_(torch.from_numpy(hb))
        for buf in (bt, bq, bd, bh, br, bm, bmq, bms, bmd, bc):
            buf.view(torch.uint8).fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        what = f"replay {rnd}"
        wt = X.stream("triad", "f32", ha, hb, s)
        wq = F.quantize(wt, "f32", "e4m3", -3)
        wd = F.dequantize(wq, "e4m3", "f32", -3)
        wh = V.convert(wd, "f32", "bf16")
        wmq, wms = M.quantize(wt, "f32", "e5m2", 64, "nosat")
        for got, want, fmt, buf, k in ((t, wt, "f32", bt, n), (q, wq, "e4m3", bq, n), (dq, wd, "f32", bd, n),
                                       (h, wh, "bf16", bh, n), (r, _amax(D.dot(wh, wh, "bf16")), "f64", br, 1),
                                       (m, _amax(F.amax(wt, "f32")), "f64", bm, 1), (mq, wmq, "e5m2", bmq, n),
                                       (ms, wms, "u8", bms, wms.size),
                                       (md, M.dequantize(wmq, wms, "e5m2", "f16", 64), "f16", bmd, n),
                                       (c, oracle.vadd(ha, hb), "f32", bc, n)):
            assert_matches(got, to_dev(np.ascontiguousarray(want), fmt), fmt, f"{what} {fmt}", nan_class=fmt != "u8")
            assert_guards(buf, GUARD, k, f"{what} {fmt}")
    del g


# ------------------------------------------------------------------------------------------- not capturable
def test_loop_forms_inside_a_capture():
    """b200va_add_f32_loop with graph_batch > 1 and b200va_loop_create allocate and synchronize: inside a capture they
    return an error code, and afterwards direct launches work.  b200va_add_f32_loop refuses before it touches the
    capturing stream, so the rest of that capture stays valid.  b200va_loop_run of a handle made outside the capture
    cannot replay the handle's graph into it: the driver refuses the graph launch and invalidates the capture, and the
    handle still runs afterwards."""
    n = (1 << 20) + 3
    a, b = ctr_inputs(n)
    c, c2 = torch.empty_like(a), torch.empty_like(a)
    torch.cuda.synchronize()
    stream_ptr = lambda: torch.cuda.current_stream().cuda_stream
    # the one-shot loop: refused up front, so the rest of the capture stays valid
    g = torch.cuda.CUDAGraph()
    codes = {}
    with torch.cuda.graph(g):
        for v in ("auto", "k2"):
            codes[v] = capi.lib.b200va_add_f32_loop(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, capi.VARIANTS[v], 8, 4,
                                                    stream_ptr())
        va.add(a, b, c2, variant="k2")
    assert codes == {"auto": CUDA_CAPTURE_UNSUPPORTED, "k2": CUDA_CAPTURE_UNSUPPORTED}, codes
    c2.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    check_add(a, b, c2, n, "the add captured after the refused loops")
    del g
    # b200va_loop_create and b200va_loop_run make the driver invalidate the capture; torch.cuda.graph leaves its
    # capture stream current when the capture fails, so they run in a process of their own
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_gpu_graph_capture as m; m.loop_capture_child()"
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("REPORT ")]
    assert p.returncode == 0 and lines, f"exit {p.returncode}\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    rep = json.loads(lines[-1][len("REPORT "):])
    print(rep)
    assert rep["create"][0] < 0 and rep["create"][1:] == [False, False], rep   # refused, no handle, capture invalid
    assert rep["run"] == [CUDA_CAPTURE_UNSUPPORTED, False], rep                # a handle's graph is not replayed into a capture
    assert all(v == "ok" for k, v in rep.items() if k not in ("create", "run")), rep


def loop_capture_child():
    """b200va_loop_create (k2, graph_batch 4) and b200va_loop_run of a k2 handle, each inside a global-mode capture on
    a private stream; then direct add_loop and loop.run calls, verified.  Prints a JSON report."""
    n = (1 << 20) + 3
    a, b = ctr_inputs(n)
    c = torch.empty_like(a)
    torch.cuda.synchronize()
    rep = {}

    def inside_capture(fn):
        g, s, out = torch.cuda.CUDAGraph(), torch.cuda.Stream(), {}
        with torch.cuda.stream(s):
            g.capture_begin()
            try:
                out["rc"] = fn(s.cuda_stream)
            finally:
                try:
                    g.capture_end()
                    out["valid"] = True
                except RuntimeError:
                    out["valid"] = False
        torch.cuda.synchronize()
        return g, out["rc"], out["valid"]

    h = C.c_void_p()
    g, rc, valid = inside_capture(lambda st: capi.lib.b200va_loop_create(C.byref(h), a.data_ptr(), b.data_ptr(),
                                                                         c.data_ptr(), n, capi.K2_TMA, 4))
    rep["create"] = [rc, bool(h.value), valid]
    del g

    def add_loops():
        for v in ("auto", "k2"):
            c.fill_(-1.0)
            va.add_loop(a, b, c, 9, graph_batch=4, variant=v)
            torch.cuda.synchronize()
            check_add(a, b, c, n, f"add_loop {v} after the capture")

    rep["add_loop after"] = _report(add_loops)
    with va.Loop(a, b, c, graph_batch=4, variant="k2") as loop:
        g, rc, valid = inside_capture(lambda st: capi.lib.b200va_loop_run(loop._h, 9, st))
        rep["run"] = [rc, valid]
        if rc == 0 and valid:
            def replays():
                for _ in range(2):
                    c.fill_(-1.0)
                    g.replay()
                    torch.cuda.synchronize()
                    check_add(a, b, c, n, "loop_run captured and replayed")
            rep["replays"] = _report(replays)
        del g

        def run():
            c.fill_(-1.0)
            loop.run(9)
            torch.cuda.synchronize()
            check_add(a, b, c, n, "loop.run after the capture")

        rep["loop.run after"] = _report(run)
    print("REPORT " + json.dumps(rep))
