"""Stream order through chains of programmatic (PDL) launches, checked bit for bit against exact references.

The early-load forms of the f32 add (EARLY = 1: B200VA_F_INPUTS_STABLE, and launches 2.. of every launch chain)
read A and B before griddepcontrol.wait.  That is legal only while the one launch still allowed to run beside them
is the launch immediately before them on the stream.  Each case here is one chain on one stream:

  poison X (torch) -> W: X = P + Q -> 0..3 middle launches on small unrelated buffers -> a tail that reads a window of X

and the tail's output is compared with the exact reference of its operation applied to the exact window.

W is the production "k2" add (K2d, the TMA ring under the dynamic tile scheduler) at n = 2^28.  Its grid is
persistent, one 544-thread CTA per SM with about 128 KiB of shared memory, so every CTA starts, and passes its
trigger, at once; it then streams for about a millisecond, and the scheduler hands out tiles in order, so the end
of X (where the window lies) is written last.  Each SM keeps about 1500 threads free, so the small middle and tail
grids become resident beside it: a read of X that escapes the chain's order lands in a window about 1 ms wide and
sees the poison.  A multi-wave writer would not do: its last wave passes the trigger only just before it ends.
Nor would a K1d writer: its persistent grid fills the SMs, and nothing else becomes resident beside it.

Middle launches fit beside W (about 2^16 elements).  k0, the mixed-phase stream op and fill_ctr are launched
without the PDL attribute: they end the chain, and the cases behind them pass whatever the kernels do.

One run per case: the window is wide enough that one run decides it.  The same matrix runs once more in a
subprocess with B200VA_NO_PDL=1 (the library reads it once per process), where every launch is an ordinary one.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from conftest import ROOT, has_gpu
from oracle import convert_exact as V
from oracle import dot_exact as D
from oracle import stream_exact as X

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va
    from test_gpu_parity import k1d_tunes

N = 1 << 28                        # W's length: the HBM class, about 1 ms of streaming on an H100
LO = N - (1 << 18) - 3             # the window X[LO:LO + M]: ragged, 4 bytes past a 16-byte boundary
M = (1 << 18) - 5
SEED_P, SEED_Q, SEED_B = 0x0A, 0x0B, 0x0C
POISON = 0x5A5A5A5A                # a finite f32 (about 1.5e16): a stale read gives a definite wrong value
SMALL = 1 << 16                    # middle launches: grids that fit beside W
SCALE = 3.0


@pytest.fixture(scope="module")
def env():
    free, _ = torch.cuda.mem_get_info()
    if free < (4 << 30):
        pytest.skip(f"needs about 4 GiB of free device memory, {free >> 20} MiB free")
    e = {}
    e["P"] = va.fill_ctr(torch.empty(N, dtype=torch.float32, device="cuda"), SEED_P)
    e["Q"] = va.fill_ctr(torch.empty(N, dtype=torch.float32, device="cuda"), SEED_Q)
    e["X"] = torch.empty(N, dtype=torch.float32, device="cuda")
    # tail operands and outputs share the window's 16-byte phase (one element past it), so the vector forms run
    e["B"] = va.fill_ctr(torch.empty(M + 1, dtype=torch.float32, device="cuda"), SEED_B)[1:]
    e["C"] = torch.empty(M + 1, dtype=torch.float32, device="cuda")[1:]
    e["H"] = torch.empty(M + 1, dtype=torch.float16, device="cuda")[1:]
    e["dot"] = torch.empty(1, dtype=torch.float64, device="cuda")
    e["ws"] = torch.empty(max(capi.lib.b200va_dot_workspace_bytes(max(M, SMALL)), 8), dtype=torch.uint8, device="cuda")
    # the middle launches' own buffers
    e["ma"] = va.fill_ctr(torch.empty(SMALL + 4, dtype=torch.float32, device="cuda"), 0x1A)
    e["mb"] = va.fill_ctr(torch.empty(SMALL + 4, dtype=torch.float32, device="cuda"), 0x1B)
    e["mc"] = torch.empty(SMALL + 4, dtype=torch.float32, device="cuda")
    e["mh"] = torch.empty(SMALL, dtype=torch.float16, device="cuda")
    e["mdot"] = torch.empty(1, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    host_b = e["B"].cpu().numpy()
    window = oracle.vadd(oracle.fill_ctr(M, SEED_P, LO), oracle.fill_ctr(M, SEED_Q, LO))
    e["ref_window"] = window
    e["ref_add"] = oracle.vadd(window, host_b)
    e["ref_scale"] = X.stream("scale", "f32", window, None, SCALE)
    e["ref_triad"] = X.stream("triad", "f32", window, host_b, SCALE)
    e["ref_f16"] = V.convert(window, "f32", "f16")
    e["ref_dot"] = D.dot(window, host_b, "f32")
    yield e
    del e
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- middle launches
def _middles(e):
    """name -> (launch, launched with the PDL attribute)."""
    a, b, c = e["ma"][:SMALL], e["mb"][:SMALL], e["mc"][:SMALL]
    k1d = k1d_tunes()[0]
    m = {
        "add auto": (lambda: va.add(a, b, c), True),
        "add k1": (lambda: va.add(a, b, c, variant="k1"), True),
        "add k3": (lambda: va.add(a, b, c, variant="k3"), True),
        "add k2 (K2d below the HBM class)": (lambda: va.add(a, b, c, variant="k2"), True),
        "add k0": (lambda: va.add(a, b, c, variant="k0"), False),
        "add K4 (mixed phase)": (lambda: va.add(e["ma"][:SMALL], e["mb"][1:SMALL + 1], e["mc"][2:SMALL + 2]), True),
        "add K1d tune": (lambda: va.add(a, b, c, tune=k1d), True),
        "stream copy": (lambda: va.stream("copy", a, out=c), True),
        "stream scale": (lambda: va.stream("scale", a, out=c, scalar=SCALE), True),
        "stream add": (lambda: va.stream("add", a, b, c), True),
        "stream triad": (lambda: va.stream("triad", a, b, c, scalar=SCALE), True),
        "stream add (mixed phase)": (lambda: va.stream("add", e["ma"][1:SMALL + 1], e["mb"][:SMALL], e["mc"][:SMALL]), False),
        "convert f32->f16": (lambda: va.convert(a, "f16", e["mh"]), True),
        "dot f32": (lambda: va.dot(a, b, out=e["mdot"], workspace=e["ws"]), True),
        "probe copy": (lambda: va.probe("copy", a, None, c), True),
        "fill_ctr": (lambda: va.fill_ctr(c, 0x1C), False),
    }
    return m


def _chains(e):
    """The middle sequences: none, each middle alone, and runs of two and three."""
    m = _middles(e)
    chains = [()] + [(k,) for k in m]
    chains += [("add auto", "stream add"), ("convert f32->f16", "dot f32"), ("probe copy", "add K1d tune"),
               ("add k2 (K2d below the HBM class)", "add k3"), ("stream triad", "add k0"),
               ("add k1", "stream copy", "add auto"), ("dot f32", "add K4 (mixed phase)", "stream scale"),
               ("fill_ctr", "add auto", "add k1"), ("add auto", "add k0", "stream add")]
    return m, chains


# ------------------------------------------------------------------------------------------- tails
def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32 if x.dtype == np.float32 else np.uint16)


def _tails(e):
    """name -> (run on the window, check -> None or a message, early loads: needs a middle launch before it)."""
    B, C, H = e["B"], e["C"], e["H"]

    def same(got, want):
        g, w = _bits(got), _bits(want)
        if np.array_equal(g, w):
            return None
        bad = np.flatnonzero(g != w)
        return f"{bad.size} of {w.size} elements differ, first at {bad[0]}"

    def add_ok():
        return same(C.cpu().numpy(), e["ref_add"])

    def scale_ok():
        return same(C.cpu().numpy(), e["ref_scale"])

    def triad_ok():
        return same(C.cpu().numpy(), e["ref_triad"])

    def f16_ok():
        return same(H.cpu().view(torch.int16).numpy().view(np.uint16), e["ref_f16"])

    def dot_ok():
        got, want = float(e["dot"].item()), e["ref_dot"]
        return None if np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64) else f"dot {got!r}, want {want!r}"

    return {
        "add_loop x2": (lambda w: va.add_loop(w, B, C, 2), add_ok, False),
        "add_loop x5": (lambda w: va.add_loop(w, B, C, 5), add_ok, False),
        "add_loop x3, graph_batch 16": (lambda w: va.add_loop(w, B, C, 3, graph_batch=16), add_ok, False),
        "Loop(batch 16).run(3)": (lambda w: e["loop"].run(3), add_ok, False),
        "add inputs_stable": (lambda w: va.add(w, B, C, inputs_stable=True), add_ok, True),
        "add inputs_stable cold": (lambda w: va.add(w, B, C, inputs_stable=True, cold=True), add_ok, True),
        "add": (lambda w: va.add(w, B, C), add_ok, False),
        "stream scale": (lambda w: va.stream("scale", w, out=C, scalar=SCALE), scale_ok, False),
        "stream triad": (lambda w: va.stream("triad", w, B, C, scalar=SCALE), triad_ok, False),
        "convert f32->f16": (lambda w: va.convert(w, "f16", H), f16_ok, False),
        "dot f32": (lambda w: va.dot(w, B, out=e["dot"], workspace=e["ws"]), dot_ok, False),
    }


def _poison(e):
    e["X"].view(torch.int32).fill_(POISON)
    e["C"].fill_(-7.0)
    e["H"].fill_(-7.0)
    e["dot"].fill_(-7.0)


def _run(e, middles, names, tail):
    """One chain on the current stream, one synchronise: the tail's output is left for its check."""
    _poison(e)
    va.add(e["P"], e["Q"], e["X"], variant="k2")
    for k in names:
        middles[k][0]()
    tail(e["X"][LO:LO + M])
    torch.cuda.synchronize()


def test_early_load_sizes_resolve_to_register_loads_ahead_of_the_wait():
    """The window's length is in the classes where B200VA_F_INPUTS_STABLE, with or without B200VA_F_COLD, gives
    the register-load form; W is the dynamically scheduled TMA ring."""
    for flags in (capi.F_INPUTS_STABLE, capi.F_INPUTS_STABLE | capi.F_COLD):
        assert capi.resolve(capi.K_AUTO, M, flags).early_loads == 1
    t = capi.resolve(capi.K2_TMA, N)
    assert (t.kind, t.store_mode, t.threads) == (capi.K2_TMA, 2, 512)


def test_the_same_chains_without_programmatic_launch():
    """The whole matrix again with B200VA_NO_PDL=1, in a process of its own: the references and the harness are
    right, so a failure above depends on programmatic launch."""
    torch.cuda.empty_cache()                        # what earlier modules left cached, so the child finds its 4 GiB
    env_ = dict(os.environ, B200VA_NO_PDL="1")
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.abspath(__file__), "-k", "not without_programmatic_launch"],
                       cwd=ROOT, env=env_, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-6000:] + p.stderr[-3000:]
    assert " passed" in p.stdout and "skipped" not in p.stdout, p.stdout[-3000:]


@pytest.mark.parametrize("tail", ["add_loop x2", "add_loop x5", "add_loop x3, graph_batch 16", "Loop(batch 16).run(3)",
                                  "add inputs_stable", "add inputs_stable cold", "add", "stream scale", "stream triad",
                                  "convert f32->f16", "dot f32"])
def test_tail_reads_what_the_writer_wrote(env, tail):
    """Every middle sequence in front of one tail.  An early-load tail (B200VA_F_INPUTS_STABLE) needs at least
    one middle launch: the header lets it overlap the launch immediately before it, which must not write its
    inputs."""
    middles, chains = _chains(env)
    run, check, early = _tails(env)[tail]
    with va.Loop(env["X"][LO:LO + M], env["B"], env["C"], graph_batch=16) as loop:
        env["loop"] = loop
        failures = []
        for names in chains:
            if early and not names:
                continue
            _run(env, middles, names, run)
            bad = check()
            if bad:
                failures.append(f"W -> {' -> '.join(names) or '(nothing)'} -> {tail}: {bad}")
        del env["loop"]
    assert not failures, "\n".join(failures)


def test_captured_chain_replays_in_stream_order(env):
    """W -> a PDL middle -> the launch loop's direct chain, captured into a torch CUDA graph (so the programmatic
    edges are in the graph), replayed twice with X poisoned again outside the graph before each replay."""
    middles, _ = _chains(env)
    B, C = env["B"], env["C"]
    window = env["X"][LO:LO + M]

    def chain():
        va.add(env["P"], env["Q"], env["X"], variant="k2")
        middles["add k1"][0]()
        va.add_loop(window, B, C, 3)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                      # every library setup call happens before the capture
        _poison(env)
        chain()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        chain()
    for replay in range(2):
        _poison(env)
        g.replay()
        torch.cuda.synchronize()
        got = _bits(C.cpu().numpy())
        bad = np.flatnonzero(got != _bits(env["ref_add"]))
        assert bad.size == 0, f"replay {replay}: {bad.size} elements differ, first at {bad[0]}"
    del g
