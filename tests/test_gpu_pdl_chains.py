"""Stream order through chains of programmatic (PDL) launches, checked bit for bit against exact references.

The early-load forms of the f32 add (EARLY = 1: B200VA_F_INPUTS_STABLE, and launches 2.. of every launch chain)
read A and B before griddepcontrol.wait.  That is legal only while the one launch still allowed to run beside them
is the launch immediately before them on the stream.  Each case here is one chain on one stream:

  poison X (torch) -> W: X = P + Q -> 0..3 middle launches on small unrelated buffers -> a tail that reads a window of X

and the tail's output is compared with the exact reference of its operation applied to the exact window.

gpu_helpers.py sets up W, the window and the middle launches, and says why they are chosen as they are.

One run per case: the window is wide enough that one run decides it.  The same matrix runs once more in a
subprocess with B200VA_NO_PDL=1 (the library reads it once per process), where every launch is an ordinary one.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from gpu_helpers import LO, M, N, SCALE, _chains, _poison, _run
    from gpu_helpers import env  # noqa: F401  (the module-scoped fixture)
    from k8s_gpu_hpa_b200 import capi, vector_add as va


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
