"""What the GPU test modules share: the format tables, poisoned device buffers and one bit-pattern comparator,
restatements of the library's launch plans, a profiler capture behind a marker kernel, and the stream-order chains of
programmatic launches.

It imports torch, so a test module imports it inside its `if has_gpu():` block, as it imports torch.
"""
import ctypes as C
import json
import re

import numpy as np
import pytest
import torch

import oracle
from k8s_gpu_hpa_b200 import capi, vector_add as va
from oracle import convert_exact as V
from oracle import dot_exact as D
from oracle import stream_exact as X

# ------------------------------------------------------------------------------------------- formats
TORCH = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16,
         "e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "u8": torch.uint8}
INT = {"f32": torch.int32, "f64": torch.int64, "f16": torch.int16, "bf16": torch.int16,
       "e4m3": torch.uint8, "e5m2": torch.uint8, "u8": torch.uint8}
ES = {"f32": 4, "f64": 8, "f16": 2, "bf16": 2, "e4m3": 1, "e5m2": 1}
DT_CODE = {"f32": 0, "f64": 1, "f16": 2, "bf16": 3}
F8_CODE = {"e4m3": 0, "e5m2": 1}
# A pattern is a NaN iff its bits without the sign lie above these: exponent all ones and a nonzero mantissa (E4M3,
# which has no infinity, only S.1111.111).
NAN_ABOVE = {"f32": 0x7F800000, "f64": 0x7FF0000000000000, "f16": 0x7C00, "bf16": 0x7F80, "e4m3": 0x7E, "e5m2": 0x7C}


def hbm_n(es):
    """The smallest n in the HBM class: n elements of es bytes (the wider operand's) hold at least 2^25 four-byte
    words."""
    return (1 << 25) * 4 // es


# ------------------------------------------------------------------------------------------- device buffers
POISON = 0x5A               # byte fill: finite in every type (f16 0x5A5A = 203.25, bf16 1.5e16, f32 1.5e16, f64 ~4e127)
GUARD = 8                   # guard elements on each side; 8 elements of 2 bytes or more keep element 0 16-byte aligned


def to_dev(bits, fmt):
    """A device copy of host storage (values, or bit patterns for f16, bf16 and FP8) as fmt."""
    return torch.from_numpy(np.ascontiguousarray(bits)).cuda().view(TORCH[fmt])


def tiled(bits, n, fmt):
    """A device tensor of n elements: the host block repeated."""
    t = to_dev(bits, fmt).view(INT[fmt])
    t = t.repeat(-(-n // t.numel()))[:n] if n > t.numel() else t[:n].contiguous()
    return t.view(TORCH[fmt])


def poisoned(n, fmt, off=0):
    """(buffer, view): GUARD + off + n + GUARD elements of POISON bytes, the view is the n after GUARD + off."""
    buf = torch.empty(GUARD + off + n + GUARD, dtype=TORCH[fmt], device="cuda")
    buf.view(torch.uint8).fill_(POISON)
    return buf, buf[GUARD + off:GUARD + off + n]


def assert_guards(buf, start, n, what=""):
    """The GUARD elements before `start` and after start + n in buf still hold the poison."""
    es = buf.element_size()
    u8 = buf.view(torch.uint8)
    lo, hi = u8[max(0, start - GUARD) * es:start * es], u8[(start + n) * es:(start + n + GUARD) * es]
    assert bool((lo == POISON).all()) and bool((hi == POISON).all()), f"{what}: a guard element was written"


def _nan(bits, fmt):
    return (bits & ((1 << (8 * ES[fmt] - 1)) - 1)) > NAN_ABOVE[fmt]


def assert_matches(got, want, fmt, what="", nan_class=True, chunk=1 << 28):
    """Element by element on the device: the bit patterns are equal, or (if nan_class) both are NaNs of fmt."""
    assert got.numel() == want.numel(), what
    mask = (1 << (8 * got.element_size())) - 1
    for lo in range(0, got.numel(), chunk):
        g, w = got[lo:lo + chunk].view(INT[fmt]), want[lo:lo + chunk].view(INT[fmt])
        bad = g != w
        if nan_class:
            bad &= ~(_nan(g, fmt) & _nan(w, fmt))
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            raise AssertionError(f"{what}: {int(bad.sum())} mismatches, first at {lo + i} of {got.numel()}: "
                                 f"got {int(g[i]) & mask:#x} want {int(w[i]) & mask:#x} (bits)")


def dev(x: np.ndarray):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def assert_bits_equal(got, want: np.ndarray, what=""):
    g = got.cpu().numpy() if not isinstance(got, np.ndarray) else got
    bad = oracle.first_mismatch(g, want)
    assert bad < 0, f"{what}: first mismatch at {bad}: got {g.view(np.uint32)[bad]:08x} want {want.view(np.uint32)[bad]:08x}"


# ------------------------------------------------------------------------------------------- launch plans
SIZES = [0, 1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 255, 256, 257, 1023, 4095, 4096, 4097,
         50000, (1 << 16) - 1, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 3_000_017]


def geometry(t, n, lib=None):
    """b200va_geometry for tune t at n elements on the current device: (return code, grid, block)."""
    grid, block = C.c_uint(), C.c_uint()
    rc = (lib or capi.lib).b200va_geometry(C.byref(t), n, torch.cuda.current_device(), C.byref(grid), C.byref(block), None)
    return rc, grid.value, block.value


def expected_add_launch(t, n, pa, pb, pc, lib=None):
    """(return code, kernel, grid, block) of plan_launch (b200va_add.cu) for tune t, every field of its kind set, adding
    n elements at addresses pa and pb into pc.  The alias rules (.nc loads become plain, early register loads the L2
    prefetch, when C is A or B), the vector width and head (K3 drops to the 16-byte body, mixed phase to K4 at
    256 x 8) are restated here.  The grid is b200va_geometry's for the vector body alone, n_eff = nvec * vw elements
    with the effective tune: its notional aligned operands have no head, so they give the same tiles."""
    e = capi.Tune(**t.as_dict())
    if pc in (pa, pb):
        if e.ld_hint == 4:
            e.ld_hint = 0
        if e.early_loads == 1:
            e.early_loads = 2
    vw = {capi.K3_VEC256: 8, capi.K1_VEC128: 4, capi.K2_TMA: 4}.get(e.kind, 0)
    head = 0
    while vw:
        mask = vw * 4 - 1
        if pa & mask == pb & mask == pc & mask:
            head = ((vw * 4 - (pa & mask)) & mask) // 4
            break
        vw = 4 if vw == 8 else 0
    n_eff = n
    if vw:
        n_eff = (n - min(head, n)) // vw * vw
        if e.kind == capi.K3_VEC256 and vw == 4:
            e.kind = capi.K1_VEC128
    elif e.kind not in (capi.K0_SCALAR, capi.K4_SCALAR_MLP):
        e.kind, e.threads, e.unroll = capi.K4_SCALAR_MLP, 256, 8
    rc, grid, block = geometry(e, n_eff, lib)
    return rc, e.kernel_name(), grid, block


def expected_stream_launch(op, dtype, n, head=0, override=None):
    """(kernel, grid, block) launch_stream_typed (b200va_typed.cu) picks for n elements whose vector body starts head
    elements in.  override: (threads, unroll, skip_l1_stores) of B200VA_STREAM_GEOMETRY, which only the tune library
    reads; one it does not accept leaves the table's plan."""
    m = n * ES[dtype] // 4
    binary = op in ("add", "triad")
    if m >= 1 << 25:
        threads, unroll, st = (512, 1, 1) if binary else (1024, 2, 1)
    elif m > 1 << 23:
        threads, unroll, st = 128, 2, 0
    elif m >= 1 << 21:
        threads, unroll, st = 256, 2, 0
    elif m >= 1 << 19:
        threads, unroll, st = 512, 1, 0
    else:
        threads, unroll, st = 128, 1, 0
    if override and 32 <= override[0] <= 1024 and override[0] % 32 == 0 and override[1] in (1, 2, 4):
        threads, unroll, st = override[0], override[1], int(override[2] != 0)
    nvec = (n - min(head, n)) * ES[dtype] // 16
    grid = max(1, -(-nvec // (threads * unroll)))
    return f"stream_vec<{DT_CODE[dtype]},{capi.OPS[op]},{unroll},0,{st}>", grid, threads


def k1d_tunes():
    """The K1d (dynamic tile scheduler) tunes the production library carries."""
    return (capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=2, st_hint=1, scheduler=1),
            capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=4, st_hint=1, scheduler=1, early_loads=1))


def expected_cast_launch(kernel, esa, esc, n, a_ptr, c_ptr, units_per_group=1):
    """(kernel, grid, block) of plan_cast (b200va_typed.cu): n elements of esa bytes at a_ptr cast to esc bytes at
    c_ptr, with units_per_group units of work per group."""
    G = 16 // min(esa, esc)
    head, h = n, ((16 - a_ptr % 16) % 16) // esa
    while h < G:
        if (c_ptr + h * esc) % 16 == 0:
            head = h
            break
        h += 16 // esa
    head = min(head, n)
    ngroups = (n - head) // G
    units = ngroups * units_per_group
    edges = n - ngroups * G
    threads, unroll = (512, 2) if n >= hbm_n(max(esa, esc)) else (256, 1)
    blocks = max(-(-units // (threads * unroll)), -(-edges // threads))
    return kernel, max(1, min(blocks, 2 ** 31 - 1)), threads


def expected_mx_launch(kind, es, n, block, aligned):
    """(kernel, grid, block) of launch_mx_typed (b200va_typed.cu)."""
    nblocks = -(-n // block)
    if kind == "q":
        ngroups = n // block * (block // 16) if aligned else 0
        units, edges = ngroups, nblocks - ngroups * 16 // block
    else:
        ngroups = n // 16 if aligned else 0
        units, edges = ngroups * es, n - ngroups * 16
    threads, unroll = (512, 2) if n >= hbm_n(es) else (256, 1)
    blocks = max(-(-units // (threads * unroll)), -(-edges // threads))
    return f"mx_{'quant' if kind == 'q' else 'dequant'}_vec<{es}>", max(1, min(blocks, 2 ** 31 - 1)), threads


# ------------------------------------------------------------------------------------------- profiler traces
def profiled_kernel_name(name: str) -> str:
    """A kernel name as the profiler prints it, in Tune.kernel_name()'s form: no namespace, parameter list, casts
    or spaces, and bools as 0/1."""
    name = re.sub(r"\((?:int|bool|unsigned int)\)", "", name).replace("true", "1").replace("false", "0")
    return re.match(r"(?:void )?(?:b200va::)?(\w+(?:<[^>]*>)?)", name).group(1).replace(" ", "")


def trace_events(prof, tmp_path, cats):
    """The events of categories cats in the profiler's chrome trace, in order of their start."""
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    return sorted((e for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") in cats), key=lambda e: e["ts"])


def kernels_after_marker(tmp_path, run_plan, ours):
    """[(kernel, grid, block)] of every kernel and memset of the second of two run_plan() calls under the profiler.

    Late in a long test session the trace can miss the first kernels after the profiler starts (three warm-up
    kernels and the plan's first launch, seen once).  So the plan runs twice, a fill kernel marks the start of the
    second pass, and the second pass is returned.  Only kernels whose names contain one of the substrings in ours
    may follow the marker: any other kernel or memset there fails the marker check."""
    marker = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_plan()
        marker.fill_(1.0)
        torch.cuda.synchronize()
        run_plan()
    events = trace_events(prof, tmp_path, ("kernel", "gpu_memset"))
    m = max(i for i, e in enumerate(events) if not any(o in e["name"] for o in ours))
    assert events[m].get("cat") == "kernel" and "ill" in events[m]["name"], events[m]["name"]
    return [(profiled_kernel_name(e["name"]), e["args"]["grid"][0], e["args"]["block"][0]) for e in events[m + 1:]]


# ------------------------------------------------------------------------------------------- stream-order chains
# One chain on one stream: poison X -> W: X = P + Q -> 0..3 middle launches on small unrelated buffers -> a tail that
# reads the window X[LO:LO + M], whose output is compared with the exact reference of the window.
#
# W is the production "k2" add (K2d, the TMA ring under the dynamic tile scheduler) at n = 2^28.  Its grid is
# persistent, one 544-thread CTA per SM with about 128 KiB of shared memory, so every CTA starts, and passes its
# trigger, at once; it then streams for about a millisecond, and the scheduler hands out tiles in order, so the end
# of X (where the window lies) is written last.  Each SM keeps about 1500 threads free, so the small middle and tail
# grids become resident beside it: a read of X that escapes the chain's order lands in a window about 1 ms wide and
# sees the poison.  A multi-wave writer would not do: its last wave passes the trigger only just before it ends.
# Nor would a K1d writer: its persistent grid fills the SMs, and nothing else becomes resident beside it.
#
# Middle launches fit beside W (about 2^16 elements).  k0, the mixed-phase stream op and fill_ctr are launched
# without the PDL attribute: they end the chain, and the cases behind them pass whatever the kernels do.
N = 1 << 28                        # W's length: the HBM class, about 1 ms of streaming on an H100
LO = N - (1 << 18) - 3             # the window X[LO:LO + M]: ragged, 4 bytes past a 16-byte boundary
M = (1 << 18) - 5
SEED_P, SEED_Q, SEED_B = 0x0A, 0x0B, 0x0C
X_POISON = 0x5A5A5A5A              # X's f32 word: finite (about 1.5e16), so a stale read gives a definite wrong value
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


def _poison(e):
    e["X"].view(torch.int32).fill_(X_POISON)
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
