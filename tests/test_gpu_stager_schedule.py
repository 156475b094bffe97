"""The stager's chunk pipelines as the GPU runs them, read from a profiler trace: per mode, the chunk lengths,
the copies and the add of each chunk, the streams they run on, and the order that data flow and slot reuse
impose between them."""
import json

import numpy as np
import pytest

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va
    from test_gpu_parity import _profiled_kernel_name, geometry

MODES = [0, 2, 3, 4]        # slot streams, lanes, pageable bounce ring, register-once
CASES = [                   # (n, chunk, depth)
    (3_000_011, 1 << 20, 1),            # depth 1: no taper, and every chunk reuses the one slot
    ((23 << 19) + 13, 4 << 20, 3),      # the lanes taper the tail once; more chunks than slots
    ((20 << 20) + 5, 16 << 20, 2),      # the bounce chunk is capped at 2^23; the lanes taper three times
    (1_000_003, 1 << 16, 2),            # many small chunks over two slots
]


def schedule(mode: int, n: int, chunk: int, depth: int) -> list[int]:
    """The chunk lengths b200va_stager_add_f32 stages n elements in (chunk a multiple of 64, depth given)."""
    out, off = [], 0
    while off < n:
        left = n - off
        if mode == capi.STAGE_BOUNCE:
            m = min(chunk, 1 << 23, left)
        elif mode == capi.STAGE_SLOTS or left > chunk or depth == 1:
            m = min(chunk, left)
        else:
            m = (left // 2 + 63) & ~63
            if m < 1 << 20 or m >= left:
                m = left
        out.append(m)
        off += m
    return out


def test_schedule_restatement_tapers_the_lanes_tail():
    assert schedule(2, (20 << 20) + 5, 16 << 20, 2) == [16 << 20, (2 << 20) + 64, 1 << 20, (1 << 20) - 59]
    assert schedule(3, (20 << 20) + 5, 16 << 20, 2) == [8 << 20, 8 << 20, (4 << 20) + 5]
    assert schedule(0, (20 << 20) + 5, 16 << 20, 2) == [16 << 20, (4 << 20) + 5]
    assert schedule(2, 3_000_011, 1 << 20, 1) == [1 << 20, 1 << 20, 3_000_011 - (2 << 20)]


@pytest.fixture(scope="module")
def marker():
    return torch.zeros(1, device="cuda")


def _host_arrays(mode, n):
    """Pinned tensors for the modes made for pinned memory, plain numpy arrays for the bounce ring and register-once."""
    ha, hb = oracle.fill_ctr(n, 0x0A, 7), oracle.fill_ctr(n, 0x0B, 7)
    hc = np.full(n, -1.0, np.float32)
    if mode in (capi.STAGE_SLOTS, capi.STAGE_LANES):
        return [torch.from_numpy(x).pin_memory() for x in (ha, hb, hc)]
    return [ha, hb, hc]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n,chunk,depth", CASES)
def test_stager_trace_follows_the_chunk_schedule(tmp_path, marker, mode, n, chunk, depth):
    ha, hb, hc = _host_arrays(mode, n)
    lens = schedule(mode, n, chunk, depth)
    torch.cuda.synchronize()
    with va.Stager(0, chunk, depth) as st:
        # A trace can miss the GPU work of the first milliseconds after the profiler starts (a whole first call
        # and the marker after it, seen once).  So the call runs twice, a fill kernel between the two, and the
        # second call is checked.
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            st.add(ha, hb, hc, mode=mode)
            marker.fill_(1.0)
            torch.cuda.synchronize()
            st.add(ha, hb, hc, mode=mode)
        assert st.last_mode == mode
    assert oracle.first_mismatch(np.asarray(hc), oracle.vadd(np.asarray(ha), np.asarray(hb))) == -1

    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    # Every call to the runtime gets the next correlation id, so sorting by it puts the GPU work in issue order.
    events = sorted((e for e in json.loads(trace.read_text())["traceEvents"]
                     if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["args"]["correlation"])
    ours = [e for e in events if e["cat"] == "gpu_memcpy" or (e["cat"] == "kernel" and "vadd" in e["name"])]
    # The second call is the last 4 events per chunk: its two H2D copies, its add, its D2H copy.  The trace must
    # hold something issued before it (the first call, the marker), so it began before the second call did.
    run = ours[-4 * len(lens):]
    assert len(events) > len(run), [e["name"] for e in events[:8]]
    assert events[-len(run):] == run, [e["name"] for e in events[-len(run) - 1:][:8]]
    chunks = [run[4 * k:4 * k + 4] for k in range(len(lens))]

    start = lambda e: round(e["ts"] * 1000)               # noqa: E731 -- ns, exact: the trace has µs to 3 places
    end = lambda e: start(e) + round(e["dur"] * 1000)     # noqa: E731
    for k, (mk, (a, b, kern, c)) in enumerate(zip(lens, chunks)):
        # sizes and kernels
        assert [e["cat"] for e in (a, b, kern, c)] == ["gpu_memcpy", "gpu_memcpy", "kernel", "gpu_memcpy"], k
        assert "HtoD" in a["name"] and "HtoD" in b["name"] and "DtoH" in c["name"], k
        assert a["args"]["bytes"] == b["args"]["bytes"] == c["args"]["bytes"] == 4 * mk, (k, mk)
        t = capi.resolve(capi.K_AUTO, mk, capi.F_COLD)
        rc, grid, block = geometry(t, mk)
        assert rc == capi.OK
        assert (_profiled_kernel_name(kern["name"]), kern["args"]["grid"][0], kern["args"]["block"][0]) == \
               (t.kernel_name(), grid, block), (k, mk)
        # data flow: the add reads what the H2D copies wrote, the D2H copy reads what the add wrote
        assert start(kern) >= max(end(a), end(b)), k
        assert start(c) >= end(kern), k
        # slot reuse: chunk k overwrites slot k % depth only after chunk k - depth's result has left it
        if k >= depth:
            assert min(start(a), start(b)) >= end(chunks[k - depth][3]), k

    stream = lambda e: e["args"]["stream"]  # noqa: E731
    if mode == capi.STAGE_SLOTS:
        for k, ch in enumerate(chunks):
            assert len({stream(e) for e in ch}) == 1, k
            assert stream(ch[0]) == stream(chunks[k % depth][0]), k
        assert len({stream(ch[0]) for ch in chunks}) == min(depth, len(chunks))
    else:
        lanes = [{stream(ch[i]) for ch in chunks} for i in range(4)]
        assert lanes[0] == lanes[1] and len(lanes[0]) == 1 and len(lanes[2]) == 1 and len(lanes[3]) == 1
        assert len(lanes[0] | lanes[2] | lanes[3]) == 3
