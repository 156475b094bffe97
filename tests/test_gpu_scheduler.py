"""The dynamic tile scheduler of K1d (vadd_vec_dyn) and K2d (vadd_tma_dyn, what variant k2 runs): every tile is
written exactly once, also when a ticket counter is used again.

A dynamically scheduled launch claims tiles from a two-word counter that must be zero when it starts; its last CTA
zeroes the counter again.  Direct launches take their counter from the device's ring of 4096 slots, a loop handle's
graph from the handle (csrc/b200va_add.cu: sched_slot, b200va_loop).  A counter that is not zero makes a launch
skip tiles and report nothing, so every launch here writes into an output poisoned beforehand with a finite pattern
and is verified afterwards: the device recompute, the oracle's digest, and the oracle element by element on windows
at the head, the middle and the ragged tail, plus guard elements on both sides that must keep the poison.  Most
launches have at least 3x as many tiles as the persistent grid; only then does a ticket offset left behind by an
earlier launch reach tiles that would otherwise be written.
"""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    import k8s_gpu_hpa_b200 as pkg
    from gpu_helpers import SIZES, assert_bits_equal, dev
    from k8s_gpu_hpa_b200 import capi, vector_add as va

RING = 4096                 # ticket-counter slots per device (kSchedSlots)
POISON = 0x7F7F7F7F         # a 0x7F byte fill: 3.39e38, finite (NaN would match NaN in the bit comparison)
WIN = 128                   # elements per oracle window
GUARD = 4                   # elements past the end (and one before a misaligned start) that must stay poisoned
ROUND = 256                 # launches between two synchronisations


class Form:
    """A dynamically scheduled form of the production library: a K1d tune, or variant k2 in one size class."""

    def __init__(self, name, device, tune=None, k2_n=0):
        self.name, self.tune = name, tune
        t = tune if tune is not None else capi.resolve(capi.K2_TMA, k2_n)
        assert t.kind == capi.K2_TMA or t.scheduler == 1
        # variant k2 resolves its geometry from n: the shapes of a k2 form stay in k2_n's size class
        self.n_range = (1, 1 << 40) if tune is not None else (1 << 25, 1 << 40) if k2_n >= 1 << 25 else (1, (1 << 25) - 1)
        self.tile = t.tile_bytes // 4 if t.kind == capi.K2_TMA else t.threads * t.unroll * 4       # elements per tile
        grid, block, smem = C.c_uint(), C.c_uint(), C.c_uint()
        probe = k2_n if tune is None else 1 << 28
        capi.check(capi.lib.b200va_geometry(C.byref(t), probe, device, C.byref(grid), C.byref(block), C.byref(smem)),
                   "b200va_geometry")
        self.grid = grid.value                                   # the persistent grid: every CTA resident at once
        assert self.grid < (probe + self.tile - 1) // self.tile  # (not capped by the probe's tile count)

    def n(self, shape: str) -> int:
        """big: >= 3x as many tiles as the grid (+ a ragged tail); exact: as many tiles as the grid; few: fewer;
        tiny1..3: no vector body (the edges travel with tile 0)."""
        if shape.startswith("tiny"):
            return int(shape[4:])
        n = {"big": (3 * self.grid + 1) * self.tile + 3, "exact": self.grid * self.tile,
             "few": (self.grid // 2) * self.tile + 5}[shape]
        n = max(n, self.n_range[0] + 3)
        assert n <= self.n_range[1], (self.name, shape, n)
        return n

    def launch(self, a, b, c, stream):
        if self.tune is None:
            va.add(a, b, c, variant="k2", stream=stream)
        else:
            va.add(a, b, c, tune=self.tune, stream=stream)


def production_forms(device):
    k1d = lambda unroll, early: capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=unroll, st_hint=1, scheduler=1,
                                          early_loads=early)
    return {"k1d_early0": Form("k1d_early0", device, k1d(2, 0)),
            "k1d_early1": Form("k1d_early1", device, k1d(4, 1)),
            "k1d_early2": Form("k1d_early2", device, k1d(2, 2)),
            "k2_small": Form("k2_small", device, k2_n=(1 << 25) - 1),
            "k2_large": Form("k2_large", device, k2_n=1 << 25)}


# (form, shape, offset of A, B and C in elements).  Big shapes on the even positions, everything else on the odd
# ones; 17 entries, so that the launch 4096 later -- the next user of a launch's ring slot -- sits one position
# earlier in the cycle (4096 = 16 mod 17): the slot of every small launch is next used by a big one.
CYCLE = [("k1d_early0", "big", 0), ("k1d_early2", "tiny1", 0), ("k2_small", "big", 0), ("k1d_early0", "few", 0),
         ("k1d_early1", "big", 1), ("k2_small", "exact", 0), ("k2_large", "big", 0), ("k2_small", "tiny3", 2),
         ("k1d_early2", "big", 0), ("k1d_early0", "exact", 0), ("k2_small", "big", 3), ("k2_small", "few", 1),
         ("k1d_early1", "big", 0), ("k1d_early0", "tiny2", 1), ("k1d_early2", "big", 2), ("k1d_early1", "few", 0),
         ("k1d_early0", "big", 3)]


class Expected:
    """What the oracle says about C[off:off+n] for the counter-generated inputs (A[i] = ctr(0x0A, i), B[i] = ctr(0x0B, i))."""

    def __init__(self, device):
        self.device, self.cache = device, {}

    def __call__(self, n, off):
        if (n, off) not in self.cache:
            spans = [(0, min(n, WIN)), (max(0, n // 2 - WIN // 2), min(n, n // 2 + WIN // 2)), (max(0, n - WIN), n)]
            idx = [np.arange(off + lo, off + hi) for lo, hi in spans]
            want = [oracle.vadd(oracle.fill_ctr(hi - lo, oracle.SEED_A, off + lo), oracle.fill_ctr(hi - lo, oracle.SEED_B, off + lo))
                    .view(np.uint32) for lo, hi in spans]
            guards = np.array(([off - 1] if off else []) + list(range(off + n, off + n + GUARD)))
            idx = np.concatenate(idx + [guards])
            want = np.concatenate(want + [np.full(guards.size, POISON, np.uint32)])
            pad = 3 * WIN + 1 + GUARD - idx.size                   # a fixed width: repeat the first element
            idx = np.concatenate([idx, np.full(pad, idx[0])])
            want = np.concatenate([want, np.full(pad, want[0], np.uint32)])
            self.cache[(n, off)] = (oracle.ctr_vadd_digest(n, off), torch.from_numpy(idx).to(self.device), want)
        return self.cache[(n, off)]


def inputs(n, device):
    a = torch.empty(n, dtype=torch.float32, device=device)
    b = torch.empty_like(a)
    va.fill_ctr(a, oracle.SEED_A)
    va.fill_ctr(b, oracle.SEED_B)
    return a, b


def poison(c, end=None):
    c[:end].view(torch.int32).fill_(POISON)


class Checker:
    """Checks of C[off:off+n] enqueued on `stream` right behind the add that wrote it; resolved once per round."""

    def __init__(self, device, stream, expected):
        self.stream, self.expected = stream, expected
        self.res = torch.empty((ROUND, 4), dtype=torch.int64, device=device)       # verify (count, first), digest
        self.win = torch.empty((ROUND, 3 * WIN + 1 + GUARD), dtype=torch.int32, device=device)
        self.pending = []
        self.checked = 0

    def record(self, a, b, c, n, off, what):
        k = len(self.pending)
        digest, idx, want = self.expected(n, off)
        pa, pb, pc = (x.data_ptr() + 4 * off for x in (a, b, c))
        st = self.stream.cuda_stream
        capi.check(capi.lib.b200va_verify_f32(pa, pb, pc, n, self.res[k].data_ptr(), st), "b200va_verify_f32")
        capi.check(capi.lib.b200va_digest_f32(pc, n, self.res[k, 2:].data_ptr(), st), "b200va_digest_f32")
        with torch.cuda.stream(self.stream):
            torch.index_select(c.view(torch.int32), 0, idx, out=self.win[k])
        self.pending.append((n, off, what, digest, want))
        if len(self.pending) == ROUND:
            self.flush()

    def flush(self):
        self.stream.synchronize()
        res = self.res[:len(self.pending)].cpu().numpy().view(np.uint64)
        win = self.win[:len(self.pending)].cpu().numpy().view(np.uint32)
        for k, (n, off, what, digest, want) in enumerate(self.pending):
            bad, first = int(res[k, 0]), int(res[k, 1])
            assert bad == 0, f"{what}: {bad} of {n} elements wrong, the first at {first}"
            assert (int(res[k, 2]), int(res[k, 3])) == digest, f"{what}: digest differs from the oracle's"
            wrong = np.nonzero(win[k] != want)[0]
            assert wrong.size == 0, f"{what}: window element {wrong[0]} is {win[k][wrong[0]]:08x}, want {want[wrong[0]]:08x}"
        self.checked += len(self.pending)
        self.pending.clear()


def run_direct_launches(device, stream, count, forms, cycle, buffers=4):
    """`count` direct launches of `cycle` on `stream`, each into one of `buffers` rotating outputs poisoned right
    before it and checked right after it."""
    shapes = [(forms[f], forms[f].n(s), off, f"{f} {s}") for f, s, off in cycle]
    end = max(n + off for _, n, off, _ in shapes) + GUARD
    a, b = inputs(end, device)
    outs = [torch.empty(end, dtype=torch.float32, device=device) for _ in range(buffers)]
    check = Checker(device, stream, Expected(device))
    for i in range(count):
        form, n, off, what = shapes[i % len(shapes)]
        c = outs[i % buffers]
        with torch.cuda.stream(stream):
            poison(c, off + n + GUARD)
        form.launch(a[off:off + n], b[off:off + n], c[off:off + n], stream)
        check.record(a, b, c, n, off, f"launch {i} ({what}, n={n}, offset {off})")
    check.flush()
    assert check.checked == count


def check_now(a, b, c, n, what):
    """Synchronous form of the Checker's checks, for a whole output."""
    assert va.verify(a, b, c) == (0, -1), what
    assert va.digest(c) == oracle.ctr_vadd_digest(n), what
    for lo in (0, n // 2 - WIN // 2, n - WIN):
        assert_bits_equal(c[lo:lo + WIN], oracle.vadd(oracle.fill_ctr(WIN, oracle.SEED_A, lo), oracle.fill_ctr(WIN, oracle.SEED_B, lo)),
                          f"{what} [{lo}, {lo + WIN})")


def devices():
    count = torch.cuda.device_count() if has_gpu() else 0
    last = pytest.mark.skipif(count < 2, reason="one device: the ring of device 0 is covered by the other case")
    return [pytest.param(0, id="device0"), pytest.param(max(count - 1, 1), id="last_device", marks=last)]


def test_k1d_vec_kernel_ragged_sizes_and_offsets():
    """K1d, the sm_90a replacement of the cluster-launch-control vec kernel: the vec tile body with
    tiles handed out by the ticket counter -- every tile exactly once, the scalar head/tail travel
    with tile 0."""
    nmax = max(SIZES)
    ha, hb = oracle.fill_ctr(nmax + 8, 0x0A, 78), oracle.fill_ctr(nmax + 8, 0x0B, 78)
    a, b = dev(ha), dev(hb)
    for t in (capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=2, st_hint=1, scheduler=1),
              capi.Tune(kind=capi.K1_VEC128, threads=64, unroll=4, st_hint=1, scheduler=1, early_loads=1),
              capi.Tune(kind=capi.K3_VEC256, threads=32, unroll=1, st_hint=1, scheduler=1)):
        for n in SIZES:
            for off in (0, 1, 3):
                out = torch.full((n + 16,), -3.0, dtype=torch.float32, device="cuda")
                va.add(a[off:off + n], b[off:off + n], out[off:off + n], tune=t, full_matrix=True)
                torch.cuda.synchronize()
                assert_bits_equal(out[off:off + n], oracle.vadd(ha[off:off + n].copy(), hb[off:off + n].copy()), f"k1d n={n} off={off}")
                assert (out[:off] == -3.0).all() and (out[off + n:] == -3.0).all()
    n = 1 << 24
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    y = torch.empty_like(x)
    z = torch.empty_like(x)
    va.fill_ctr(x, 0x0A)
    va.fill_ctr(y, 0x0B)
    t = capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=2, st_hint=1, scheduler=1, early_loads=1)
    for _ in range(50):
        va.add(x, y, z, tune=t)
    assert va.digest(z) == oracle.ctr_vadd_digest(n) and va.verify(x, y, z) == (0, -1)
    # ctas_per_sm (static persistent split) and the dynamic scheduler exclude each other
    with pytest.raises(pkg.B200VAError):
        va.add(x, y, z, tune=capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=2, st_hint=1, scheduler=1, ctas_per_sm=2))


def test_k2d_tma_kernel_ragged_sizes_and_offsets():
    """store_mode 2 (on sm_90a the dynamic tile scheduler takes the place of cluster launch control):
    a persistent grid whose CTAs claim tiles from the ticket counter -- every tile must be processed
    exactly once whatever the tile count."""
    nmax = max(SIZES)
    ha, hb = oracle.fill_ctr(nmax + 8, 0x0A, 77), oracle.fill_ctr(nmax + 8, 0x0B, 77)
    a, b = dev(ha), dev(hb)
    for t in (capi.Tune(kind=capi.K2_TMA, threads=128, st_hint=1, stages=4, tile_bytes=8192, store_mode=2),
              capi.Tune(kind=capi.K2_TMA, threads=64, st_hint=0, stages=3, tile_bytes=2048, store_mode=2)):
        for n in SIZES:
            for off in (0, 1, 3):
                out = torch.full((n + 16,), -3.0, dtype=torch.float32, device="cuda")
                va.add(a[off:off + n], b[off:off + n], out[off:off + n] if off + n <= n + 16 else out[:n], tune=t)
                torch.cuda.synchronize()
                got = out[off:off + n] if off + n <= n + 16 else out[:n]
                assert_bits_equal(got, oracle.vadd(ha[off:off + n].copy(), hb[off:off + n].copy()), f"k2d n={n} off={off}")
    # back-to-back launches (PDL chain) keep producing the same bits
    n = 1 << 24
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    y = torch.empty_like(x)
    z = torch.empty_like(x)
    va.fill_ctr(x, 0x0A)
    va.fill_ctr(y, 0x0B)
    t = capi.Tune(kind=capi.K2_TMA, threads=128, st_hint=1, stages=4, tile_bytes=8192, store_mode=2)
    for _ in range(50):
        va.add(x, y, z, tune=t)
    assert va.digest(z) == oracle.ctr_vadd_digest(n) and va.verify(x, y, z) == (0, -1)


@pytest.mark.parametrize("device", devices())
def test_ticket_ring_wraps_twice_with_every_launch_verified(device):
    """2 x 4096 + 64 direct K1d / K2d launches on one stream: every slot of the device's ring is used at least
    twice, whatever earlier tests left its cursor at, so a slot that one launch leaves non-zero shows up in a later
    one.  K1d at early loads 0, 1 and 2 and variant k2 in both size classes; more tiles than the grid, exactly as
    many, fewer, no vector body at all, misaligned heads."""
    with torch.cuda.device(device):
        stream = torch.cuda.Stream(device=device)
        run_direct_launches(device, stream, 2 * RING + 64, production_forms(device), CYCLE)


@pytest.mark.parametrize("batch", [2, 7, 50])
@pytest.mark.parametrize("n", [(1 << 24) + 5, (1 << 25) + 5], ids=["k2_small", "k2_large"])
def test_k2_loop_graph_replays_write_every_tile(n, batch):
    """Every replay of a loop handle's graph reuses the counters of its nodes.  C is poisoned before every run: the
    nodes of a replay all write the same C, so without the poison a node that skipped tiles would be hidden by the
    node before it."""
    form = Form("k2", 0, k2_n=n)
    assert n >= 3 * form.grid * form.tile
    a, b = inputs(n, "cuda")
    c = torch.empty_like(a)
    with va.Loop(a, b, c, graph_batch=batch, variant="k2") as loop:
        for iters in (batch, batch, batch, 2 * batch + 1):      # one replay each, then two and a direct launch
            poison(c)
            loop.run(iters)
            check_now(a, b, c, n, f"Loop(graph_batch={batch}).run({iters})")
    for _ in range(2):
        poison(c)
        va.add_loop(a, b, c, 2 * batch + 1, graph_batch=batch, variant="k2")
        check_now(a, b, c, n, f"add_loop(iters={2 * batch + 1}, graph_batch={batch})")


def test_k2_loop_graph_next_to_direct_launches_on_another_stream():
    """A k2 loop graph replays on stream X while a second host thread issues more than 4096 direct K1d / K2d
    launches into its own buffers on stream Y: the ring hands out every slot during the replays, and none of them
    may be a counter the graph uses.  Every Y launch and every X replay is verified."""
    n, batch = (1 << 24) + 5, 50
    a, b = inputs(n, "cuda")
    c = torch.empty_like(a)
    forms = production_forms(0)
    cycle = [e for e in CYCLE if e[0] != "k2_large"]
    errors, done = [], threading.Event()

    def direct():
        try:
            torch.cuda.set_device(0)
            run_direct_launches(0, torch.cuda.Stream(), RING + 64, forms, cycle)
        except BaseException as e:      # noqa: BLE001 -- reported to the main thread
            errors.append(repr(e))
        finally:
            done.set()

    sx = torch.cuda.Stream()
    y = threading.Thread(target=direct)
    replays = 0
    with torch.cuda.stream(sx), va.Loop(a, b, c, graph_batch=batch, variant="k2") as loop:
        y.start()
        try:
            while replays < 4 or (not done.is_set() and replays < 2000):
                poison(c)
                loop.run(batch)
                check_now(a, b, c, n, f"replay {replays}")
                replays += 1
        finally:
            y.join()
    assert not errors, errors
