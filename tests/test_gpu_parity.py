"""Parity tests proper: the CUDA path, called through the C ABI, against the CPU oracle --
bit-exact (this is fp32 add.rn: one correct answer per element).

Small/medium sizes: element-by-element against the oracle on the same seeded inputs and
the committed golden fixtures.  BASELINE.json's full sizes (2^28 on one GPU, 2^30 in 8
shards): through size-independent properties -- the order-independent digest of the
result equals the oracle's digest of A+B (a checksum of checksums over shards), the
device-side recompute finds no mismatch, commutativity, idempotence, in-place == out-of-place.
"""
import json
import os

import numpy as np
import pytest

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    import k8s_gpu_hpa_b200 as pkg
    from gpu_helpers import (SIZES, assert_bits_equal, dev, geometry, k1d_tunes, profiled_kernel_name,
                             trace_events)
    from k8s_gpu_hpa_b200 import capi, vector_add as va

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ALL = ["auto", "k0", "k1", "k2", "k3"]


@pytest.mark.parametrize("variant", ALL)
def test_sample_recipe_n50000_known_answer(variant):
    """The reference default: N = 50000, never-seeded rand() inputs (config 1 on the GPU)."""
    ha, hb = va.fill_rand_host(50000)
    c = va.add(dev(ha), dev(hb), variant=variant)
    torch.cuda.synchronize()
    hc = c.cpu().numpy()
    assert oracle.fnv1a64(hc) == 0x000CC9DBE012E750
    assert_bits_equal(hc, oracle.vadd(ha, hb), variant)
    assert va.digest(c) == (53174197755249, 0x0118998B)
    assert oracle.verify_sample_tolerance(ha, hb, hc) == -1          # the sample's own check


@pytest.mark.parametrize("variant", ALL)
def test_ragged_sizes_against_oracle(variant):
    nmax = max(SIZES)
    ha, hb = oracle.fill_ctr(nmax, 0x0A), oracle.fill_ctr(nmax, 0x0B)
    want = oracle.vadd(ha, hb)
    a, b = dev(ha), dev(hb)
    for n in SIZES:
        out = torch.full((n + 16,), -3.0, dtype=torch.float32, device="cuda")
        va.add(a[:n], b[:n], out[:n], variant=variant)
        torch.cuda.synchronize()
        assert_bits_equal(out[:n], want[:n], f"{variant} n={n}")
        assert (out[n:] == -3.0).all(), f"{variant} n={n}: wrote past the end"


@pytest.mark.parametrize("variant", ALL)
def test_every_misalignment_of_the_three_pointers(variant):
    """Pointers need only 4-byte alignment: same offset (head peel), and mixed offsets
    (scalar path) for A, B, C, with ragged tails."""
    n = 10_007
    pad = 16
    ha, hb = oracle.fill_ctr(n + pad, 0x0A, 99), oracle.fill_ctr(n + pad, 0x0B, 99)
    a, b = dev(ha), dev(hb)
    offs = [(o, o, o) for o in range(9)] + [(1, 2, 3), (0, 4, 0), (4, 4, 0), (0, 0, 1), (3, 3, 7), (8, 4, 12), (5, 1, 5)]
    for oa, ob, oc in offs:
        for m in (n, n - 1, n - 5, 6, 3):
            out = torch.full((n + 2 * pad,), -3.0, dtype=torch.float32, device="cuda")
            va.add(a[oa:oa + m], b[ob:ob + m], out[oc:oc + m], variant=variant)
            torch.cuda.synchronize()
            assert_bits_equal(out[oc:oc + m], oracle.vadd(ha[oa:oa + m].copy(), hb[ob:ob + m].copy()),
                              f"{variant} offs={(oa, ob, oc)} m={m}")
            assert (out[:oc] == -3.0).all() and (out[oc + m:] == -3.0).all()


@pytest.mark.parametrize("variant", ALL)
def test_golden_special_values(variant):
    """+-0, subnormals (no FTZ), +-Inf, NaN, overflow, ties-to-even, catastrophic cancellation."""
    g = np.load(os.path.join(GOLD, "special_values.npz"))
    ua, ub, uc = g["a_bits"], g["b_bits"], g["c_bits"]
    reps = 37                                        # long enough for vector bodies and TMA tiles
    c = va.add(dev(np.tile(ua, reps).view(np.float32)), dev(np.tile(ub, reps).view(np.float32)), variant=variant)
    torch.cuda.synchronize()
    assert_bits_equal(c, np.tile(uc, reps).view(np.float32), variant)
    # subnormal results really are produced (FTZ would zero them)
    got = c.cpu().numpy().view(np.uint32)
    assert ((got & 0x7F800000) == 0).any() and ((got & 0x7FFFFFFF) > 0)[((got & 0x7F800000) == 0)].any()


@pytest.mark.parametrize("variant", ALL)
def test_golden_ctr_fixture(variant):
    g = json.load(open(os.path.join(GOLD, "ctr_1m.json")))
    n, first = g["n"], g["first"]
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    va.fill_ctr(a, g["seed_a"], first)
    va.fill_ctr(b, g["seed_b"], first)
    assert f"{oracle.fnv1a64(a.cpu().numpy()):016x}" == g["fnv1a64"]["A"]   # device generator == host generator
    assert f"{oracle.fnv1a64(b.cpu().numpy()):016x}" == g["fnv1a64"]["B"]
    c = va.add(a, b, variant=variant)
    assert f"{oracle.fnv1a64(c.cpu().numpy()):016x}" == g["fnv1a64"]["C"]
    assert va.digest(c) == (g["C_bits_sum"], int(g["C_bits_xor"], 16))


@pytest.mark.parametrize("variant", ALL)
def test_exact_aliasing_and_overlap_rules(variant):
    n = 70_001
    ha, hb = oracle.fill_ctr(n, 0x0A, 5), oracle.fill_ctr(n, 0x0B, 5)
    want = oracle.vadd(ha, hb)
    a, b = dev(ha), dev(hb)
    va.add(a, b, a, variant=variant)                 # C == A
    assert_bits_equal(a, want, f"{variant} C==A")
    a = dev(ha)
    va.add(a, b, b, variant=variant)                 # C == B
    assert_bits_equal(b, want, f"{variant} C==B")
    x = dev(ha)
    va.add(x, x, x, variant=variant)                 # A == B == C
    assert_bits_equal(x, oracle.vadd(ha, ha), f"{variant} A==B==C")
    big = dev(np.concatenate([ha, hb]))
    with pytest.raises(pkg.B200VAError) as e:        # C partially overlaps A
        va.add(big[:n], big[n:2 * n], big[4:n + 4], variant=variant)
    assert e.value.code == capi.ERR_OVERLAP


def test_argument_errors():
    a = torch.zeros(64, dtype=torch.float32, device="cuda")
    assert capi.lib.b200va_add_f32(None, a.data_ptr(), a.data_ptr(), 64, 0, None) == capi.ERR_INVALID
    assert capi.lib.b200va_add_f32(a.data_ptr() + 2, a.data_ptr(), a.data_ptr(), 8, 0, None) == capi.ERR_ALIGN
    assert capi.lib.b200va_add_f32(a.data_ptr(), a.data_ptr(), a.data_ptr(), 64, 17, None) == capi.ERR_VARIANT
    assert capi.lib.b200va_add_f32(None, None, None, 0, 0, None) == capi.OK       # n == 0 is a no-op
    t = capi.Tune(kind=capi.K1_VEC128, threads=100, unroll=4)
    with pytest.raises(pkg.B200VAError):
        va.add(a, a, tune=t)
    t = capi.Tune(kind=capi.K2_TMA, threads=256, stages=64, tile_bytes=1 << 20, store_mode=1)
    with pytest.raises(pkg.B200VAError):
        va.add(a, a, tune=t)
    with pytest.raises(pkg.B200VAError):
        va.add(a, a, tune=capi.Tune(kind=capi.K1_VEC128, threads=128, unroll=2, early_loads=7))
    b = torch.ones_like(a)
    va.add(a, b, a, tune=capi.Tune(kind=capi.K1_VEC128, threads=128, unroll=2, early_loads=2))      # the L2 prefetch is legal in place
    va.add(a, b, a, tune=capi.Tune(kind=capi.K1_VEC128, threads=128, unroll=2, early_loads=1))      # register loads are swapped for it
    torch.cuda.synchronize()
    assert bool((a == 2.0).all())


def test_tuned_geometries_are_all_bit_exact():
    """Every knob of the tune struct (unroll, CTA size, persistence, hints, ring depth,
    tile size, store mode) changes the schedule, never the bits."""
    n = 2_500_003
    ha, hb = oracle.fill_ctr(n, 0x0A, 1 << 40), oracle.fill_ctr(n, 0x0B, 1 << 40)
    want = oracle.vadd(ha, hb)
    a, b = dev(ha), dev(hb)
    geos = []
    for kind in (capi.K1_VEC128, capi.K3_VEC256):
        for unroll in (1, 2, 4, 8):
            for cps in (0, 2):
                geos.append(capi.Tune(kind=kind, threads=256, unroll=unroll, ctas_per_sm=cps, ld_hint=1, st_hint=1))
        for ld in range(6):
            for st in range(4):
                geos.append(capi.Tune(kind=kind, threads=128, unroll=2, ctas_per_sm=0, ld_hint=ld, st_hint=st))
        for threads in (32, 64, 512, 1024):
            geos.append(capi.Tune(kind=kind, threads=threads, unroll=1, ctas_per_sm=1))
    for mode in (0, 1):
        for stages, tile in ((2, 2048), (3, 8192), (6, 16384), (4, 28672), (8, 4096)):
            for threads in (32, 128, 512):
                for ld in (0, 3):
                    geos.append(capi.Tune(kind=capi.K2_TMA, threads=threads, ctas_per_sm=1, ld_hint=ld, st_hint=1,
                                          stages=stages, tile_bytes=tile, store_mode=mode))
        geos.append(capi.Tune(kind=capi.K2_TMA, threads=256, ctas_per_sm=2, stages=3, tile_bytes=16384, store_mode=mode))
    for stages, tile in ((2, 2048), (3, 8192), (4, 8192), (5, 4096), (6, 16384), (4, 28672)):      # dynamic tile scheduler
        for threads in (32, 128, 512):
            geos.append(capi.Tune(kind=capi.K2_TMA, threads=threads, ld_hint=0, st_hint=1, stages=stages, tile_bytes=tile,
                                  store_mode=2))
    for threads in (32, 256, 1024):                                  # 4-byte accesses, U loads per array in flight
        for unroll in (4, 8, 16):
            geos.append(capi.Tune(kind=capi.K4_SCALAR_MLP, threads=threads, unroll=unroll))
    for kind in (capi.K1_VEC128, capi.K3_VEC256):                    # early loads / L2 prefetch and the dynamic scheduler (K1d)
        for early in (0, 1, 2):
            for unroll in (1, 2, 4, 8):
                for threads in (64, 256, 512):
                    geos.append(capi.Tune(kind=kind, threads=threads, unroll=unroll, ld_hint=0, st_hint=1, early_loads=early, scheduler=1))
            geos.append(capi.Tune(kind=kind, threads=128, unroll=2, ctas_per_sm=2, ld_hint=3, st_hint=0, early_loads=early))
    geos.append(capi.Tune(kind=capi.K3_VEC256, threads=1024, unroll=8))
    for t in geos:
        out = torch.full((n,), -1.0, dtype=torch.float32, device="cuda")
        geo_rc = geometry(t, n, capi.tune_lib())[0]           # b200va_geometry refuses exactly what the launch refuses
        if t.kind == capi.K3_VEC256 and t.threads == 1024 and t.unroll == 8:
            with pytest.raises(pkg.B200VAError) as e:        # 1024 threads x 8 32-byte vectors per array: register-limited, refused
                va.add(a, b, out, tune=t, full_matrix=True)
            assert e.value.code == capi.ERR_VARIANT and geo_rc == capi.ERR_VARIANT
            va.add(a, b, out)                                  # and the refusal leaves no latched CUDA error behind
            torch.cuda.synchronize()
            assert_bits_equal(out, want, "after refused launch")
            continue
        try:
            va.add(a, b, out, tune=t, full_matrix=True)
        except pkg.B200VAError as e:
            # register-limited CTA sizes are refused up front (ERR_VARIANT), never fail at launch
            live = t.threads * t.unroll * (2 if t.kind == capi.K3_VEC256 else 1)
            assert e.code == capi.ERR_VARIANT and t.kind in (capi.K1_VEC128, capi.K3_VEC256) and live >= 8192, t.as_dict()
            assert geo_rc == e.code, t.as_dict()
            continue
        assert geo_rc == capi.OK, t.as_dict()
        torch.cuda.synchronize()
        assert_bits_equal(out, want, str(t.as_dict()))


PRODUCTION_SIZES = (1 << 10, 1 << 20, 1 << 21, 1 << 22, 1 << 23, 1 << 24, 1 << 28)


def production_tunes():
    """(size, tune): what AUTO and the named variants resolve to for each size class and hint."""
    return [(size, pkg.resolve(v, size, flags)) for size in PRODUCTION_SIZES for v in pkg.VARIANTS.values()
            for flags in (0, capi.F_INPUTS_STABLE, capi.F_COLD, capi.F_COLD | capi.F_INPUTS_STABLE)]


def test_production_library_carries_the_production_set_only():
    """libb200va.so: what AUTO and the named variants resolve to (+ early loads, + K1d) runs; a
    geometry only the A/B matrix has is refused with ERR_VARIANT -- and runs in libb200va_tune.so.
    b200va_geometry of the same library answers for exactly the tunes that run."""
    n = 300_003
    ha, hb = oracle.fill_ctr(n, 0x0A), oracle.fill_ctr(n, 0x0B)
    want = oracle.vadd(ha, hb)
    a, b = dev(ha), dev(hb)
    # the geometry of each size class and hint, run on our n
    for t in [t for _, t in production_tunes()] + list(k1d_tunes()):
        out = torch.full((n,), -1.0, dtype=torch.float32, device="cuda")
        va.add(a, b, out, tune=t)
        assert geometry(t, n)[0] == capi.OK, t.as_dict()
        assert_bits_equal(out, want, str(t.as_dict()))
    exotic = capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=8, ld_hint=2, st_hint=2)
    with pytest.raises(pkg.B200VAError) as e:
        va.add(a, b, tune=exotic)
    assert e.value.code == capi.ERR_VARIANT
    assert geometry(exotic, n)[0] == capi.ERR_VARIANT
    assert_bits_equal(va.add(a, b, tune=exotic, full_matrix=True), want, "tune library")
    assert geometry(exotic, n, capi.tune_lib())[0] == capi.OK


def test_launched_kernel_has_the_geometry_and_name_the_library_reports(tmp_path):
    """Every tune the production library resolves, and its K1d tunes, launched once under the profiler on
    256-byte-aligned buffers of the n it was resolved for: the kernel in the trace has b200va_geometry's grid and
    block, and Tune.kernel_name() is its name."""
    cases = {}
    for size, t in production_tunes() + [(size, t) for size in PRODUCTION_SIZES for t in k1d_tunes()]:
        cases.setdefault((size, tuple(t.as_dict().values())), t)
    nmax = max(PRODUCTION_SIZES)
    a, b, c = (torch.empty(nmax, dtype=torch.float32, device="cuda") for _ in range(3))
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    assert all(x.data_ptr() % 256 == 0 for x in (a, b, c))
    torch.cuda.synchronize()
    want = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for (n, _), t in cases.items():
            rc, grid, block = geometry(t, n)
            assert rc == capi.OK, t.as_dict()
            va.add(a[:n], b[:n], c[:n], tune=t)
            want.append((t.kernel_name(), grid, block, n))
        torch.cuda.synchronize()
    events = trace_events(prof, tmp_path, ("kernel",))
    got = [(profiled_kernel_name(e["name"]), e["args"]["grid"][0], e["args"]["block"][0]) for e in events]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w[:3], (g, w)


def test_early_loads_chain_of_launches_is_bit_exact():
    """B200VA_F_INPUTS_STABLE: back-to-back launches whose loads run ahead of the dependency on the
    previous launch.  Rotating disjoint buffer sets (the stager's / sweep's shape), the same set
    repeatedly (the launch loop's shape), and a consumer chain C -> next launch's A, where the
    flag must NOT be given -- stream order of C has to hold either way."""
    n = (1 << 22) + 5
    sets = 5
    A = [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(sets)]
    B = [torch.empty_like(A[0]) for _ in range(sets)]
    Cs = [torch.zeros_like(A[0]) for _ in range(sets)]
    for s in range(sets):
        va.fill_ctr(A[s], 0x0A, s * n)
        va.fill_ctr(B[s], 0x0B, s * n)
    torch.cuda.synchronize()
    for variant in ("auto", "k1", "k3", "k2", "k0"):
        for c in Cs:
            c.zero_()
        for i in range(40):
            s = i % sets
            va.add(A[s], B[s], Cs[s], variant=variant, inputs_stable=True)
        for s in range(sets):
            assert va.verify(A[s], B[s], Cs[s]) == (0, -1), (variant, s)
            assert va.digest(Cs[s]) == oracle.ctr_vadd_digest(n, s * n)
        # same buffers every launch
        for _ in range(30):
            va.add(A[0], B[0], Cs[1], variant=variant, inputs_stable=True)
        assert va.verify(A[0], B[0], Cs[1]) == (0, -1)
        # the cold-data hint only changes the geometry AUTO picks, never the bits
        for i in range(12):
            s = i % sets
            va.add(A[s], B[s], Cs[s], variant=variant, inputs_stable=bool(i & 1), cold=True)
        for s in range(sets):
            assert va.verify(A[s], B[s], Cs[s]) == (0, -1), (variant, s)
    # write-after-write order on C is kept: the later launch's values must win
    for _ in range(20):
        va.add(A[0], B[0], Cs[0], inputs_stable=True)
        va.add(A[1], B[1], Cs[0], inputs_stable=True)
    assert va.verify(A[1], B[1], Cs[0]) == (0, -1)
    # aliasing: the hint is dropped inside the library (C == A feeds the next launch)
    x = A[2].clone()
    for _ in range(8):
        va.add(x, B[2], x, inputs_stable=True)
    ref = oracle.fill_ctr(n, 0x0A, 2 * n)
    hb = oracle.fill_ctr(n, 0x0B, 2 * n)
    for _ in range(8):
        ref = oracle.vadd(ref, hb)
    assert_bits_equal(x, ref, "in-place chain")
    assert capi.lib.b200va_add_f32_ex(x.data_ptr(), x.data_ptr(), x.data_ptr(), n, 0, 0x80, None) == capi.ERR_INVALID


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 1023, 1 << 16, (1 << 20) + 3, 7_000_001])
def test_support_kernels_vector_and_scalar_paths_agree(n):
    """fill_ctr / verify / digest have a 128-bit form for 16-byte-aligned pointers and a scalar one otherwise:
    both must give the host generator's values, the oracle's digest and the same verdict (count and FIRST bad index)."""
    big = torch.empty(3 * (n + 8), dtype=torch.float32, device="cuda")
    for off in (0, 1):                                    # 16-byte aligned / misaligned views
        a, b, c = (big[k * (n + 8) + off: k * (n + 8) + off + n] for k in range(3))
        va.fill_ctr(a, 0x0A, 12345)
        va.fill_ctr(b, 0x0B, 12345)
        ha, hb = oracle.fill_ctr(n, 0x0A, 12345), oracle.fill_ctr(n, 0x0B, 12345)
        assert_bits_equal(a, ha, f"fill off={off}")
        assert_bits_equal(b, hb, f"fill off={off}")
        va.add(a, b, c)
        assert va.verify(a, b, c) == (0, -1)
        assert va.digest(c) == oracle.bits_digest(oracle.vadd(ha, hb))
        if n >= 5:
            bad = sorted({n - 1, n // 2, 4 if n > 8 else 2})        # the ragged tail, the middle, an early element
            for i in bad:
                c.view(torch.int32)[i] ^= 0x10
            assert va.verify(a, b, c) == (len(bad), bad[0]), (off, bad)


def test_ceiling_probes_move_the_bytes_they_claim():
    """b200va_probe_f32: FILL writes 1.0 to every vector element, COPY copies A, READ2 leaves one partial sum per CTA
    (so its loads cannot have been elided) and touches nothing else; argument errors are refused."""
    n = (1 << 20) + 4 * 123
    ha, hb = oracle.fill_ctr(n, 0x0A), oracle.fill_ctr(n, 0x0B)
    a, b = dev(ha), dev(hb)
    c = torch.full((n,), -3.0, dtype=torch.float32, device="cuda")
    va.probe("fill", None, None, c)
    assert bool((c == 1.0).all())
    va.probe("copy", a, None, c)
    assert_bits_equal(c, ha, "copy probe")
    c.fill_(-3.0)
    va.probe("read2", a, b, c)
    torch.cuda.synchronize()
    ctas = (n // 4 + 511) // 512
    got = c.cpu().numpy()
    assert (got[ctas:] == -3.0).all()
    for k in (0, 1, ctas - 1):                     # thread 0 of CTA k summed vector 512 k of A and of B
        v = 512 * k * 4
        want = np.float32(0)
        for x, y in zip(ha[v:v + 4], hb[v:v + 4]):
            want = np.float32(np.float32(want + x) + y)
        assert got[k] == want
    assert capi.lib.b200va_probe_f32(7, a.data_ptr(), b.data_ptr(), c.data_ptr(), n, None) == capi.ERR_VARIANT
    assert capi.lib.b200va_probe_f32(0, a.data_ptr() + 4, b.data_ptr(), c.data_ptr(), n, None) == capi.ERR_ALIGN
    assert capi.lib.b200va_probe_f32(0, None, b.data_ptr(), c.data_ptr(), n, None) == capi.ERR_INVALID


def test_device_verify_and_digest_detect_a_single_flipped_bit():
    n = 1_000_001
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    c = va.add(a, b)
    assert va.verify(a, b, c) == (0, -1)
    good = va.digest(c)
    assert good == oracle.ctr_vadd_digest(n)
    c.view(torch.int32)[777_777] ^= 1
    assert va.verify(a, b, c) == (1, 777_777)
    assert va.digest(c) != good


@pytest.mark.parametrize("variant", ["auto", "k1", "k2", "k3"])
def test_full_size_2p28_properties(variant):
    """BASELINE.json configs[1]: N = 2^28 on one H100 (3 GiB of operands)."""
    n = 1 << 28
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    c = torch.empty_like(a)
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    va.add(a, b, c, variant=variant)
    want = oracle.ctr_vadd_digest(n)                       # oracle on the box's host cores, streaming
    assert va.digest(c) == want                            # checksum of the whole result
    assert va.verify(a, b, c) == (0, -1)                   # device recompute, bit for bit
    # element-by-element against the oracle on a sampled window at a ragged offset
    lo, m = (1 << 27) + 12345, 1 << 20
    assert_bits_equal(c[lo:lo + m], oracle.vadd(oracle.fill_ctr(m, 0x0A, lo), oracle.fill_ctr(m, 0x0B, lo)), variant)
    # commutativity and idempotence
    c2 = torch.empty_like(c)
    va.add(b, a, c2, variant=variant)
    assert va.digest(c2) == want and bool((c.view(torch.int32) == c2.view(torch.int32)).all())
    va.add(a, b, c2, variant=variant)
    va.add(a, b, c2, variant=variant)
    assert va.digest(c2) == want
    del c2
    # in place == out of place
    va.add(a, b, a, variant=variant)
    assert va.digest(a) == want


def test_full_size_2p30_in_8_shards_checksum_of_checksums():
    """BASELINE.json configs[2]: N = 2^30 sharded 8 ways (here: the 8 shards run one after
    another on one GPU; tests of the real 8-GPU run live in bench.py / the CLI)."""
    n, world = 1 << 30, 8
    s, x = 0, 0
    a = torch.empty(n // world, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    c = torch.empty_like(a)
    for r in range(world):
        lo, hi = pkg.shard_range(n, world, r)
        assert hi - lo == n // world
        va.fill_ctr(a, 0x0A, lo)                           # global index: sharding invisible in the data
        va.fill_ctr(b, 0x0B, lo)
        va.add(a, b, c)
        ds, dx = va.digest(c)
        assert (ds, dx) == oracle.ctr_vadd_digest(hi - lo, lo)
        assert va.verify(a, b, c) == (0, -1)
        s, x = (s + ds) & ((1 << 64) - 1), x ^ dx
    assert (s, x) == oracle.ctr_vadd_digest(n)


def test_beyond_32_bit_indexing_n_2p32_plus():
    """n > 2^32 elements (48 GiB of operands): every index and byte offset must be 64-bit.
    The sample's `int numElements` shape would wrap here; checked through the digest of the
    whole result and the device recompute, plus an oracle window straddling element 2^32."""
    n = (1 << 32) + 12_345
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * 4 * n + (2 << 30):
        pytest.skip("needs ~50 GiB of free device memory")
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty(n, dtype=torch.float32, device="cuda")
    c = torch.empty(n, dtype=torch.float32, device="cuda")
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    want = oracle.ctr_vadd_digest(n)
    lo, m = (1 << 32) - 4096, 12_000                       # window across the 2^32 boundary
    win = oracle.vadd(oracle.fill_ctr(m, 0x0A, lo), oracle.fill_ctr(m, 0x0B, lo))
    for variant in ("auto", "k2", "k0"):
        c.zero_()
        va.add(a, b, c, variant=variant)
        assert va.digest(c) == want, variant
        assert va.verify(a, b, c) == (0, -1), variant
        assert_bits_equal(c[lo:lo + m], win, variant)
        assert_bits_equal(c[n - 5000:], oracle.vadd(oracle.fill_ctr(5000, 0x0A, n - 5000), oracle.fill_ctr(5000, 0x0B, n - 5000)), variant)


def test_launch_loop_matches_single_launch_with_and_without_graphs():
    """Every variant, in the one-shot loop and a persistent loop handle.  C is poisoned (a finite 0x7F byte pattern)
    before every run and checked after it: every launch of a run writes the same C, so only a fresh pattern shows a
    launch that left part of C unwritten."""
    import ctypes as C

    n = 1 << 22
    a = torch.empty(n, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    va.fill_ctr(a, 0x0A)
    va.fill_ctr(b, 0x0B)
    want = oracle.ctr_vadd_digest(n)
    c = torch.empty_like(a)
    s = torch.cuda.Stream()
    for variant in ALL:
        with torch.cuda.stream(s):
            for iters, batch in ((1, 0), (7, 0), (50, 10), (53, 10), (5, 8)):
                c.view(torch.int32).fill_(0x7F7F7F7F)
                va.add_loop(a, b, c, iters, graph_batch=batch, variant=variant)
                s.synchronize()
                assert va.digest(c) == want, (variant, iters, batch)
        # the legacy default stream is fine too: the batch is captured on a private stream
        c.view(torch.int32).fill_(0x7F7F7F7F)
        rc = capi.lib.b200va_add_f32_loop(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, capi.VARIANTS[variant], 20, 10, None)
        assert rc == capi.OK
        torch.cuda.synchronize()
        assert va.digest(c) == want, variant
        # persistent loop handle: one capture, many replays
        h = C.c_void_p()
        assert capi.lib.b200va_loop_create(C.byref(h), a.data_ptr(), b.data_ptr(), c.data_ptr(), n, capi.VARIANTS[variant], 16) == capi.OK
        for iters in (16, 40, 3, 16):
            with torch.cuda.stream(s):
                c.view(torch.int32).fill_(0x7F7F7F7F)
            assert capi.lib.b200va_loop_run(h, iters, s.cuda_stream) == capi.OK
            s.synchronize()
            assert va.digest(c) == want, (variant, iters)
        assert capi.lib.b200va_loop_destroy(h) == capi.OK
