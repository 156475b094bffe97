"""Property-based parity (hypothesis): random lengths, pointer offsets, kernel variants and
bit patterns -- whatever the draw, the CUDA path returns the oracle's bits and writes
nothing outside [0, n)."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va

SPECIAL = np.array([0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000,
                    0xFF800000, 0x7FC00000, 0x3F800000, 0xBF800000, 0x33800000, 0x4B000000], dtype=np.uint32)
POOL = 1 << 18


@pytest.fixture(scope="module")
def pools():
    rng = np.random.default_rng(1234)
    ha = oracle.fill_ctr(POOL + 64, 0x0A, 11).view(np.uint32).copy()
    hb = oracle.fill_ctr(POOL + 64, 0x0B, 11).view(np.uint32).copy()
    # a quarter of the positions get arbitrary bit patterns, some get IEEE special values
    for h in (ha, hb):
        idx = rng.integers(0, h.size, h.size // 4)
        h[idx] = rng.integers(0, 1 << 32, idx.size, dtype=np.uint64).astype(np.uint32)
        idx = rng.integers(0, h.size, h.size // 16)
        h[idx] = SPECIAL[rng.integers(0, SPECIAL.size, idx.size)]
    ha, hb = ha.view(np.float32), hb.view(np.float32)
    return ha, hb, torch.from_numpy(ha).cuda(), torch.from_numpy(hb).cuda()


@settings(max_examples=150, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(n=st.one_of(st.integers(0, 70), st.integers(0, POOL)), oa=st.integers(0, 9), ob=st.integers(0, 9),
       oc=st.integers(0, 9), variant=st.sampled_from(["auto", "k0", "k1", "k2", "k3"]), same=st.booleans(), stable=st.booleans())
def test_random_lengths_offsets_variants(pools, n, oa, ob, oc, variant, same, stable):
    ha, hb, a, b = pools
    if same:
        ob = oc = oa            # equal misalignment: vector body with peeled head
    out = torch.full((n + 32,), -3.0, dtype=torch.float32, device="cuda")
    va.add(a[oa:oa + n], b[ob:ob + n], out[oc:oc + n], variant=variant, inputs_stable=stable)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = oracle.vadd(ha[oa:oa + n].copy(), hb[ob:ob + n].copy())
    assert oracle.first_mismatch(got[oc:oc + n].copy(), want) == -1
    assert (got[:oc] == -3.0).all() and (got[oc + n:] == -3.0).all()


@settings(max_examples=60, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(n=st.integers(1, POOL), threads=st.sampled_from([32, 64, 96, 128, 256, 320, 512, 1024]),
       unroll=st.sampled_from([1, 2, 4, 8]), cps=st.sampled_from([0, 1, 3]), ld=st.integers(0, 5), stt=st.integers(0, 3),
       wide=st.booleans(), early=st.integers(0, 2), dyn=st.booleans())
def test_random_vec_geometries(pools, n, threads, unroll, cps, ld, stt, wide, early, dyn):
    ha, hb, a, b = pools
    t = capi.Tune(kind=capi.K3_VEC256 if wide else capi.K1_VEC128, threads=threads, unroll=unroll, ctas_per_sm=0 if dyn else cps,
                  ld_hint=ld, st_hint=stt, early_loads=int(early), scheduler=int(dyn))
    try:
        out = va.add(a[:n], b[:n], tune=t, full_matrix=True)
    except capi.B200VAError as e:
        # the only legal refusal: a register-limited CTA size (>= 8192 live 128-bit vectors per array per CTA,
        # e.g. 1024 threads x 8, or 512 x 8 of the 256-bit kernel) -- refused up front, never a launch error
        assert e.code == capi.ERR_VARIANT and threads * unroll * (2 if wide else 1) >= 8192
        return
    torch.cuda.synchronize()
    assert oracle.first_mismatch(out.cpu().numpy(), oracle.vadd(ha[:n].copy(), hb[:n].copy())) == -1


@settings(max_examples=60, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(n=st.integers(1, POOL), threads=st.sampled_from([32, 64, 128, 256, 512]), stages=st.integers(2, 9),
       tile_k=st.sampled_from([2048, 4096, 8192, 12288, 16384]), mode=st.integers(0, 2), hint=st.booleans())
def test_random_tma_geometries(pools, n, threads, stages, tile_k, mode, hint):
    ha, hb, a, b = pools
    t = capi.Tune(kind=capi.K2_TMA, threads=threads, ctas_per_sm=1, ld_hint=3 if hint else 0, st_hint=1, stages=stages,
                  tile_bytes=tile_k, store_mode=mode)
    ring = stages * 2 * tile_k + (20 if mode == 2 else 16) * stages
    if ring > 227 * 1024:           # does not fit the 227 KiB opt-in shared memory: must be refused, not launched
        with pytest.raises(capi.B200VAError) as e:
            va.add(a[:n], b[:n], tune=t, full_matrix=True)
        assert e.value.code == capi.ERR_VARIANT
        return
    out = va.add(a[:n], b[:n], tune=t, full_matrix=True)
    torch.cuda.synchronize()
    assert oracle.first_mismatch(out.cpu().numpy(), oracle.vadd(ha[:n].copy(), hb[:n].copy())) == -1


@settings(max_examples=40, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(n=st.integers(0, POOL), chunk_log=st.integers(10, 17), depth=st.integers(1, 4), mode=st.sampled_from([-1, 0, 2, 3, 4]),
       pinned=st.booleans(), off=st.integers(0, 5))
def test_random_host_path_shapes(pools, n, chunk_log, depth, mode, pinned, off):
    """The host-buffer path with random lengths, chunk sizes, ring depths, pipelines and host memory kinds
    (pinned vs plain malloc, misaligned starts): always the oracle's bits, never a byte outside [0, n)."""
    ha, hb, _, _ = pools
    n = min(n, POOL - off)
    a, b = ha[off:off + n], hb[off:off + n]
    if pinned:
        a, b = torch.from_numpy(a.copy()).pin_memory(), torch.from_numpy(b.copy()).pin_memory()
        out = torch.full((n + 8,), -3.0).pin_memory()
        view, got = out[:n], out.numpy()
    else:
        a, b = a.copy(), b.copy()
        got = np.full(n + 8, -3.0, np.float32)
        view = got[:n]
    with va.Stager(0, 1 << chunk_log, depth) as stg:
        stg.add(a, b, view, mode=mode)
        stg.add(a, b, view, mode=mode)                      # second call: cached registration / reused ring
    want = oracle.vadd(ha[off:off + n].copy(), hb[off:off + n].copy())
    assert oracle.first_mismatch(got[:n].copy(), want) == -1
    assert (got[n:] == -3.0).all()
