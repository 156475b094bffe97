"""The host-buffer path (a3 + a4 + a6-copy of one ./vectorAdd process) and the drop-in
executable, on a real GPU, against the oracle."""
import json

import numpy as np
import pytest

import oracle
from conftest import has_gpu

pytestmark = pytest.mark.gpu
if has_gpu():
    import torch

    from k8s_gpu_hpa_b200 import capi, vector_add as va


@pytest.mark.parametrize("n", [0, 1, 5, 50000, (1 << 22) + 3, 3 * (1 << 22) + 17, 5 * (1 << 23) + 1234567])
def test_add_host_pageable_arrays(n):
    ha, hb = oracle.fill_ctr(n, 0x0A, 3), oracle.fill_ctr(n, 0x0B, 3)
    out = va.add_host(ha, hb)
    assert oracle.first_mismatch(out, oracle.vadd(ha, hb)) == -1


@pytest.mark.parametrize("zero_copy", [0, 1, 2, 3])      # slot streams, zero-copy kernel, lanes, pageable bounce
@pytest.mark.parametrize("chunk,depth", [(1 << 16, 2), (1 << 20, 3), (1 << 18, 1), (0, 0)])
def test_stager_pinned_pipeline(zero_copy, chunk, depth):
    n = 5_000_011
    ha = torch.from_numpy(oracle.fill_ctr(n, 0x0A, 1)).pin_memory()
    hb = torch.from_numpy(oracle.fill_ctr(n, 0x0B, 1)).pin_memory()
    hc = torch.full((n,), -1.0).pin_memory()
    want = oracle.vadd(ha.numpy(), hb.numpy())
    with va.Stager(0, chunk, depth) as st:
        for m in (n, n - 3, 1 << 16, 7):
            hc.fill_(-1.0)
            ms = st.add(ha[:m], hb[:m], hc[:m], mode=zero_copy)
            assert ms > 0
            assert oracle.first_mismatch(hc[:m].numpy(), want[:m]) == -1
            assert bool((hc[m:] == -1.0).all())


def test_stager_pageable_mode_on_plain_numpy_arrays():
    n = 30_000_001
    ha, hb = oracle.fill_ctr(n, 0x0A, 9), oracle.fill_ctr(n, 0x0B, 9)
    want = oracle.vadd(ha, hb)
    for chunk, depth in ((1 << 20, 1), (1 << 21, 2), (1 << 22, 3), (0, 0)):
        with va.Stager(0, chunk, depth) as st:
            for m in (n, n - 5, 123):
                hc = np.full(n, -1.0, np.float32)
                st.add(ha[:m], hb[:m], hc[:m], mode=3)
                assert oracle.first_mismatch(hc[:m].copy(), want[:m].copy()) == -1
                assert (hc[m:] == -1.0).all()


def test_stager_register_once_on_plain_malloced_arrays():
    """Mode 4 / AUTO: pageable arrays are page-locked in place on first sight, the registration is
    cached by address range, and later calls run the pinned lanes pipeline on the same arrays."""
    n = 12_000_017
    ha, hb = oracle.fill_ctr(n, 0x0A, 21), oracle.fill_ctr(n, 0x0B, 21)
    want = oracle.vadd(ha, hb)
    hc = np.full(n, -1.0, np.float32)

    with va.Stager(0, 1 << 21, 3) as st:
        ms_first = st.add(ha, hb, hc, mode=capi.STAGE_AUTO)
        assert st.last_mode == capi.STAGE_REGISTER and ms_first > 0
        assert oracle.first_mismatch(hc, want) == -1
        for m in (n, n - 7, 1 << 20):                         # sub-ranges of the cached registrations
            hc.fill(-1.0)
            st.add(ha[:m], hb[:m], hc[:m], mode=capi.STAGE_AUTO)
            assert st.last_mode == capi.STAGE_LANES             # now page-locked: AUTO sees pinned memory, nothing to register
            st.add(ha[:m], hb[:m], hc[:m], mode=capi.STAGE_REGISTER)
            assert st.last_mode == capi.STAGE_REGISTER          # explicit mode 4: cache hit, same pipeline
            assert oracle.first_mismatch(hc[:m].copy(), want[:m].copy()) == -1 and (hc[m:] == -1.0).all()
        # a pinned array is recognised as such (no double registration), tiny arrays take the bounce ring
        pc = torch.empty(n, dtype=torch.float32).pin_memory()
        st.add(ha, hb, pc, mode=capi.STAGE_REGISTER)
        assert oracle.first_mismatch(pc.numpy(), want) == -1
        small = np.full(1000, -1.0, np.float32)
        st.add(ha[:1000].copy(), hb[:1000].copy(), small, mode=capi.STAGE_AUTO)
        assert st.last_mode == capi.STAGE_BOUNCE and oracle.first_mismatch(small, want[:1000].copy()) == -1
        # explicit release: the arrays are ordinary pageable memory again and can be re-registered
        st.release_host()
        hc.fill(-1.0)
        st.add(ha, hb, hc, mode=capi.STAGE_AUTO)
        assert st.last_mode == capi.STAGE_REGISTER and oracle.first_mismatch(hc, want) == -1
        # a new array overlapping a cached range (here: a window that starts inside ha and runs past its
        # registered sub-range) replaces the stale registration instead of failing
        st.release_host()
        st.add(ha[:n // 2], hb[:n // 2], hc[:n // 2], mode=capi.STAGE_REGISTER)
        st.add(ha, hb, hc, mode=capi.STAGE_REGISTER)
        assert oracle.first_mismatch(hc, want) == -1
    # the stager unregistered everything on destroy: registering by hand works again
    rt = torch.cuda.cudart()
    assert int(rt.cudaHostRegister(ha.ctypes.data, ha.nbytes, 0)) == 0
    assert int(rt.cudaHostUnregister(ha.ctypes.data)) == 0
    # pinned arrays through AUTO pick the lanes pipeline
    pa = torch.from_numpy(ha).pin_memory()
    pb = torch.from_numpy(hb).pin_memory()
    with va.Stager(0, 1 << 21, 3) as st:
        st.add(pa, pb, pc, mode=capi.STAGE_AUTO)
        assert st.last_mode == capi.STAGE_LANES and oracle.first_mismatch(pc.numpy(), want) == -1
        with pytest.raises(capi.B200VAError):
            st.add(pa, pb, pc, mode=9)


def test_device_entry_point_on_host_mapped_memory_large_enough_for_the_prefetch_form():
    """b200va_add_f32 on pinned host memory addressed directly by the GPU (UVA), at a size where AUTO
    resolves to the L2-prefetch form: the bulk prefetch is only a hint, the result must be the oracle's."""
    n = (1 << 25) + 77
    t = capi.resolve(capi.K_AUTO, n)
    assert t.early_loads == 2
    bufs = [va.PinnedBuffer(n) for _ in range(3)]
    try:
        ha, hb, hc = (b.array for b in bufs)
        ha[:] = oracle.fill_ctr(n, 0x0A, 5)
        hb[:] = oracle.fill_ctr(n, 0x0B, 5)
        hc[:] = -1.0
        stream = torch.cuda.current_stream().cuda_stream
        for _ in range(2):                                   # twice: the second launch prefetches while the first drains
            rc = capi.lib.b200va_add_f32(ha.ctypes.data, hb.ctypes.data, hc.ctypes.data, n, capi.K_AUTO, stream)
            assert rc == capi.OK, capi.strerror(rc)
        torch.cuda.synchronize()
        assert oracle.first_mismatch(np.array(hc), oracle.vadd(np.array(ha), np.array(hb))) == -1
        # the host rewrites an input between two launches: the second launch must see the new values
        ha[: 1 << 20] = 0.5
        rc = capi.lib.b200va_add_f32(ha.ctypes.data, hb.ctypes.data, hc.ctypes.data, n, capi.K_AUTO, stream)
        assert rc == capi.OK
        torch.cuda.synchronize()
        assert oracle.first_mismatch(np.array(hc), oracle.vadd(np.array(ha), np.array(hb))) == -1
    finally:
        for b in bufs:
            b.free()


def test_concurrent_callers_on_one_device():
    """The library is re-entrant: four host threads, each with its own stream and its own stager, call the
    device entry points and the host-buffer path at the same time on the same GPU (ctypes releases the GIL)."""
    import threading

    n = 3_000_001
    errors: list = []

    def worker(k: int):
        try:
            torch.cuda.set_device(0)
            ha, hb = oracle.fill_ctr(n, 0x0A, k * n), oracle.fill_ctr(n, 0x0B, k * n)
            want = oracle.vadd(ha, hb)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                a, b = torch.from_numpy(ha).cuda(), torch.from_numpy(hb).cuda()
                for i in range(25):
                    c = va.add(a, b, variant=("auto", "k2", "k3", "k1")[(i + k) % 4], inputs_stable=bool(i & 1))
                stream.synchronize()
                assert oracle.first_mismatch(c.cpu().numpy(), want) == -1
            hc = np.empty_like(ha)
            with va.Stager(0, 1 << 19, 2) as st:
                for mode in (capi.STAGE_BOUNCE, capi.STAGE_AUTO, capi.STAGE_AUTO):
                    hc.fill(-1.0)
                    st.add(ha, hb, hc, mode=mode)
                    assert oracle.first_mismatch(hc, want) == -1
        except BaseException as e:      # noqa: BLE001 -- reported to the main thread
            errors.append((k, repr(e)))

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_stager_restores_the_callers_current_device():
    """Entry points that take a `device` leave the calling thread on the device it was on (ADVICE r01)."""
    n = 1 << 20
    ha, hb = oracle.fill_ctr(n, 0x0A), oracle.fill_ctr(n, 0x0B)
    last = torch.cuda.device_count() - 1
    before = torch.cuda.current_device()
    for target in {0, last}:
        out = va.add_host(ha, hb, device=target)
        assert oracle.first_mismatch(out, oracle.vadd(ha, hb)) == -1
        with va.Stager(target, 1 << 18, 2) as st:
            hc = np.empty_like(ha)
            st.add(ha, hb, hc, mode=capi.STAGE_BOUNCE)
            assert oracle.first_mismatch(hc, oracle.vadd(ha, hb)) == -1
        assert torch.cuda.current_device() == before
        # and a device call right after lands on the caller's device, not on `target`
        x = torch.ones(1024, device=f"cuda:{before}")
        y = va.add(x, x)
        assert y.device.index == before and float(y.sum()) == 2048.0


def _fail_in_the_middle(mode: int) -> None:
    """A failure in the middle of the pipeline (injected right after chunk 1's H2D copies were
    queued) returns an error code only after every stream of the stager has drained: the caller
    may overwrite or free its arrays at once, and the stager works on the next call."""
    import os
    import subprocess
    import sys
    import textwrap

    from conftest import ROOT

    code = textwrap.dedent(f"""
        import numpy as np, torch, oracle
        from k8s_gpu_hpa_b200 import capi, vector_add as va
        mode, n = {mode}, 6 * (1 << 20) + 11
        ha = torch.from_numpy(oracle.fill_ctr(n, 0x0A)).pin_memory()
        hb = torch.from_numpy(oracle.fill_ctr(n, 0x0B)).pin_memory()
        hc = torch.full((n,), -1.0).pin_memory()
        want = oracle.vadd(ha.numpy(), hb.numpy())
        with va.Stager(0, 1 << 20, 3) as st:
            try:
                st.add(ha, hb, hc, mode=mode)
                raise SystemExit("the injected fault did not surface")
            except capi.B200VAError as e:
                assert e.code == capi.ERR_INVALID, e
            # drained: nothing of chunk 2.. was ever started, and chunk 0 completed (its D2H landed) -- in mode 3
            # its result would leave the bounce ring for C only two chunks later
            got = hc.numpy()
            if mode != capi.STAGE_BOUNCE:
                assert oracle.first_mismatch(got[:1 << 20].copy(), want[:1 << 20].copy()) == -1
            assert (got[2 << 20:] == -1.0).all()
            ha.zero_(); ha.copy_(torch.from_numpy(oracle.fill_ctr(n, 0x0A)))   # scribbling over A right away is safe
            st.add(ha, hb, hc, mode=mode)                                       # the hook fires once: this call is clean
            assert oracle.first_mismatch(hc.numpy(), want) == -1
        x = torch.ones(16, device="cuda")
        assert float(va.add(x, x).sum()) == 32.0                                 # no latched CUDA error either
        print("OK")
    """)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, B200VA_TEST_FAIL_CHUNK="1", PYTHONPATH=ROOT))
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout + p.stderr


def test_stager_error_in_the_middle_leaves_nothing_in_flight():
    _fail_in_the_middle(capi.STAGE_LANES)


@pytest.mark.parametrize("mode", [0, 3])      # slot streams, pageable bounce: the same chunk loop as the lanes
def test_stager_error_in_the_middle_of_the_slot_and_bounce_pipelines(mode):
    _fail_in_the_middle(mode)


def test_cli_zero_arguments_is_the_reference_process():
    """`./vectorAdd` exactly as cuda-test-deployment.yaml:19 runs it."""
    p = va.run_cli()
    assert p.returncode == 0, p.stderr
    lines = p.stdout.strip().splitlines()
    assert lines[0] == "[Vector addition of 50000 elements]"
    assert lines[1] == "Copy input data from the host memory to the CUDA device"
    assert lines[2].startswith("CUDA kernel launch with ") and lines[2].endswith(" threads")
    assert lines[3] == "Copy output data from the CUDA device to the host memory"
    assert lines[4] == "Test PASSED" and lines[5] == "Done"


def test_cli_bash_launch_loop_shape():
    """The Deployment's bash loop, shortened: every iteration a fresh process, exit status ignored."""
    import subprocess

    p = subprocess.run(["bash", "-c", "for (( c=1; c<=3; c++ )); do ./vectorAdd; done"],
                       cwd=capi._HERE, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.count("Test PASSED") == 3


@pytest.mark.parametrize("kernel", ["auto", "k0", "k1", "k2", "k3"])
def test_cli_sample_mode_options(kernel):
    p = va.run_cli("--n", "1000003", "--iters", "5", "--kernel", kernel)
    assert p.returncode == 0 and "Test PASSED" in p.stdout, p.stderr
    p = va.run_cli("--n", "2^20", "--gen", "ctr", "--iters", "12", "--graph", "4", "--kernel", kernel)
    assert p.returncode == 0 and "Test PASSED" in p.stdout, p.stderr


def test_cli_resident_mode_reports_oracle_digest():
    n = (1 << 24) + 40
    p = va.run_cli("--mode", "resident", "--n", str(n), "--iters", "20")
    assert p.returncode == 0, p.stderr
    r = json.loads(p.stdout.strip().splitlines()[-1])
    s, x = oracle.ctr_vadd_digest(n)
    assert r["mismatches"] == 0 and int(r["digest_sum"], 16) == s and int(r["digest_xor"], 16) == x
    assert r["launches_per_gpu"] == 20 and r["elements_per_s"] > 1e9


def test_cli_seed_changes_the_data_not_the_verdict():
    n = 1 << 20
    digests = set()
    for seed in ("0x0A", "77"):
        p = va.run_cli("--mode", "resident", "--n", str(n), "--iters", "3", "--seed", seed)
        assert p.returncode == 0, p.stderr
        r = json.loads(p.stdout.strip().splitlines()[-1])
        assert r["mismatches"] == 0
        digests.add(r["digest_sum"])
        if seed == "0x0A":
            assert int(r["digest_sum"], 16) == oracle.ctr_vadd_digest(n)[0]
    assert len(digests) == 2


def test_cli_verify_none_never_claims_a_pass():
    p = va.run_cli("--n", "4096", "--verify", "none")
    assert p.returncode == 0 and "Test PASSED" not in p.stdout and "Test SKIPPED" in p.stdout and "Done" in p.stdout


def test_cli_staged_mode_and_duty_cycle():
    p = va.run_cli("--mode", "staged", "--n", str((1 << 23) + 1), "--iters", "2")
    assert p.returncode == 0, p.stderr
    r = json.loads(p.stdout.strip().splitlines()[-1])
    assert r["mismatches"] == 0 and r["stage_mode"] == capi.STAGE_LANES and r["host_mem"].startswith("pinned")
    # the reference process's own kind of memory: malloc'd arrays, page-locked once by the stager
    p = va.run_cli("--mode", "staged", "--host-mem", "pageable", "--n", str((1 << 23) + 1), "--iters", "3")
    assert p.returncode == 0, p.stderr
    r = json.loads(p.stdout.strip().splitlines()[-1])
    assert r["mismatches"] == 0 and r["host_mem"].startswith("pageable")
    assert r["first_stage_mode"] == capi.STAGE_REGISTER      # pass 1 page-locked the malloc'd arrays ...
    assert r["stage_mode"] == capi.STAGE_LANES               # ... so the later passes see pinned memory
    assert r["first_pass_wall_ms"] > 0
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        prom = d + "/gpu.prom"
        p = va.run_cli("--n", "2^22", "--iters", "50", "--duration", "1.5", "--target-util", "30", "--metrics-file", prom)
        assert p.returncode == 0, p.stderr
        r = json.loads(p.stdout.strip().splitlines()[-1])
        assert r["mismatches"] == 0 and 0.2 < r["gpu_busy_frac"] < 0.4
        # the CLI's verdict is the HPA's: outside the 10 % tolerance band only
        assert r["hpa_would_scale"] == (r["nvml_util_mean"] > r["hpa_threshold"] * 1.1)
        from k8s_gpu_hpa_b200 import hpa_replay
        assert r["hpa_would_scale"] == hpa_replay.would_scale_up(r["nvml_util_mean"])
        text = open(prom).read()                       # the series the reference's recording rule reads
        assert "# TYPE dcgm_gpu_utilization gauge" in text
        sample = [l for l in text.splitlines() if l.startswith("dcgm_gpu_utilization{")][0]
        assert 'gpu="0"' in sample and "uuid=\"GPU-" in sample and 0 <= int(sample.rsplit(" ", 1)[1]) <= 100
        assert 'namespace="default"' in sample
    import os
    with tempfile.TemporaryDirectory() as d:
        prom = d + "/gpu.prom"
        import subprocess
        p = subprocess.run([capi.CLI_PATH, "--n", "2^20", "--iters", "20", "--duration", "0.8", "--metrics-file", prom],
                           capture_output=True, text=True, timeout=120, env=dict(os.environ, POD_NAMESPACE="gpu-demo"))
        assert p.returncode == 0, p.stderr
        assert 'namespace="gpu-demo"' in open(prom).read()


@pytest.mark.parametrize("gpus", [2, 4, 8])
def test_cli_shards_across_gpus(gpus):
    """BASELINE.json configs[2] shape on however many GPUs the box has: contiguous shards, no
    collective, digest identical to the unsharded oracle."""
    if torch.cuda.device_count() < gpus:
        pytest.skip(f"needs {gpus} GPUs")
    n = (1 << 26) + 12345
    p = va.run_cli("--gpus", str(gpus), "--n", str(n), "--iters", "10")
    assert p.returncode == 0, p.stderr
    r = json.loads(p.stdout.strip().splitlines()[-1])
    s, x = oracle.ctr_vadd_digest(n)
    assert r["gpus"] == gpus and r["mismatches"] == 0
    assert int(r["digest_sum"], 16) == s and int(r["digest_xor"], 16) == x
