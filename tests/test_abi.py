"""No-GPU checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/b200va.h declares, its host-side entry points (a2 input recipes, a6 verify, shard
arithmetic) agree with the oracle, and -- without a GPU -- every compute entry point and
the executable fail loudly instead of falling back to a CPU path."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import k8s_gpu_hpa_b200 as pkg
import oracle
from conftest import ROOT, has_gpu
from k8s_gpu_hpa_b200 import capi, vector_add as va


def header_symbols():
    text = open(capi.HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200va_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(capi.lib, s), f"{s} declared in include/b200va.h but not exported"
    assert set(syms) == set(capi.EXPORTED), "ctypes binding and header disagree"
    for path in (capi.LIB_PATH, capi.TUNE_LIB_PATH):          # the tune library is the same ABI, more geometries
        out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
        exported = set(re.findall(r" T (b200va_\w+)", out))
        assert exported == set(syms), (path, exported ^ set(syms))
    assert capi.tune_lib().b200va_abi_version() == pkg.abi_version()


def test_struct_layouts_match_the_header():
    """ctypes mirrors of the two structs: field order and count as declared in include/b200va.h."""
    text = re.sub(r"/\*.*?\*/", "", open(capi.HEADER_PATH).read(), flags=re.S)
    body = re.search(r"typedef struct b200va_tune \{(.*?)\} b200va_tune_t;", text, flags=re.S).group(1)
    fields = re.findall(r"int\s+(\w+)\s*;", body)
    assert fields == [n for n, _ in capi.Tune._fields_]
    assert C.sizeof(capi.Tune) == 4 * len(fields) == 44


def test_abi_version_and_strerror():
    assert pkg.abi_version() == 2
    assert pkg.strerror(0) == "success"
    for code in (-1, -2, -3, -4, -5, -6, -7):
        assert pkg.strerror(code) not in ("success", "unknown error")
    assert "memory" in pkg.strerror(-1002).lower()          # cudaErrorMemoryAllocation


def test_library_is_sm90a_only_and_uses_tma_and_the_ticket_scheduler():
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, archs
    assert "UBLKCP" in sass            # cp.async.bulk (TMA)
    assert "SYNCS" in sass             # mbarrier
    assert "ATOMG.E.ADD" in sass       # the dynamic tile scheduler's ticket counter (K2d, K1d)
    assert "ACQBULK" in sass and "PREEXIT" in sass           # griddepcontrol.wait / launch_dependents (PDL)
    assert not re.search(r"[LS][DT]G\.E\S*\.256", sass)     # sm_90 has no 256-bit global access
    assert re.search(r"LDG\.E\S*\.128", sass) and re.search(r"STG\.E\S*\.128", sass)
    assert "HMMA" not in sass and "GMMA" not in sass         # a stream, not a contraction
    # "fat binary + PTX" (SURVEY.md 8(f)2): the production library also embeds its compute_90a PTX
    ptx = subprocess.run(["cuobjdump", "-lptx", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a.ptx" in ptx, ptx
    # the production library carries the production set, the tune library the whole matrix
    n_prod = sass.count("Function :")
    n_tune = subprocess.run(["cuobjdump", "-sass", capi.TUNE_LIB_PATH], capture_output=True, text=True).stdout.count("Function :")
    assert n_prod < 200 < n_tune, (n_prod, n_tune)


def test_early_load_variant_issues_its_loads_before_the_dependency_wait():
    """SASS of the EARLY kernel: both LDG.E.128 come before the first ACQBULK (griddepcontrol.wait)
    and the store after it; the plain kernel waits first."""
    def body(early: int) -> list[str]:
        fn = f"_ZN6b200va8vadd_vecILi4ELi1ELi0ELi1ELi{early}EEEvPKfS2_Pfmmmm"
        out = subprocess.run(["cuobjdump", "-sass", "-fun", fn, capi.LIB_PATH], capture_output=True, text=True).stdout
        return re.findall(r"\b(LDG\.E\.128|STG\.E\S*\.128|ACQBULK|UBLKPF\.L2)\b", out)
    early, plain, prefetch = body(1), body(0), body(2)
    assert early and plain and prefetch
    assert early.index("ACQBULK") > [i for i, m in enumerate(early) if m.startswith("LDG")][1]
    assert early.index("ACQBULK") < [i for i, m in enumerate(early) if m.startswith("STG")][0]
    assert plain[0] == "ACQBULK"
    # the always-legal form: two bulk L2 prefetches (A tile, B tile) ahead of the wait, loads and stores after it
    assert prefetch[:3] == ["UBLKPF.L2", "UBLKPF.L2", "ACQBULK"] and "LDG.E.128" in prefetch[3:]


def test_host_rand_recipe_matches_oracle_and_known_answers():
    a, b = va.fill_rand_host(50000)
    oa, ob = oracle.fill_rand(50000)
    assert np.array_equal(a, oa) and np.array_equal(b, ob)
    assert oracle.fnv1a64(a) == 0x1CDB0A2BFB6AA671 and oracle.fnv1a64(b) == 0xA798316A39E5FF4E


@pytest.mark.parametrize("n,seed,first", [(0, 1, 0), (1, 0x0A, 0), (100_003, 0x0A, 0), (4097, 0x0B, 1 << 33)])
def test_host_ctr_generator_matches_oracle(n, seed, first):
    assert np.array_equal(va.fill_ctr_host(n, seed, first), oracle.fill_ctr(n, seed, first))


def test_host_verify_is_bitwise_and_nan_tolerant():
    a, b = oracle.fill_rand(5000)
    c = oracle.vadd(a, b)
    assert va.verify_host(a, b, c) == -1
    c2 = c.copy()
    c2.view(np.uint32)[1234] ^= 1                            # one ulp: inside the sample's 1e-5, caught here
    assert oracle.verify_sample_tolerance(a, b, c2) == -1
    assert va.verify_host(a, b, c2) == 1234
    a[7] = np.nan
    c3 = oracle.vadd(a, b)
    c3.view(np.uint32)[7] = 0x7FFFFFFF
    assert va.verify_host(a, b, c3) == -1


@pytest.mark.parametrize("n,world", [(1 << 28, 1), (1 << 30, 8), (1 << 28, 2), (50000, 8), (7, 8), (0, 4), (1000003, 3)])
def test_shard_ranges_tile_the_index_space(n, world):
    prev = 0
    for r in range(world):
        b, e = pkg.shard_range(n, world, r)
        assert b == prev and b <= e <= n
        assert b % 8 == 0 or b == n                          # shard starts stay 32-byte aligned
        prev = e
    assert prev == n
    if n in (1 << 28, 1 << 30):
        assert pkg.shard_range(n, world, 0)[1] == n // world  # BASELINE sizes: equal powers of two
    assert capi.lib.b200va_shard_range(n, world, world, C.byref(C.c_size_t()), C.byref(C.c_size_t())) == capi.ERR_INVALID


def test_kernel_names_key_the_ncu_table():
    """Tune.kernel_name() is the key under which a per-kernel profile is filed and the name bench.py
    reports for the kernel it timed: it must name what the resolved geometry launches."""
    assert pkg.resolve(capi.K_AUTO, 1 << 28).kernel_name() == "vadd_vec<4,1,0,1,2>"                         # L2 prefetch ahead of the wait
    assert pkg.resolve(capi.K_AUTO, 1 << 28, capi.F_INPUTS_STABLE).kernel_name() == "vadd_vec<4,1,0,1,1>"
    assert pkg.resolve(capi.K_AUTO, 1 << 24, capi.F_COLD).kernel_name() == "vadd_vec<4,1,0,0,2>"           # cold-tuned class
    assert pkg.resolve(capi.K_AUTO, 1 << 22, capi.F_COLD | capi.F_INPUTS_STABLE).kernel_name() == "vadd_vec<4,2,0,0,2>"
    assert pkg.resolve(capi.K_AUTO, 1 << 21, capi.F_COLD | capi.F_INPUTS_STABLE).kernel_name() == "vadd_vec<4,4,0,0,1>"
    with pytest.raises(pkg.B200VAError):
        pkg.resolve(capi.K_AUTO, 1 << 20, 0x40)
    assert pkg.resolve(capi.K_AUTO, 1 << 24).kernel_name() == "vadd_vec<4,2,3,0,0>"
    assert pkg.resolve(capi.K2_TMA, 1 << 28).kernel_name() == "vadd_tma_dyn<0,1>"
    assert pkg.resolve(capi.K3_VEC256, 1 << 28).kernel_name() == "vadd_vec<8,1,0,1,0>"
    assert pkg.resolve(capi.K0_SCALAR, 50000).kernel_name() == "vadd_scalar"
    assert capi.Tune(kind=capi.K1_VEC128, threads=256, unroll=2, st_hint=1, scheduler=1).kernel_name() == "vadd_vec_dyn<4,2,0,1,0>"


def test_numa_node_of_a_device_is_minus_one_without_a_gpu_or_a_small_int():
    assert -1 <= capi.lib.b200va_device_numa_node_of(0) < 64


def test_resolve_geometry():
    for v in pkg.VARIANTS.values():
        t = pkg.resolve(v, 1 << 28)
        assert t.kind in (capi.K0_SCALAR, capi.K1_VEC128, capi.K2_TMA, capi.K3_VEC256)
    assert pkg.resolve(capi.K0_SCALAR, 50000).threads == 256   # the sample's launch shape (a5)
    with pytest.raises(pkg.B200VAError):
        pkg.resolve(99, 10)


@pytest.mark.skipif(has_gpu(), reason="checks the no-GPU failure mode")
def test_compute_entry_points_fail_loudly_without_a_gpu():
    a = np.ones(16, np.float32)
    # device entry points: error code, never a silent CPU result
    rc = capi.lib.b200va_add_f32(a.ctypes.data, a.ctypes.data, a.ctypes.data, 16, 0, None)
    assert rc != capi.OK
    assert capi.lib.b200va_add_f32_ex(a.ctypes.data, a.ctypes.data, a.ctypes.data, 16, 0, capi.F_INPUTS_STABLE, None) != capi.OK
    out = np.full(16, -7.0, np.float32)
    with pytest.raises(pkg.B200VAError):
        va.add_host(a, a, out)
    assert (out == -7.0).all()
    with pytest.raises(pkg.B200VAError):
        pkg.query(0)
    with pytest.raises(pkg.B200VAError):
        va.Stager(0)


@pytest.mark.skipif(has_gpu(), reason="checks the no-GPU failure mode")
def test_cli_fails_loudly_without_a_gpu():
    p = va.run_cli()
    assert p.returncode == 1 and "Failed to" in p.stderr and "Test PASSED" not in p.stdout
    p = va.run_cli("--n", "1024", "--gpus", "2", "--iters", "3")
    assert p.returncode == 1 and "Failed to" in p.stderr


def test_cli_rejects_bad_options():
    assert va.run_cli("--bogus").returncode == 1
    assert va.run_cli("--host-mem", "floppy").returncode == 1
    assert va.run_cli("--mode", "sample", "--gpus", "2").returncode == 1
    assert va.run_cli("--help").returncode == 0


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing under the package, the header or the
    executable sources may import, include or link it."""
    pkg_dir = os.path.join(ROOT, "k8s-gpu-hpa_b200")
    for dirpath, _, files in os.walk(pkg_dir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")) or f == "Makefile":
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"(^|\n)\s*(import|from)\s+oracle\b", text), f
                assert "liboracle" not in text and "vadd_oracle" not in text, f
    ldd = subprocess.run(["ldd", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in ldd
