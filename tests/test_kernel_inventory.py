"""The add and STREAM kernels each library carries, restated here and compared with its SASS (no GPU needed).

The production set is stated once per kernel family in the sources, by four predicates: carries_vec, carries_tma
and carries_tma_dyn (csrc/b200va_add.cu) and carries_stream (csrc/b200va_typed.cu); the tune library
(-DB200VA_TUNE_MATRIX) carries every combination the kernel pick can name.  This module states them again, as
sets of kernel names in Tune.kernel_name()'s form, and checks each library's SASS against them.  An edit to a
predicate therefore shows here as the kernels it adds or drops.

It also pins that every function of libb200va.so is the tune library's function of the same name, instruction for
instruction.  So a test that runs a kernel from the tune library has run the production kernel too.

test_gpu_tune_matrix.py runs every kernel listed here through its library and compares it with the oracle.
"""
import pytest

import sass
from k8s_gpu_hpa_b200 import capi

# tune.ld_hint / tune.st_hint (b200va_ptx.cuh)
LD_PLAIN, LD_NA, LD_CS, LD_NA_EF, LD_NC_NA, LD_NA_256 = range(6)
ST_PLAIN, ST_NA, ST_CS, ST_NA_EF = range(4)
OP_COPY, OP_SCALE, OP_ADD, OP_TRIAD = range(4)
LIBS = {"production": capi.LIB_PATH, "tune": capi.TUNE_LIB_PATH}

# The values each with_value level of the kernel picks can take.
VEC_WIDTHS, VEC_UNROLLS, VEC_EARLY, VEC_SCHED = (4, 8), (1, 2, 4, 8), (0, 1, 2), (0, 1)
STREAM_UNROLLS, STREAM_STORES = (1, 2, 4), (ST_PLAIN, ST_NA)
K4_UNROLLS = (4, 8, 16)


def carries_vec(lib, vw, unroll, ld, st, early, sched):
    if lib == "tune":
        return True
    if sched == 1:
        return vw == 4 and ld == LD_PLAIN and st == ST_NA and unroll in (2, 4)
    return unroll <= 4 and ld in (LD_PLAIN, LD_NA_EF) and st in (ST_PLAIN, ST_NA)


def carries_tma(lib, mode, hint, st):
    if mode == 1 and st != ST_PLAIN:
        return False
    return lib == "tune" or (not hint and (mode == 1 or st == ST_NA))


def carries_tma_dyn(lib, hint, st):
    return lib == "tune" or st in (ST_PLAIN, ST_NA)


def carries_stream(lib, op, unroll, st):
    return lib == "tune" or (unroll <= 2 and (st == ST_PLAIN or unroll == (1 if op in (OP_ADD, OP_TRIAD) else 2)))


def add_tunes(lib):
    """One tune per add kernel the library carries, in a fixed order.  Only the fields that pick the kernel are set:
    the geometry (threads, ctas_per_sm, stages, tile_bytes) is left for the caller to choose."""
    out = []
    for vw in VEC_WIDTHS:
        for u in VEC_UNROLLS:
            for ld in range(6):
                for st in range(4):
                    for e in VEC_EARLY:
                        for s in VEC_SCHED:
                            if carries_vec(lib, vw, u, ld, st, e, s):
                                out.append(capi.Tune(kind=capi.K1_VEC128 if vw == 4 else capi.K3_VEC256, unroll=u,
                                                     ld_hint=ld, st_hint=st, early_loads=e, scheduler=s))
    for mode in (0, 1):
        for hint in (0, 1):
            for st in range(4):
                if carries_tma(lib, mode, hint, st):
                    out.append(capi.Tune(kind=capi.K2_TMA, ld_hint=LD_NA_EF if hint else LD_PLAIN, st_hint=st,
                                         store_mode=mode))
    for hint in (0, 1):
        for st in range(4):
            if carries_tma_dyn(lib, hint, st):
                out.append(capi.Tune(kind=capi.K2_TMA, ld_hint=LD_NA_EF if hint else LD_PLAIN, st_hint=st, store_mode=2))
    out += [capi.Tune(kind=capi.K4_SCALAR_MLP, unroll=u) for u in K4_UNROLLS]
    out.append(capi.Tune(kind=capi.K0_SCALAR))
    return out


def add_kernels(lib):
    return {t.kernel_name() for t in add_tunes(lib)}


def stream_kernels(lib):
    """stream_vec<DT,OP,UNROLL,LD,ST> (loads are always plain) and stream_scalar<DT,OP>, which both libraries carry
    for every pair."""
    out = set()
    for dt in range(4):
        for op in range(4):
            out.add(f"stream_scalar<{dt},{op}>")
            for u in STREAM_UNROLLS:
                for st in STREAM_STORES:
                    if carries_stream(lib, op, u, st):
                        out.add(f"stream_vec<{dt},{op},{u},{LD_PLAIN},{st}>")
    return out


def sass_kernels(lib, prefix):
    return {sass.kernel_name(fn) for fn in sass.functions(LIBS[lib]) if sass.parse(fn)[0].startswith(prefix)}


@pytest.mark.parametrize("lib, n_add, n_stream", [("production", 88, 64), ("tune", 1174, 112)])
def test_the_restated_sets_are_the_kernels_in_the_sass(lib, n_add, n_stream):
    """Every vadd_* and stream_* function in the library's SASS, and nothing else, is in the restated set."""
    assert len(add_tunes(lib)) == len(add_kernels(lib)) == n_add
    assert len(stream_kernels(lib)) == n_stream
    for prefix, want in (("vadd_", add_kernels(lib)), ("stream_", stream_kernels(lib))):
        got = sass_kernels(lib, prefix)
        assert got == want, f"{lib} {prefix}*: in the SASS only {sorted(got - want)[:8]}, restated only {sorted(want - got)[:8]}"


def test_the_production_set_is_a_subset_of_the_tune_set():
    assert add_kernels("production") < add_kernels("tune")
    assert stream_kernels("production") < stream_kernels("tune")


def test_every_production_function_is_the_tune_librarys_function_of_the_same_name():
    """Instruction text equal line by line, addresses and encodings stripped: all 199 functions, the cast, dot and
    support kernels included."""
    prod, tune = sass.functions(capi.LIB_PATH), sass.functions(capi.TUNE_LIB_PATH)
    missing = sorted(set(prod) - set(tune))
    assert not missing, f"only in the production library: {missing[:8]}"
    for fn, body in prod.items():
        a, b = sass.instructions(body), sass.instructions(tune[fn])
        assert a, fn
        if a != b:
            i = next((k for k, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
            pa, pb = a[i] if i < len(a) else "<end>", b[i] if i < len(b) else "<end>"
            raise AssertionError(f"{sass.kernel_name(fn)} ({fn}) differs at instruction {i}: production {pa!r}, "
                                 f"tune {pb!r} ({len(a)} and {len(b)} instructions)")
