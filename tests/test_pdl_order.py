"""What every kernel of both libraries does before griddepcontrol.wait, read from the SASS (no GPU needed).

A kernel launched with programmatic stream serialization (PDL) may start while the launch before it on the stream
is still running; griddepcontrol.wait (SASS ACQBULK) is where it waits for that launch.  So, in text order, before
the first ACQBULK of each kernel:
- nothing stores to or atomically updates global memory;
- nothing loads global memory, except the early-load forms (EARLY = 1) of vadd_vec and vadd_vec_dyn, which load
  their first tile there on the caller's promise (B200VA_F_INPUTS_STABLE, or the launch loop);
- the trigger griddepcontrol.launch_dependents (SASS PREEXIT) does not come either: a kernel releases the launch
  after it only once it has waited itself, so the launch immediately before a kernel is the only one that can
  still be running beside it.
The kernels without ACQBULK are exactly the ones the library launches without the PDL attribute.
"""
import re

import pytest

import sass
from k8s_gpu_hpa_b200 import capi

# launched with <<<>>> (no PDL attribute): the K0 control, the mixed-phase stream op, the support kernels
NO_WAIT = {"vadd_scalar", "stream_scalar", "fill_ctr", "fill_ctr_vec", "verify_bits", "verify_bits_vec",
           "digest_bits", "digest_bits_vec", "reset_verify", "reset_digest"}
GLOBAL_WRITE = re.compile(r"(STG|ST\.E|ST\b|ATOMG|ATOM\b|ATOM\.|REDG|RED\b|RED\.|UBLKCP\.G\.S|UTMASTG|UTMAREDG)")
GLOBAL_READ = re.compile(r"(LDG|LD\.E|LD\b|UBLKCP\.S\.G|UTMALDG)")
# every other instruction that names memory must be one of these before the wait
ALLOWED = re.compile(r"(LDC|ULDC|PREEXIT|UBLKPF\.L2|CREATEPOLICY)\b")
MEMORY = re.compile(r"(LD|ST|ATOM|RED|UBLK|UTMA|SYNCS|SU|TLD|TEX|CCTL|PREEXIT|MEMBAR|FENCE)")


@pytest.fixture(scope="module", params=["production", "tune"])
def kernels(request):
    """Mangled name -> the kernel's opcodes in text order."""
    path = capi.LIB_PATH if request.param == "production" else capi.TUNE_LIB_PATH
    out = {fn: sass.opcodes(body) for fn, body in sass.functions(path).items()}
    for fn, ops in out.items():
        assert ops, fn
    return out


def _early_loads(name: str, targs: list[int]) -> bool:
    return name in ("vadd_vec", "vadd_vec_dyn") and targs[4] == 1


def test_kernels_without_a_wait_are_the_ones_launched_without_pdl(kernels):
    names = {sass.parse(fn)[0] for fn in kernels}
    assert {"vadd_vec", "vadd_vec_dyn", "vadd_tma", "vadd_tma_dyn", "vadd_scalar_unrolled", "stream_vec", "convert_vec",
            "dot_vec", "dot_scalar", "dot_final", "probe_read2", "probe_fill", "probe_copy"} <= names
    no_wait = {sass.parse(fn)[0] for fn, ops in kernels.items() if "ACQBULK" not in ops}
    assert no_wait == NO_WAIT
    for fn, ops in kernels.items():
        if sass.parse(fn)[0] in NO_WAIT:
            assert "ACQBULK" not in ops and "PREEXIT" not in ops, fn


def test_nothing_writes_global_memory_before_the_wait(kernels):
    """In text order before the first ACQBULK: no global store, atomic, reduction or bulk store in any kernel.
    One exception, read from the source: in vadd_vec_dyn<..., EARLY = 1> the loop's `ask_early` ticket request
    (one ATOMG and the STS that publishes it) sits in the loop body ahead of the first wait in text order, but
    `ask_early` is false until the CTA has waited, so the first pass skips it."""
    for fn, ops in kernels.items():
        if "ACQBULK" not in ops:
            continue
        name, targs = sass.parse(fn)
        before = ops[:ops.index("ACQBULK")]
        writes = [o for o in before if GLOBAL_WRITE.match(o)]
        if name == "vadd_vec_dyn" and targs[4] == 1:
            assert writes == ["ATOMG.E.ADD.STRONG.GPU"], (fn, writes)
        else:
            assert not writes, (fn, writes)


def test_only_the_early_load_forms_load_before_the_wait(kernels):
    """Before the first ACQBULK: global loads in exactly the EARLY = 1 forms of vadd_vec and vadd_vec_dyn (every
    one of them), and otherwise only constant loads, the L2 bulk prefetch, createpolicy and (in the TMA ring of
    vadd_tma and vadd_tma_dyn) the mbarrier set-up in shared memory with its CTA-scope fences."""
    early = 0
    for fn, ops in kernels.items():
        if "ACQBULK" not in ops:
            continue
        name, targs = sass.parse(fn)
        before = ops[:ops.index("ACQBULK")]
        loads = [o for o in before if GLOBAL_READ.match(o)]
        if _early_loads(name, targs):
            early += 1
            assert loads and all(o.startswith("LDG.E") for o in loads), (fn, loads)
            rest = [o for o in before if MEMORY.match(o) and not GLOBAL_READ.match(o) and not ALLOWED.match(o)]
            if name == "vadd_vec_dyn":
                rest = [o for o in rest if o not in ("ATOMG.E.ADD.STRONG.GPU", "STS")]   # the ticket request above
            assert not rest, (fn, rest)
            continue
        assert not loads, (fn, loads)
        rest = [o for o in before if MEMORY.match(o) and not ALLOWED.match(o)]
        if name in ("vadd_tma", "vadd_tma_dyn"):
            rest = [o for o in rest if not re.match(r"SYNCS|FENCE\.VIEW\.ASYNC\.S|MEMBAR\.ALL\.CTA", o)]
        assert not rest, (fn, rest)
    assert early in (26, 384), early   # the EARLY = 1 vec kernels: 26 in the production library, 384 in the tune library


def test_each_kernel_releases_its_successor_only_after_its_own_wait(kernels):
    """PREEXIT (griddepcontrol.launch_dependents) never precedes the first ACQBULK: launch N + 1 is scheduled only
    once every CTA of launch N has waited for launch N - 1, so an early-load launch overlaps at most the launch
    immediately before it -- what B200VA_F_INPUTS_STABLE promises about, and, in the launch loop, the same add."""
    for fn, ops in kernels.items():
        if "ACQBULK" not in ops:
            continue
        assert "PREEXIT" in ops, fn
        assert ops.index("PREEXIT") > ops.index("ACQBULK"), fn
