"""The SASS of the built libraries, for the tests that read it (no GPU needed).

The only place the tests run cuobjdump.  A full listing of a library takes seconds (the tune library's the most),
and dumping one function with `-fun` still reads the whole fatbinary, so each library is dumped once per session
and split into its functions here.
"""
import functools
import re
import subprocess

OPCODE = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")
# one instruction line: its address, the instruction text, its encoding word
INSTRUCTION = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*/\*\s*0x[0-9a-f]{16}\s*\*/\s*$", re.M)


@functools.lru_cache(maxsize=None)
def dump(path: str) -> str:
    """The whole `cuobjdump -sass` listing of a library."""
    return subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout


@functools.lru_cache(maxsize=None)
def functions(path: str) -> dict[str, str]:
    """Mangled name -> the function's SASS, split from dump(path).  Each name appears once."""
    parts = re.split(r"^\s*Function : (\S+)\s*$", dump(path), flags=re.M)
    out = {}
    for fn, body in zip(parts[1::2], parts[2::2]):
        assert fn not in out, fn
        out[fn] = body
    return out


def opcodes(body: str) -> list[str]:
    """The opcodes of a function's SASS in text order, predicates stripped."""
    return OPCODE.findall(body)


def instructions(body: str) -> list[str]:
    """The instruction text of a function's SASS in text order, without addresses and encodings."""
    return INSTRUCTION.findall(body)


def parse(mangled: str) -> tuple[str, list[int]]:
    """_ZN6b200va8vadd_vecILi4ELi1ELi0ELi1ELi1EEEv... -> ("vadd_vec", [4, 1, 0, 1, 1])."""
    m = re.match(r"_ZN6b200va(\d+)", mangled)
    assert m, mangled
    name = mangled[m.end():m.end() + int(m.group(1))]
    targs = re.match(r"I((?:L[a-z]\d+E)+)E", mangled[m.end() + len(name):])
    return name, [int(v) for v in re.findall(r"L[a-z](\d+)E", targs.group(1))] if targs else []


def kernel_name(mangled: str) -> str:
    """A kernel's name as a profiler trace gives it, in Tune.kernel_name()'s form: "vadd_vec<4,1,0,1,1>",
    "vadd_tma_dyn<1,0>" (bools as 0/1), "vadd_scalar"."""
    name, targs = parse(mangled)
    return f"{name}<{','.join(map(str, targs))}>" if targs else name


def ptx(path: str) -> str:
    """The `cuobjdump -lptx` listing of a library: the PTX files it embeds."""
    return subprocess.run(["cuobjdump", "-lptx", path], capture_output=True, text=True, check=True).stdout
