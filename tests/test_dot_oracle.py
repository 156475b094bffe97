"""CPU checks of oracle/dot_exact.py, the reference of b200va_dot, and of the constants the library exports.

- The vectorised reference equals a plain scalar restatement of the three rules (below, written separately with a
  per-element Fraction fma and a recursive tree) at n around every lane and chunk edge, for all four types.
- It lies within the a-priori error bound of the exact sum; the exactly representable family gives the exact sum.
- The adversarial sets separate the contract from plausible wrong kernels, each implemented here in numpy: other
  lane counts and chunk sizes, a sequential sum, an f32 accumulator, mul+add instead of fma for f64, a chunk edge
  or head peel off by one, and FTZ.
- The SASS of the dot kernels keeps the programmatic-dependency discipline: nothing but the L2 prefetch and the
  trigger before griddepcontrol.wait.
"""
import math
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle import dot_exact as D
from oracle import stream_exact as X

import k8s_gpu_hpa_b200 as pkg
from k8s_gpu_hpa_b200 import capi

DTS = ["f32", "f64", "f16", "bf16"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------- scalar restatement
def fma_fraction(x: float, y: float, acc: float) -> float:
    if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(acc)):
        return x * y + acc
    return float(Fraction(x) * Fraction(y) + Fraction(acc))


def dyadic(v: list) -> float:
    """Aligned dyadic tree of v: a block's value is the sum of its halves; an empty upper half passes the lower."""
    if not v:
        return 0.0
    if len(v) == 1:
        return v[0]
    half = 1 << ((len(v) - 1).bit_length() - 1)
    lo, hi = dyadic(v[:half]), v[half:]
    return lo + dyadic(hi) if hi else lo


def restated(a, b, dtype) -> float:
    x, y = X.widen(a, dtype).tolist(), X.widen(b, dtype).tolist()
    n, values = len(x), []
    for k0 in range(0, n, D.CHUNK):
        lanes = []
        for lane in range(D.LANES):
            acc = 0.0
            for i in range(k0 + lane, min(n, k0 + D.CHUNK), D.LANES):
                acc = fma_fraction(x[i], y[i], acc)
            lanes.append(acc)
        values.append(dyadic(lanes))
    return dyadic(values)


def same_bits(x: float, y: float) -> bool:
    return (math.isnan(x) and math.isnan(y)) or np.float64(x).view(np.uint64) == np.float64(y).view(np.uint64)


EDGES = [0, 1, D.LANES - 1, D.LANES + 1, D.CHUNK - 1, D.CHUNK + 1, 3 * D.CHUNK + 5]


@pytest.mark.parametrize("dtype", DTS)
def test_vectorised_reference_equals_the_scalar_restatement(dtype):
    rng = np.random.default_rng(list(X.BITS).index(dtype))
    a, b = D.cancellation(dtype, max(EDGES), seed=3)
    a2, b2 = X.finite(dtype, max(EDGES), rng), X.finite(dtype, max(EDGES), rng)
    for n in EDGES:
        for name, (x, y) in (("cancellation", (a, b)), ("normal", (a2, b2))):
            got, want = D.dot(x[:n], y[:n], dtype), restated(x[:n], y[:n], dtype)
            assert same_bits(got, want), (dtype, n, name, got, want)
            assert not (got == 0 and math.copysign(1, got) < 0)


@pytest.mark.parametrize("dtype", DTS)
def test_reference_is_within_the_error_bound_of_the_exact_sum(dtype):
    rng = np.random.default_rng(41)
    for n in (1, D.LANES + 1, 2 * D.CHUNK + 9):
        for x, y in ((X.finite(dtype, n, rng), X.finite(dtype, n, rng)), D.cancellation(dtype, n, seed=n)):
            err = abs(Fraction(D.dot(x, y, dtype)) - D.exact_sum(x, y, dtype))
            assert err <= D.error_bound(x, y, dtype), (dtype, n)


@pytest.mark.parametrize("dtype", DTS)
def test_exact_family_gives_the_exact_sum(dtype):
    for n in (0, 1, 5, D.CHUNK + 3, 3 * D.CHUNK + 5):
        a, b = D.family(dtype, n, seed=n)
        want = D.exact_sum(a, b, dtype)
        assert D.family_sum(a, b, dtype) == want
        if dtype != "f64" or n <= X.FRACTION_LIMIT:
            assert Fraction(D.dot(a, b, dtype)) == want
    a, b = D.family(dtype, 1001, seed=9)            # repeated to n: q whole periods and a prefix
    n = 5 * 1001 + 17
    assert D.family_sum(a, b, dtype, n) == D.exact_sum(np.resize(a, n), np.resize(b, n), dtype)


# ------------------------------------------------------------------------------------------- wrong kernels
def wrong(a, b, dtype, lanes=D.LANES, chunk=D.CHUNK, edge=0, head_peel=False, seq=False, acc32=False, muladd=False,
          ftz=False):
    """A dot product computed with one of the listed mistakes (everything else as the contract)."""
    x, y = X.widen(a, dtype), X.widen(b, dtype)
    if ftz:
        tiny = float(np.finfo(np.float16 if dtype == "f16" else np.float32).tiny)   # subnormals of the operand type
        x, y = (np.where(np.abs(v) < tiny, 0.0, v) for v in (x, y))
    n = x.size
    exact_products = dtype != "f64" or muladd
    with np.errstate(all="ignore"):
        p = x * y
        if seq:
            return float(np.cumsum(p)[-1]) if n else 0.0
        bounds = [0] + [k * chunk - edge for k in range(1, -(-n // chunk) + 1) if k * chunk - edge < n] + [n]
        first = 1 if head_peel else 0
        ft = np.float32 if acc32 else np.float64
        values = []
        for s, e in zip(bounds[:-1], bounds[1:]):
            s = max(s, first)
            m = e - s
            rows = -(-m // lanes)
            if exact_products:
                q = np.concatenate([p[s:e], np.zeros(rows * lanes - m)]).reshape(rows, lanes)
                acc = np.zeros(lanes, ft)
                for r in range(rows):
                    acc = (acc.astype(np.float64) + q[r]).astype(ft)
            else:
                acc = np.zeros(lanes)
                for lane in range(lanes):
                    v = 0.0
                    for i in range(s + lane, e, lanes):
                        v = fma_fraction(float(x[i]), float(y[i]), v)
                    acc[lane] = v
            values.append(D.tree(acc.astype(ft)) if not acc32 else _tree32(acc))
        total = float(D.tree(np.array(values, np.float64))) if not acc32 else float(_tree32(np.array(values, np.float32)))
        return total + float(p[0]) if head_peel and n else total


def _tree32(x):
    x = np.asarray(x, np.float32)
    width = 1 << max(0, (x.size - 1).bit_length())
    x = np.concatenate([x, np.zeros(width - x.size, np.float32)])
    while x.size > 1:
        x = x[0::2] + x[1::2]
    return x[0]


VARIANTS = {
    "1024 lanes": dict(lanes=1024), "4096 lanes": dict(lanes=4096),
    "chunk 2^15": dict(chunk=1 << 15), "chunk 2^17": dict(chunk=1 << 17),
    "sequential sum": dict(seq=True), "chunk edge off by one": dict(edge=1), "head peel off by one": dict(head_peel=True),
}


@pytest.mark.parametrize("dtype", DTS)
def test_adversarial_sets_separate_the_contract_from_wrong_kernels(dtype):
    """Every wrong kernel gives other bits on at least one cancellation set, and the chunk-edge mistake on the set
    built for it; FTZ on the subnormal set; the special-value sets give the expected class of result."""
    sets = {name: (a, b) for name, a, b in D.adversarial(dtype)}
    cancel = {name: (a, b, D.dot(a, b, dtype)) for name, (a, b) in sets.items() if name.startswith("cancellation")}
    assert len(cancel) == 5 and all(math.isfinite(w) for _, _, w in cancel.values())
    variants = dict(VARIANTS)
    if dtype == "f32":
        variants["f32 accumulator"] = dict(acc32=True)
    if dtype == "f64":
        variants["mul+add instead of fma"] = dict(muladd=True)
    for name, kw in variants.items():
        separated = [s for s, (a, b, w) in cancel.items() if not same_bits(wrong(a, b, dtype, **kw), w)]
        assert separated, f"{dtype}: no cancellation set separates '{name}' from the contract"
        if kw.get("edge"):
            assert "cancellation: edge" in separated, (dtype, name, separated)
    # subnormal operands: flushing them to zero changes the sum
    a, b = sets["subnormals"]
    want = D.dot(a, b, dtype)
    assert want != 0 and Fraction(want) != 0
    if dtype != "f64":
        assert not same_bits(wrong(a, b, dtype, ftz=True), want), f"{dtype}: FTZ gives the contract's bits"
    # special values: the class of the result is known
    expect = {"+inf": math.inf, "-inf": -math.inf}
    for name, x, y in D.specials(dtype):
        got = D.dot(x, y, dtype)
        if name in expect:
            assert got == expect[name], (dtype, name, got)
        else:
            assert math.isnan(got), (dtype, name, got)


def test_subnormal_products_are_kept_where_ftz_would_flush_them():
    """f32 subnormal operands times ordinary ones, f16 subnormals: the exact sums are nonzero."""
    for dtype in ("f32", "f16", "bf16"):
        a, b = D.subnormals(dtype, 4096)
        assert (X.widen(a, dtype) != 0).all() and abs(X.widen(a, dtype)).max() < np.finfo(np.float32 if dtype != "f16" else np.float16).tiny
        assert Fraction(D.dot(a, b, dtype)) - D.exact_sum(a, b, dtype) <= D.error_bound(a, b, dtype)


# ------------------------------------------------------------------------------------------- the library's constants
def test_constants_and_workspace_size_match_the_header():
    text = open(os.path.join(ROOT, "include", "b200va.h")).read()
    assert int(re.search(r"#define B200VA_DOT_LANES\s+(\d+)", text).group(1)) == capi.DOT_LANES == D.LANES
    assert int(re.search(r"#define B200VA_DOT_CHUNK\s+(\d+)", text).group(1)) == capi.DOT_CHUNK == D.CHUNK
    ws = capi.lib.b200va_dot_workspace_bytes
    for n in (0, 1, D.CHUNK - 1, D.CHUNK, D.CHUNK + 1, 3 * D.CHUNK + 5, (1 << 32) + 4099, 1 << 40):
        assert ws(n) == 8 * -(-n // D.CHUNK), n
    assert ws(1 << 40) == 8 << 24
    assert ws(2 ** 64 - 1) == 8 * -(-(2 ** 64 - 1) // D.CHUNK)          # no wrap-around in the rounding up


def _sass(fn: str) -> list[str]:
    out = subprocess.run(["cuobjdump", "-sass", "-fun", fn, capi.LIB_PATH], capture_output=True, text=True).stdout
    return re.findall(r"\b(LDG\.E\S*|LDS\S*|STG\.E\S*|ACQBULK|UBLKPF\.L2|PREEXIT)\b", out)


def test_dot_kernels_load_nothing_and_release_nothing_before_the_dependency_wait():
    """Before griddepcontrol.wait (ACQBULK) only the two L2 prefetches of the HBM class; the trigger (PREEXIT) and
    every global load and store after it."""
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    names = sorted(set(re.findall(r"Function : (_ZN6b200va\d+dot_\w+)", sass)))
    assert len(names) == 9, names                    # dot_vec and dot_scalar per type, dot_final
    for fn in names:
        ops = _sass(fn)
        assert "ACQBULK" in ops, fn
        before = ops[:ops.index("ACQBULK")]
        want = [] if "dot_final" in fn else ["UBLKPF.L2", "UBLKPF.L2"]
        assert before == want, (fn, before)
        assert "PREEXIT" in ops[ops.index("ACQBULK"):], fn
        assert any(o.startswith("LDG") for o in ops[ops.index("ACQBULK"):]), fn
    vec = [fn for fn in names if "dot_vec" in fn]
    assert len(vec) == 4 and all(any(o.startswith("LDG.E.128") for o in _sass(fn)) for fn in vec)
