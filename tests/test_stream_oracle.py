"""Row f4 oracle pinned: the integer half/bfloat16 conversions against numpy/torch over
every 16-bit pattern and adversarial fp32 inputs, and the op semantics against numpy."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle
from oracle import stream_exact as X


def test_half_conversions_match_numpy_exhaustively():
    h = np.arange(65536, dtype=np.uint16)
    fn = h.view(np.float16).astype(np.float32)
    assert oracle.first_mismatch(oracle.half_to_float(h), fn) == -1
    rng = np.random.default_rng(7)
    x = rng.integers(0, 1 << 32, 1_000_000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    finite = fn[np.isfinite(fn)]
    x = np.concatenate([x, fn, np.nextafter(finite, np.float32(np.inf)), np.nextafter(finite, np.float32(-np.inf)),
                        (finite.astype(np.float64) * (1 + 2.0 ** -11)).astype(np.float32),      # exact ties
                        np.array([65504.0, 65519.996, 65520.0, 6e-8, 2.98e-8, 2.9802322e-8, 0.0, -0.0], np.float32)])
    with np.errstate(all="ignore"):
        want = x.astype(np.float16).view(np.uint16)
    assert oracle.first_mismatch_bits(oracle.float_to_half(x), want, "f16") == -1


def test_bf16_conversions_match_torch():
    h = np.arange(65536, dtype=np.uint16)
    want = torch.from_numpy(h.view(np.int16).copy()).view(torch.bfloat16).float().numpy()
    assert oracle.first_mismatch(oracle.bf16_to_float(h), want) == -1
    rng = np.random.default_rng(8)
    x = rng.integers(0, 1 << 32, 1_000_000, dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([x, (h.astype(np.uint32) << 16) | 0x8000, (h.astype(np.uint32) << 16) | 0x7FFF,
                        (h.astype(np.uint32) << 16) | 0x8001]).view(np.float32)
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert oracle.first_mismatch_bits(oracle.float_to_bf16(x), want, "bf16") == -1


@pytest.mark.parametrize("dtype,npdt", [("f32", np.float32), ("f64", np.float64)])
def test_native_ops_match_numpy(dtype, npdt):
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal(10_001).astype(npdt), rng.standard_normal(10_001).astype(npdt)
    s = 3.0
    assert np.array_equal(oracle.stream("copy", dtype, a, None), a)
    assert np.array_equal(oracle.stream("scale", dtype, a, None, s), npdt(s) * a)
    assert np.array_equal(oracle.stream("add", dtype, a, b), a + b)
    # triad is a single fused rounding: compare with the exact result rounded once
    wide = np.longdouble if npdt is np.float64 else np.float64
    want = (a.astype(wide) + wide(s) * b.astype(wide)).astype(npdt)
    assert np.array_equal(oracle.stream("triad", dtype, a, b, s), want)


def test_f32_add_is_the_vectoradd_oracle():
    a, b = oracle.fill_rand(50000)
    assert np.array_equal(oracle.stream("add", "f32", a, b), oracle.vadd(a, b))


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_half_ops_widen_compute_round(dtype):
    rng = np.random.default_rng(4)
    to_f = oracle.half_to_float if dtype == "f16" else oracle.bf16_to_float
    to_h = oracle.float_to_half if dtype == "f16" else oracle.float_to_bf16
    a = rng.integers(0, 1 << 16, 50_000, dtype=np.uint32).astype(np.uint16)
    b = rng.integers(0, 1 << 16, 50_000, dtype=np.uint32).astype(np.uint16)
    fa, fb = to_f(a), to_f(b)
    with np.errstate(all="ignore"):
        assert oracle.first_mismatch_bits(oracle.stream("add", dtype, a, b), to_h(fa + fb), dtype) == -1
        assert oracle.first_mismatch_bits(oracle.stream("scale", dtype, a, None, 0.3), to_h(np.float32(0.3) * fa), dtype) == -1
    assert np.array_equal(oracle.stream("copy", dtype, a, None), a)
    # fp16 add computed through fp32 equals numpy's correctly rounded fp16 add (p' >= 2p+2)
    if dtype == "f16":
        with np.errstate(all="ignore"):
            want = (a.view(np.float16) + b.view(np.float16)).view(np.uint16)
        assert oracle.first_mismatch_bits(oracle.stream("add", dtype, a, b), want, dtype) == -1


# ---------------------------------------------------------------- the exact reference (oracle/stream_exact.py)
ALL_DTYPES = ["f32", "f64", "f16", "bf16"]
ALL_OPS = ["copy", "scale", "add", "triad"]
# exact in a few bits or not, a double tie and the double just above it, f32 overflow, f32 subnormal, f32 zero
SCALARS = [0.7001953125, 0.1, 1 / 3, 1 + 2.0 ** -24, 1 + 2.0 ** -24 + 2.0 ** -52, 3.5e38, 1e-45, 1e-50, -0.0,
           float("inf"), float("-inf"), float("nan")]


def random_bits(dtype, n, seed):
    ut = X.BITS[dtype][0]
    rng = np.random.default_rng(seed)
    return rng.integers(0, np.iinfo(ut).max, n, dtype=np.uint64, endpoint=True).astype(ut).view(X.STORAGE[dtype])


def assert_same(got, want, dtype, what, nan_class=True):
    if nan_class:
        bad = oracle.first_mismatch_bits(got, want, dtype)
    else:
        ut = X.BITS[dtype][0]
        idx = np.nonzero(np.ascontiguousarray(got).view(ut) != np.ascontiguousarray(want).view(ut))[0]
        bad = int(idx[0]) if idx.size else -1
    assert bad < 0, f"{what}: first mismatch at {bad}"


@pytest.mark.parametrize("dtype", ALL_DTYPES)
@pytest.mark.parametrize("op", ALL_OPS)
def test_exact_reference_matches_the_c_oracle(op, dtype):
    """Random bit patterns (every class: subnormals, inf, NaN) at every scalar, and the adversarial sets.  NaN
    matches NaN as a class, except for COPY, which keeps the bits."""
    n = 20_000 if dtype == "f64" else 200_000
    a, b = random_bits(dtype, n, 21), random_bits(dtype, n, 22)
    cases = [("random", s, a, b) for s in (SCALARS if op in ("scale", "triad") else [0.0])]
    cases += X.adversarial(op, dtype)
    binary = op in ("add", "triad")
    for name, s, a, b in cases:
        with np.errstate(all="ignore"):
            want = oracle.stream(op, dtype, a, b if binary else None, s)
        assert_same(X.stream(op, dtype, a, b if binary else None, s), want, dtype, f"{name} s={s!r}", op != "copy")


def exact_rounded_once(op, dtype, a, b, s):
    """The contract through Fraction, one finite element at a time: the exact result rounded once to f32 (f64: to
    f64), then (f16/bf16) narrowed.  An exact zero takes its sign from IEEE arithmetic on the zero operands."""
    sc = s if dtype == "f64" else X.f32_scalar(s)
    if op == "add":
        sc = 1.0
    out = []
    for x, y in zip(X.widen(a, dtype).tolist(), X.widen(b, dtype).tolist()):
        if op == "scale":
            x, y = -0.0, x                           # s*a == -0 + s*a, signed zeros included
        e = Fraction(x) + Fraction(sc) * Fraction(y)
        out.append(X.round_fraction(e, "f64" if dtype == "f64" else "f32") if e != 0 else
                   sc * y + x if x == 0 and sc * y == 0 else 0.0)
    r = np.array(out, np.float64)
    return r if dtype == "f64" else X.narrow(r.astype(np.float32), dtype)


@pytest.mark.parametrize("dtype", ALL_DTYPES)
@pytest.mark.parametrize("op", ["scale", "add", "triad"])
def test_exact_reference_is_the_exact_value_rounded_once(op, dtype):
    """A sample of finite random operands and the finite adversarial sets against Fraction rounded by
    round_fraction, which is written from the formats' definitions: the TwoSum path of the f32 family and numpy's
    f64 arithmetic are the exact value rounded once (to f32, then to the storage type)."""
    cases = [("random", s, random_bits(dtype, 3000, 31), random_bits(dtype, 3000, 32)) for s in SCALARS[:6]]
    cases += X.adversarial(op, dtype, n=1000)
    for name, s, a, b in cases:
        if not np.isfinite(s) or (dtype != "f64" and not np.isfinite(X.f32_scalar(s))):
            continue
        keep = np.isfinite(X.widen(a, dtype)) & np.isfinite(X.widen(b, dtype))
        a, b = a[keep], b[keep]
        with np.errstate(all="ignore"):
            got = X.stream(op, dtype, a, b if op != "scale" else None, s)
        assert_same(got, exact_rounded_once(op, dtype, a, b, s), dtype, f"{name} s={s!r}")


def test_round_f32_ties_and_overflow_threshold():
    """round_f32(hi, lo) where hi alone rounds wrongly: hi exactly on an f32 midpoint (normal and subnormal) with lo
    of either sign or zero, and hi exactly on FLT_MAX + ulp/2 with lo of either sign."""
    T = X.F32_OVERFLOW
    hi = np.array([1 + 2.0 ** -24, 1 + 2.0 ** -24, 1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, 1 + 3 * 2.0 ** -24,
                   2.0 ** -150, 2.0 ** -150, 3 * 2.0 ** -150, 3 * 2.0 ** -150, T, T, T, -T, -T, -T,
                   X.FLT_MAX, T - 2.0 ** 75, 2.0 ** 128])
    lo = np.array([2.0 ** -80, -2.0 ** -80, 0.0, 2.0 ** -80, -2.0 ** -80,
                   2.0 ** -200, 0.0, -2.0 ** -200, 0.0, 2.0 ** 73, -2.0 ** 73, 0.0, -2.0 ** 73, 2.0 ** 73, 0.0,
                   2.0 ** 73, 2.0 ** 73, -2.0 ** 74])
    want = [X.round_fraction(Fraction(h) + Fraction(l), "f32") for h, l in zip(hi.tolist(), lo.tolist())]
    got = X.round_f32(hi, lo)
    assert got.tolist() == want
    assert got[9] == np.inf and got[10] == X.FLT_MAX and got[12] == -np.inf and got[13] == -X.FLT_MAX
    assert got[0] == np.float32(1 + 2.0 ** -23) and got[1] == 1.0 and got[2] == 1.0
    assert got[3] == np.float32(1 + 2.0 ** -22) and got[4] == np.float32(1 + 2.0 ** -23)
    assert got[5] == 2.0 ** -149 and got[6] == 0.0 and got[7] == 2.0 ** -149 and got[8] == 2.0 ** -148


def test_c_oracle_f64_fma_is_the_exact_rational():
    """Full-size f64 TRIAD arrays are checked against the C oracle (glibc fma): here it is pinned to
    Fraction(a) + Fraction(s) Fraction(b), rounded by float(), at doubles s that are no floats."""
    rng = np.random.default_rng(41)
    n = X.FRACTION_LIMIT // 4
    for s, a, b in [(0.1, rng.standard_normal(n), rng.standard_normal(n)),
                    (-1 / 3, random_bits("f64", n, 42), random_bits("f64", n, 43)),
                    (1 + 2.0 ** -52, *X._cancellation("f64", 1 + 2.0 ** -52, rng, n)),
                    (2.0 ** -1060, X.edge_values("f64", n, 44), X.edge_values("f64", n, 45))]:
        with np.errstate(all="ignore"):
            assert_same(oracle.stream("triad", "f64", a, b, s), X.stream("triad", "f64", a, b, s), "f64", repr(s))


def test_adversarial_sets_separate_the_contract_from_near_misses():
    """The sets a GPU test leans on really do tell a subtly wrong kernel apart: an unfused TRIAD (product rounded,
    then added) differs on most of the cancellation set, a single-rounding f16/bf16 TRIAD (a native half fma) on at
    least a third of the midpoint set, and f32(s) from s for the scalars of the GPU tests."""
    for dtype in ALL_DTYPES:
        for name, s, a, b in X.adversarial("triad", dtype):
            want = X.stream("triad", dtype, a, b, s)
            ut = X.BITS[dtype][0]
            with np.errstate(all="ignore"):
                if name.startswith("fma cancellation"):
                    if dtype == "f64":
                        unfused = np.float64(s) * b + a
                    else:
                        fa, fb = X.widen(a, dtype).astype(np.float32), X.widen(b, dtype).astype(np.float32)
                        unfused = X.narrow(np.float32(X.f32_scalar(s)) * fb + fa, dtype)
                    assert (unfused.view(ut) != want.view(ut)).mean() > 0.15, (dtype, name)
                if name.startswith("storage midpoints"):
                    single = X.narrow(np.array([X.round_fraction(Fraction(x) + Fraction(X.f32_scalar(s)) * Fraction(y), dtype)
                                                for x, y in zip(X.widen(a, dtype).tolist(), X.widen(b, dtype).tolist())],
                                               np.float32), dtype)
                    assert (single != want).mean() > 1 / 3, (dtype, name)
                    inf = 0x7C00 if dtype == "f16" else 0x7F80
                    assert ((want & 0x7FFF) == inf).any()               # the midpoint above the largest finite value
    assert X.f32_scalar(1 + 2.0 ** -24) == 1.0 and X.f32_scalar(1 + 2.0 ** -24 + 2.0 ** -52) == 1 + 2.0 ** -23
    assert X.f32_scalar(3.5e38) == np.inf and X.f32_scalar(1e-45) == 2.0 ** -149 and X.f32_scalar(1e-50) == 0.0
