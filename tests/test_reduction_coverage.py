"""The planted positions of tests/test_gpu_reductions.py have teeth, shown without a GPU.

A reduction hides a dropped element unless that element holds the maximum, so the GPU tests plant one at the
positions their restated launch plans name.  Here a model of each kernel's loops, under the plan the GPU test uses,
marks the work every CTA, warp and unroll slot takes:
- cast_tiles (the 1-D vector body): tile t goes to CTA t mod grid, and thread x of it takes units t tile + x + j
  threads for each unroll slot j; a partial tile guards each unit.
- cast_edges (the head and tail, or every element in mixed phase and on the transpose's element path): global thread
  g takes edge items g, g + grid threads, ..., item i being element i in the head and body_end + i - head after.
- quant_t_tiles (the transpose's tiled path): tile t goes to CTA t mod grid, and thread x of it takes group x % 4 of
  tile row x / 4 where the tile has that row and group.
- fp8r_reduce: the thread of a line reads its blocks 0 .. nb - 1.
Without a mutant the model takes every element once.  Each mutant drops one piece, as a wrong kernel would; in every
case where that changes what is taken, some planted position must fall outside the mutant's coverage, so the GPU
test sees a wrong maximum.  Each mutant must change at least one case.
"""
import functools

import numpy as np
import pytest

import test_gpu_reductions as R

ONE_D = ["head skipped", "tail skipped", "unroll slot 1 dropped", "partial tile dropped", "last CTA dropped",
         "last warp dropped"]
TILED = ["last CTA dropped", "last warp dropped", "partial edge tile dropped"]
REDUCE = ["row-wise reduction stops at nb - nb % 4"]
H100_SMS = 132                      # the H100 SXM's SMs, for the case that needs more tiles than they hold at once


# ------------------------------------------------------------------------------------------- the cases
@functools.cache
def one_d_cases():
    """{name: (plan, positions)} of every plan whose work is cast_tiles and cast_edges: the host-k amax (CastPlan into
    FP8; the SR quantize is es = 4) and the amax pass (AmaxPlan) over every amax case of every source size, and the
    transpose's element-path cases.  A and C sit where the GPU test's buffers put them: a 16-byte boundary plus the
    layout's element offsets."""
    cases = {}
    for es in (2, 4, 8):
        for n, layout, expect in R.amax_cases(es):
            oa, oc = R.LAYOUTS[layout]
            for name, p, want in ((f"CastPlan es={es} n={n} {layout}", R.CastPlan(es, 1, n, oa * es, oc), expect),
                                  (f"AmaxPlan es={es} n={n} {layout}", R.AmaxPlan(es, n, oa * es), R.amax_pass_expect(es, n, expect))):
                R.assert_reaches(p, want, name)
                cases[name] = (p, p.positions())
        for name, p in transpose_plans(es):
            if not p.tiled:
                cases[name] = (p, p.positions())
    return cases


def transpose_plans(es):
    for rows, cols, (oa, oc, ot), expect in R.TRANSPOSE_CASES:
        name = f"TransposePlan es={es} {rows}x{cols} offsets {oa},{oc},{ot}"
        p = R.TransposePlan(es, rows, cols, oa * es, oc, ot)
        R.assert_transpose_reaches(p, expect, H100_SMS, name)
        yield name, p


@functools.cache
def tiled_cases():
    return {name: (p, p.positions()) for es in (2, 4, 8) for name, p in transpose_plans(es) if p.tiled}


# ------------------------------------------------------------------------------------------- the models
def lanes(p, drop):
    """The threads of a CTA that run: all, or all but the last warp."""
    return np.arange(p.threads - 32 if drop == "last warp dropped" else p.threads)


def ctas_of(tiles, p, drop):
    """The tiles whose CTA (tile mod grid, by the grid-stride loop) runs."""
    return tiles[tiles % p.grid < p.grid - (drop == "last CTA dropped")]


def one_d_cover(p, drop=None):
    """(how often each unit of the vector body is taken, how often each edge item is taken)."""
    units = np.zeros(p.ngroups, np.int64)
    tile = p.threads * p.unroll
    t = ctas_of(np.arange(-(-p.ngroups // tile)), p, drop)
    if drop == "partial tile dropped":
        t = t[(t + 1) * tile <= p.ngroups]
    for j in range(1 if drop == "unroll slot 1 dropped" else p.unroll):
        u = (t[:, None] * tile + j * p.threads + lanes(p, drop)[None, :]).ravel()
        units[u[u < p.ngroups]] += 1
    edges = np.zeros(p.n - p.ngroups * p.G, np.int64)
    stride = p.grid * p.threads
    g = (ctas_of(np.arange(p.grid), p, drop)[:, None] * p.threads + lanes(p, drop)[None, :]).ravel()
    for i0 in range(0, edges.size, stride):
        i = g + i0
        i = i[i < edges.size]
        if drop == "head skipped":
            i = i[i >= p.head]
        if drop == "tail skipped":
            i = i[i < p.head]
        edges[i] += 1
    return units, edges


def one_d_takes(p, cover, e):
    """Whether the cover takes element e: unit (e - head) / G of the body, or its edge item."""
    units, edges = cover
    end = p.head + p.ngroups * p.G
    if p.head <= e < end:
        return units[(e - p.head) // p.G] > 0
    return edges[e if e < p.head else p.head + e - end] > 0


def tiled_cover(p, drop=None):
    """How often each element of the rows x cols matrix is taken."""
    count = np.zeros((p.rows, p.cols), np.int64)
    x = lanes(p, drop)
    r, q = x // 4, x % 4
    for t in ctas_of(np.arange(-(-p.rows // p.T) * -(-p.cols // p.T)), p, drop):
        i0, j0, tr, tc = p.box(int(t))
        if drop == "partial edge tile dropped" and (tr < p.T or tc < p.T):
            continue
        ok = (r < tr) & (16 * q < tc)
        count[(i0 + r[ok])[:, None], (j0 + 16 * q[ok])[:, None] + np.arange(16)[None, :]] += 1
    return count


def reduce_reads(nb, drop=None):
    """The blocks fp8r_reduce reads for a line of nb blocks."""
    return range(nb - nb % 4 if drop == REDUCE[0] else nb)


# ------------------------------------------------------------------------------------------- the tests
@functools.cache
def full_one_d(name):
    return one_d_cover(one_d_cases()[name][0])


def test_every_model_takes_every_element_once():
    for name, (p, pos) in one_d_cases().items():
        units, edges = full_one_d(name)
        assert (units == 1).all() and (edges == 1).all(), name
        assert all(0 <= e < p.n for e in pos), name
    for name, (p, pos) in tiled_cases().items():
        assert (tiled_cover(p) == 1).all(), name
    for side, nb, rows, cols, oa, path in R.rowwise_cases():
        p = R.ReducePlan(rows, cols)
        assert (p.nb_row if side == "row" else p.nb_col) == nb, (side, nb, rows, cols)


@pytest.mark.parametrize("mutant", list(dict.fromkeys(ONE_D + TILED + REDUCE)))
def test_every_mutant_misses_a_planted_position(mutant):
    changed = []
    if mutant in ONE_D:
        for name, (p, pos) in one_d_cases().items():
            full, cover = full_one_d(name), one_d_cover(p, mutant)
            if all(np.array_equal(f, c) for f, c in zip(full, cover)):
                continue
            changed.append(name)
            assert not all(one_d_takes(p, cover, e) for e in pos), f"{name}: {mutant}, yet every plant is taken"
    if mutant in TILED:
        for name, (p, pos) in tiled_cases().items():
            cover = tiled_cover(p, mutant).ravel()
            if (cover == 1).all():
                continue
            changed.append(name)
            assert not all(cover[e] for e in pos), f"{name}: {mutant}, yet every plant is taken"
    if mutant in REDUCE:
        for side, nb, rows, cols, oa, path in R.rowwise_cases():
            if len(reduce_reads(nb, mutant)) == nb:
                continue
            name = f"ReducePlan {rows}x{cols} {side} side, {path} path"
            changed.append(name)
            blocks = {(j if side == "row" else i) // 128 for i, j in R.rowwise_plants(side, nb, rows, cols)}
            assert blocks - set(reduce_reads(nb, mutant)), f"{name}: {mutant}, yet every plant is read"
    assert changed, f"no case tells {mutant} from the kernel"
    print(f"{mutant}: caught in all {len(changed)} cases it changes")
