"""The order-exact betweenness oracle (oracle/bc_oracle.py bc_rows) on the CPU:
its butterfly fold and row sums against plain scalar restatements of the
kernel's order, its results against the f64 oracle and the exact-rational brute
force, the graphs of tests/bc_shapes.py against the branches they are there
for, and -- the order guard -- that the order-sensitive graphs really tell the
kernel's order apart from a sequential one and from a cut moved by one entry."""
import numpy as np
import pytest

from oracle import bc_oracle as BO
from tests import bc_shapes as B
from tests.core_cases import random_multigraph
from tests.test_bc_oracle import brute_force, closed_form_cases

INF = BO.INF


def _wide(rng, k):
    """k positive f64 values spread over 2^-60 .. 2^60, so that every sum of them rounds."""
    return rng.rand(k) * 2.0 ** rng.randint(-60, 61, size=k)


def _bits(x):
    return np.asarray(x).view(np.uint8).tobytes()


def test_warp_fold_is_the_butterfly():
    rng = np.random.RandomState(0)
    for _ in range(200):
        a = _wide(rng, 32)
        lanes = a.tolist()
        for o in (16, 8, 4, 2, 1):   # warp_sum: every lane adds the lane o apart, all at once
            lanes = [lanes[i] + lanes[i ^ o] for i in range(32)]
        assert len(set(lanes)) == 1
        x = a.tolist()
        tree = ((((x[0] + x[16]) + (x[8] + x[24])) + ((x[4] + x[20]) + (x[12] + x[28])))
                + (((x[2] + x[18]) + (x[10] + x[26])) + ((x[6] + x[22]) + (x[14] + x[30])))) \
            + ((((x[1] + x[17]) + (x[9] + x[25])) + ((x[5] + x[21]) + (x[13] + x[29])))
               + (((x[3] + x[19]) + (x[11] + x[27])) + ((x[7] + x[23]) + (x[15] + x[31]))))
        assert float(BO.warp_fold(a)) == lanes[0] == tree


def _scalar_row_sum(vals, short, chunk):
    """One row, written out the way gather_level sums it."""
    if short is None or len(vals) <= short:
        s = 0.0
        for x in vals:
            s += x
        return s
    total = 0.0
    for c0 in range(0, len(vals), chunk):
        part = vals[c0:c0 + chunk]
        lanes = [0.0] * 32
        for j, x in enumerate(part):
            lanes[j % 32] += x
        for o in (16, 8, 4, 2, 1):
            lanes = [lanes[i] + lanes[i ^ o] for i in range(32)]
        total += lanes[0]
    return total


@pytest.mark.parametrize("short,chunk", [(32, 1024), (31, 1024), (32, 1023), (None, 1024), (32, 64)])
def test_ordered_row_sums_equal_the_scalar_order(short, chunk):
    rng = np.random.RandomState(1)
    degs = [0, 1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2048, 2049, 3073, 5, 0, 700]
    n = len(degs) + 50
    term = _wide(rng, n)
    term[rng.rand(n) < 0.2] = 0.0
    rp = np.concatenate([[0], np.cumsum(degs)]).astype(np.int64)
    col = rng.randint(0, n, size=int(rp[-1]))
    vs = np.array([3, 0, 9, 1, 2, 4, 5, 6, 7, 8, 10, 11, 12, 13, 14, 15, 16])
    got = BO.ordered_row_sums(rp, col, vs, term, short, chunk)
    for i, v in enumerate(vs):
        assert got[i] == _scalar_row_sum(term[col[rp[v]:rp[v + 1]]].tolist(), short, chunk), (v, degs[v])


@pytest.mark.parametrize("seed", range(24))
def test_bc_rows_on_random_multigraphs(seed):
    n, s, d = random_multigraph(seed)
    source = int(np.random.RandomState(1000 + seed).randint(0, n))
    rp, col = BO.sorted_csr(n, s, d)
    depth, sigma, c = brute_force(n, s, d, source)
    for short in (32, None, 1):   # short=1: nearly every row goes through the chunked path
        gc, gs, gd = BO.bc_rows(n, rp, col, source, short=short)
        fc, fs, fd = BO.bc(n, s, d, source, "f64")
        assert np.array_equal(gd, fd) and _bits(gs) == _bits(fs)
        for v in range(n):
            if depth[v] is None:
                assert gd[v] == INF and gs[v] == 0 and gc[v] == 0
                continue
            assert gs[v] == float(sigma[v])
            assert abs(float(gc[v]) - float(c[v])) <= 1e-6 * max(1.0, abs(float(c[v]))), v


@pytest.mark.parametrize("case", closed_form_cases(), ids=lambda c: c[0])
def test_bc_rows_closed_forms(case):
    _, n, s, d, source, want = case
    rp, col = BO.sorted_csr(n, np.asarray(s), np.asarray(d))
    c, sigma, depth = BO.bc_rows(n, rp, col, source)
    fc, fs, fd = BO.bc(n, np.asarray(s), np.asarray(d), source, "f64")
    assert np.array_equal(depth, fd) and np.array_equal(sigma, fs)
    assert np.allclose(c, [float(x) for x in want], rtol=2 ** -22, atol=0)


def test_bc_rows_absent_and_isolated_sources():
    n, s, d = 7, np.array([0, 1, 2]), np.array([1, 2, 3])
    rp, col = BO.sorted_csr(n, s, d)
    for source in (None, n, -1):
        c, sigma, depth = BO.bc_rows(n, rp, col, source)
        assert (depth == INF).all() and not sigma.any() and not c.any()
    c, sigma, depth = BO.bc_rows(n, rp, col, 5)
    assert depth[5] == 0 and sigma[5] == 1 and c[5] == 0 and (np.delete(depth, 5) == INF).all()


def _differs(a, b):
    return any(_bits(x) != _bits(y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", B.ORDER_SENSITIVE)
def test_order_guard(name):
    """Each order-sensitive graph tells the kernel's order from a sequential sum over every row."""
    build, root = B.BC_SHAPES[name]
    n, s, d, _ = build()
    rp, col = BO.sorted_csr(n, s, d)
    got = BO.bc_rows(n, rp, col, root)
    assert _differs(got, BO.bc(n, s, d, root, "f64")), "%s: the kernel order and the f64 mode agree" % name
    assert _differs(got, BO.bc_rows(n, rp, col, root, short=None))


@pytest.mark.parametrize("cut", ["short=31", "chunk=1023"])
def test_order_guard_moves_with_each_cut(cut):
    """Moving kBcShort or kBcChunk by one entry changes a result on one of the order-sensitive graphs."""
    kw = {"short": 31} if cut == "short=31" else {"chunk": 1023}
    moved = False
    for name in B.ORDER_SENSITIVE:
        build, root = B.BC_SHAPES[name]
        n, s, d, _ = build()
        rp, col = BO.sorted_csr(n, s, d)
        moved |= _differs(BO.bc_rows(n, rp, col, root), BO.bc_rows(n, rp, col, root, **kw))
    assert moved, cut


@pytest.mark.parametrize("name", sorted(B.BC_SHAPES))
def test_bc_shapes_reach_their_branches(name):
    """On the sorted CSR (the GPU test repeats this on the fragment's own)."""
    build, root = B.BC_SHAPES[name]
    n, s, d, _ = build()
    rp, col = BO.sorted_csr(n, s, d)
    root = B.sources(n, rp, col, root)[0]
    checks = B.reach_checks(name, n, rp, col, root)
    assert all(ok for _, ok in checks), [what for what, ok in checks if not ok]


def test_step_replica_by_hand():
    # path 0-1-2-3-4 from 0, push only: level d + 1 reads the rows of level d, plus its own rows from d + 1 = 2
    n, s, d = 5, np.arange(4), np.arange(1, 5)
    rp, col = BO.sorted_csr(n, s, d)
    _, depth = BO.levels_of(n, rp, col, 0)
    assert B.forward_steps(n, rp, col, depth, 0) == [(0, 0), (0, 1), (0, 2 + 2), (0, 2 + 2), (0, 2 + 1)]
    assert B.backward_entries(rp, depth) == [1, 2, 2, 2, 1]
    # star of 30 leaves from the centre: 30 > (60 - 30) / 14 pulls level 1; every leaf probes one entry
    n, s, d = 31, np.zeros(30, dtype=np.int64), np.arange(1, 31)
    rp, col = BO.sorted_csr(n, s, d)
    _, depth = BO.levels_of(n, rp, col, 0)
    assert B.forward_steps(n, rp, col, depth, 1) == [(0, 0), (1, 30)]
    # from a leaf: level 1 (the centre) is pushed; 30 > (60 - 31) / 14 pulls level 2, where the 29
    # unvisited leaves probe one entry each and the gather reads their 29 rows
    _, depth = BO.levels_of(n, rp, col, 1)
    assert B.forward_steps(n, rp, col, depth, 1) == [(0, 0), (0, 1), (1, 29 + 29)]
    assert B.pull_probes(rp, col, depth, 1) == 29


@pytest.mark.parametrize("scale", [20])
def test_bc_rows_is_fast_enough_for_rmat(scale):
    """R-MAT 20 from its maximum-degree vertex: equal to the f64 mode in depth and sigma, in seconds."""
    import time
    from tests.util import rmat_graph
    n, s, d, _ = rmat_graph(scale, seed=1)
    source = int(np.argmax(np.bincount(np.concatenate([s, d]), minlength=n)))
    rp, col = BO.sorted_csr(n, s, d)
    t0 = time.time()
    c, sigma, depth = BO.bc_rows(n, rp, col, source)
    assert time.time() - t0 < 60
    fc, fs, fd = BO.bc(n, s, d, source, "f64")
    assert np.array_equal(depth, fd) and np.array_equal(sigma, fs)
