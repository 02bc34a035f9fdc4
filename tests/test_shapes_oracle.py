"""The CPU oracle on the constructed threshold graphs of tests/shapes.py, checked
against closed forms (it is the reference of every GPU comparison on them), and
the shape constants checked against the kernels' own `constexpr` values, so a
retuned constant cannot silently stop a shape from sitting on its boundary."""
import os
import re
from math import comb

import numpy as np
import pytest

from oracle import pyoracle
from tests import golden_io as G
from tests import shapes as S

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "libgrape-lite_b200", "csrc")
INT64_MAX = np.iinfo(np.int64).max


def graph(shape, directed=False):
    n, src, dst, w = shape
    return pyoracle.Graph(n, src, dst, w, directed=directed)


def _constexpr(fname, name, names=None):
    """Value of `constexpr T name = expr;` in csrc/fname; expr may use the constants in `names`."""
    text = open(os.path.join(CSRC, fname)).read()
    m = re.search(r"constexpr\s+[\w:]+\s+%s\s*=\s*([^;]+);" % name, text)
    assert m, "%s not found in %s" % (name, fname)
    return int(eval(re.sub(r"(\d)u\b", r"\1", m.group(1)), dict(names or {})))


@pytest.mark.parametrize("fname,name,value", [
    ("engine.cuh", "kHubDeg", S.K_HUB_DEG), ("engine.cuh", "kTileV", S.K_TILE_V),
    ("engine.cuh", "kMaxTileHubs", S.K_MAX_TILE_HUBS), ("engine.cuh", "kHubChunk", S.K_HUB_CHUNK),
    ("dense.cuh", "kDenseTile", S.K_DENSE_TILE),
    ("dense.cuh", "kDenseRows", S.K_DENSE_ROWS), ("app_pagerank.cu", "kPrHub", S.K_PR_HUB)])
def test_shape_constants_match_kernels(fname, name, value):
    assert _constexpr(fname, name) == value


def test_queue_scan_cm_cut_matches_kernel():
    """The cm / cmold cut of gl_edge_scan_queue, and the hub-list size it is checked against."""
    hub_deg = _constexpr("engine.cuh", "kHubDeg")
    assert _constexpr("primitives.cu", "kHubDegCm", {"kHubDeg": hub_deg}) == S.K_HUB_DEG_CM
    text = open(os.path.join(CSRC, "primitives.cu")).read()
    assert "m / kHubChunk + m / kHubDeg + 1024" in text      # S.hub_cap


def test_bfs_thresholds_match_kernel():
    text = open(os.path.join(CSRC, "app_bfs.cu")).read()
    m = re.search(r"fv\.ivnum >= \(1u << (\d+)\) && cfg\.reserved\[1\] == 0", text)
    assert m and (1 << int(m.group(1))) == S.HUB_FIRST_MIN_V
    m = re.search(r"depth_base == 0 && nl <= (\d+)", text)
    assert m and int(m.group(1)) == S.BFS_U8_MAX_LEVELS


# ------------------------------------------------------------ closed forms ----
@pytest.mark.parametrize("L", [2, 251, 255, 256, 259])
def test_path_bfs_depths(L):
    g = graph(S.path(L))
    assert np.array_equal(g.bfs(0)[0], np.arange(L))
    assert np.array_equal(g.bfs(L - 1)[0], np.arange(L)[::-1])


@pytest.mark.parametrize("k", [1, 1025, 4097])
@pytest.mark.parametrize("last", [False, True])
def test_star_bfs_depths(k, last):
    n, src, dst, w = S.star(k, last)
    g = graph((n, src, dst, w))
    c = n - 1 if last else 0
    want = np.ones(n, dtype=np.int64)
    want[c] = 0
    assert np.array_equal(g.bfs(c)[0], want)
    leaf = 1 if c == 0 else 0
    want = np.full(n, 2, dtype=np.int64)
    want[c], want[leaf] = 1, 0
    assert np.array_equal(g.bfs(leaf)[0], want)


def test_empty_graphs():
    for n in (1, 33, 1025):
        g = graph(S.empty(n))
        d = g.bfs(n - 1)[0]
        assert d[n - 1] == 0 and np.sum(d == INT64_MAX) == n - 1
        assert np.array_equal(g.wcc()[0], np.arange(n))
        assert np.array_equal(g.cdlp(3), np.arange(n))
        assert np.array_equal(g.lcc()[0], np.zeros(n))
        assert np.allclose(g.pagerank(0.85, 10, 0), 1.0 / n, rtol=1e-12)


@pytest.mark.parametrize("k", [2, 3, 32, 33, 200])
def test_clique_lcc(k):
    lcc, tri = graph(S.clique(k)).lcc()
    assert np.array_equal(tri, np.full(k, comb(k - 1, 2)))
    assert np.array_equal(lcc, np.full(k, 1.0 if k >= 3 else 0.0))


@pytest.mark.parametrize("n,k", [(40, 2), (1000, 5), (2048, 16)])
def test_ring_lattice_lcc(n, k):
    lcc, tri = graph(S.ring_lattice(n, k)).lcc()
    assert np.array_equal(tri, np.full(n, 3 * k * (k - 1) // 2))
    assert np.allclose(lcc, 3.0 * (k - 1) / (2.0 * (2 * k - 1)), rtol=1e-15, atol=0)


@pytest.mark.parametrize("k,last", [(5, False), (4097, False), (4097, True)])
def test_star_cdlp_rounds(k, last):
    n = k + 1
    g = graph(S.star(k, last))
    c = n - 1 if last else 0
    min_leaf = 1 if c == 0 else 0
    r1 = np.full(n, c, dtype=np.int64)      # every leaf sees only the centre
    r1[c] = min_leaf                         # all leaf labels tie once: the smallest wins
    assert np.array_equal(g.cdlp(1), r1)
    r2 = np.full(n, min_leaf, dtype=np.int64)
    r2[c] = c
    assert np.array_equal(g.cdlp(2), r2)


@pytest.mark.parametrize("a,b", [(3, 5), (40, 70)])
def test_bipartite_cdlp_oscillates_and_lcc_zero(a, b):
    g = graph(S.complete_bipartite(a, b))
    left = np.arange(a + b) < a
    assert np.array_equal(g.cdlp(1), np.where(left, a, 0))
    assert np.array_equal(g.cdlp(2), np.where(left, 0, a))
    assert np.array_equal(g.cdlp(3), np.where(left, a, 0))
    assert np.array_equal(g.lcc()[0], np.zeros(a + b))
    d = g.bfs(0)[0]
    assert np.array_equal(d, np.where(left, 2, 1) - (np.arange(a + b) == 0) * 2)


@pytest.mark.parametrize("seed", [None, 3])
def test_union_wcc_labels(seed):
    parts = [S.star(50), S.empty(3), S.path(20), S.clique(5), S.complete_bipartite(2, 3)]
    n, src, dst, w = S.union(parts, seed=seed)
    perm = np.arange(n) if seed is None else np.random.RandomState(seed).permutation(n)
    want = np.empty(n, dtype=np.int64)
    off = 0
    for pn, ps, pd, _ in parts:
        if len(ps):
            ids = perm[off:off + pn]
            want[ids] = ids.min()
        else:
            want[perm[off:off + pn]] = perm[off:off + pn]
        off += pn
    for directed in (False, True):
        assert np.array_equal(graph((n, src, dst, w), directed).wcc()[0], want)


@pytest.mark.parametrize("shape", ["star", "path", "clique", "bipartite", "multi_loop", "union", "padded"])
def test_undirected_pagerank_sums_to_one(shape):
    sh = {"star": lambda: S.star(4097), "path": lambda: S.path(300), "clique": lambda: S.clique(33),
          "bipartite": lambda: S.complete_bipartite(40, 70), "multi_loop": S.multi_loop,
          "union": lambda: S.union([S.star(1025, True), S.empty(7), S.path(256)], seed=1),
          "padded": lambda: S.pad_to(S.star(1025), 2000)}[shape]()
    g = graph(sh)
    for mode in (0, 1):
        for rounds in (1, 10):
            assert abs(g.pagerank(0.85, rounds, mode).sum() - 1.0) < 1e-12


@pytest.mark.parametrize("name,mode,app", [("star5", 0, "pagerank"), ("star5", 1, "pagerank_parallel"),
                                           ("sink4", 2, "pagerank_parallel")])
@pytest.mark.parametrize("rounds", [0, 1])
def test_pagerank_rounds_against_reference(name, mode, app, rounds):
    """After zero rounds the reference's `pagerank` app returns 0 for every vertex (its
    PEval returns before writing a rank) while `pagerank_parallel` returns 1/N, as does
    the reference's GPU app; oracle mode 0 follows the former, modes 1 and 2 the latter."""
    _, arrays = G.ref_outputs()
    want = arrays["%s_%s%d" % (name, app, rounds)]
    sh, directed = (S.star(5), False) if name == "star5" else (S.sink_heavy(4), True)
    got = graph(sh, directed).pagerank(0.85, rounds, mode)
    assert np.allclose(got, want, rtol=1e-12, atol=0)
    if rounds == 0:
        assert np.allclose(want, 0.0 if app == "pagerank" else 1.0 / sh[0], rtol=1e-12, atol=0)


def test_directed_pagerank_modes_on_a_sink():
    """A directed star into a sink: mode 2 (the reference's directed CPU app) keeps the
    dangling centre at the round's base rank; that is the rule the GPU app follows."""
    k = 100
    g = graph(S.sink_heavy(k), directed=True)
    r = g.pagerank(0.85, 1, 2)
    n = k + 1
    base = 0.15 / n + 0.85 * (1.0 / n) / n       # one dangling vertex of rank 1/n
    assert r[0] == pytest.approx(base, rel=1e-15)
    assert np.allclose(r[1:], base, rtol=1e-15)    # the sources have no in-edge


# --------------------------------------------------- path-taken preconditions ----
def test_shape_geometry():
    """The shapes reach their thresholds on the oracle's CSR layout (the same row
    order as a one-fragment GPU fragment)."""
    rp = graph(S.hub_block(33)).csr()[0]
    assert S.long_rows_per_block(rp) > S.K_MAX_TILE_HUBS
    assert S.hub_rows_unaligned(rp) > 0
    for sh in (S.star(4097), S.star(4097, True), S.path(5000)):
        assert S.max_dense_tile_rows(graph(sh).csr()[0]) > S.K_DENSE_ROWS
    rp = graph(S.multi_loop()).csr()[0]
    assert np.diff(rp.astype(np.int64)).max() > S.K_HUB_DEG
    assert S.max_dense_tile_rows(graph(S.star(1023)).csr()[0]) <= S.K_DENSE_ROWS + 1


@pytest.mark.parametrize("name", sorted(S.ENGINE_SHAPES))
def test_engine_shape_paths(name):
    """The engine-primitive graphs are bipartite covers whose side-A queues reach
    the queue scan's branches (long rows over each cut, more than kMaxTileHubs of
    them in one tile, hub items off a 4-aligned entry, hub items above hub_cap)."""
    n, src, dst, w = S.ENGINE_SHAPES[name]()
    rp, col, _ = graph((n, src, dst, w)).csr()
    side_a = np.arange(0, n, 2)
    starts = rp[side_a].astype(np.int64)
    deg = (rp[side_a + 1] - rp[side_a]).astype(np.int64)
    ent = np.repeat(starts - np.concatenate([[0], np.cumsum(deg)[:-1]]), deg) + np.arange(deg.sum())
    assert np.all(col[ent] % 2 == 1)                          # side A points into side B only
    checks = S.engine_path_checks(name, rp, side_a)
    assert checks and all(ok for _, ok in checks), [what for what, ok in checks if not ok]


def test_bipartite_cover_degrees():
    n, src, dst, w = S.bipartite_cover(S.rows_of_degree(S.ROW_DEGREES))
    rp = graph((n, src, dst, w)).csr()[0].astype(np.int64)
    assert list(np.diff(rp)[0:2 * len(S.ROW_DEGREES):2]) == S.ROW_DEGREES
    nd, sd, dd, wd = S.bipartite_cover(S.path(5), directed=True)
    assert nd == 10 and list(sd) == [0, 2, 4, 6] and list(dd) == [3, 5, 7, 9]
