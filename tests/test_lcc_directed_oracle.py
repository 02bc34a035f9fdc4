"""The directed LCC oracle (oracle/lcc_directed_oracle.py) against the definition: brute-force pair
enumeration on small random multigraphs, its oriented form on every case, and on an all-reciprocal
simple graph, where W = 2 A, the identity lcc_directed = LCC of the undirected graph
(oracle/pyoracle's lcc: 2 t / (d (d - 1)) with t triangles, d = 2 deg; here tri = 2 t and
d = deg, so both give 2 t / (deg (deg - 1)))."""
import numpy as np
import pytest

from oracle import lcc_directed_oracle as LO
from oracle import pyoracle
from tests.lcc_directed_cases import as_indices, lcc_directed_cases, multigraph, parallel_pair, reciprocal

CASES = lcc_directed_cases()


@pytest.mark.parametrize("seed", range(6))
def test_matches_brute_force(seed):
    n, s, d = multigraph(25 + 5 * seed, 120 + 40 * seed, seed)
    lcc, tri, deg = LO.lcc_directed(n, s, d)
    bt, bd = LO.brute_force(n, s, d)
    assert np.array_equal(tri, bt)
    assert np.array_equal(deg, bd)
    ok = bd >= 2
    assert np.array_equal(lcc[ok], bt[ok] / (bd[ok] * (bd[ok] - 1.0)))
    assert np.all(lcc[~ok] == 0.0)


def test_probe_graph():
    """0->1 twice, 1->2, 2->0, 0->2, a self loop on 3, 3->0, 3->1 and the isolated vertex 4."""
    s = np.array([0, 1, 2, 0, 3, 3, 0, 3])
    d = np.array([1, 2, 0, 2, 3, 0, 1, 1])
    _, tri, deg = LO.lcc_directed(5, s, d)
    assert tri.tolist() == [2, 3, 2, 2, 0]
    assert deg.tolist() == [3, 3, 2, 3, 0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oriented_form_equals_direct(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    for reference in (False, True):
        a = LO.lcc_directed(n, s, d, reference=reference)
        b = LO.lcc_directed_fast(n, s, d, reference=reference)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        assert a[0].tobytes() == b[0].tobytes()


@pytest.mark.parametrize("seed", range(3))
def test_reciprocal_equals_undirected_lcc(seed):
    n, s, d = reciprocal(80 + 20 * seed, 0.15, seed)
    half = s < d
    g = pyoracle.Graph(n, s[half], d[half], None, directed=False)
    want, _ = g.lcc()
    got, _, _ = LO.lcc_directed(n, s, d)
    assert got.tobytes() == np.asarray(want, dtype=np.float64).tobytes()


@pytest.mark.parametrize("copies", [255, 256, 300])
def test_reference_weights_wrap(copies):
    """The pair {0, 1} weighs `copies`; reference mode weighs it copies % 256 (vertex 2 and vertex 3 see
    the pair as their opposite edge); the deduplicated degrees are the same in both modes."""
    n, s, d = parallel_pair(copies)
    _, exact, d0 = LO.lcc_directed(n, s, d)
    _, ref, d1 = LO.lcc_directed(n, s, d, reference=True)
    assert np.array_equal(d0, d1)
    assert exact[2] == copies and exact[3] == copies
    assert ref[2] == copies % 256 and ref[3] == copies % 256
    assert np.array_equal(exact[:2], ref[:2])


@pytest.mark.parametrize("fnum", [2, 3])
def test_stats_shares_add_up(fnum):
    """The statistics model: on any cut of the vertices the fragments' shares of the scanned entries and
    of the frontier add up to the one-fragment values, and the one-fragment count is the sum over
    oriented entries (v, u) of |N+(u)|, counted here pair by pair."""
    n, s, d = multigraph(60, 400, fnum)
    rank = np.random.default_rng(fnum).permutation(n)
    whole = LO.stats(n, s, d, rank=rank)
    owner = np.arange(n) % fnum
    shares = [LO.stats(n, s, d, rank=rank, owned=owner == f) for f in range(fnum)]
    assert sum(x.entries_scanned for x in shares) == whole.entries_scanned
    assert sum(x.frontier_vertices for x in shares) == whole.frontier_vertices == n
    deg = np.bincount(s, minlength=n) + np.bincount(d, minlength=n)
    nbr = [set() for _ in range(n)]
    for a, b in zip(s.tolist(), d.tolist()):
        nbr[a].add(b)
        nbr[b].add(a)
    up = [{u for u in nbr[v] if u != v and (deg[u], rank[u]) < (deg[v], rank[v])} for v in range(n)]
    assert whole.entries_scanned == sum(len(up[u]) for v in range(n) for u in up[v])
    assert whole.supersteps == 3 and whole.step_mode == [0, 2, 0]
