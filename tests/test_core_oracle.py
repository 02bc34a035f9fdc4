"""CPU checks of the core decomposition / k-core oracle (oracle/core_oracle.py):
closed forms on the constructed graphs of tests/shapes.py, and a brute-force
k-core restatement on random multigraphs with self loops."""
import numpy as np
import pytest

from oracle import core_oracle as CO
from tests import shapes as S
from tests.core_cases import random_multigraph


def brute_kcore_set(n, src, dst, k):
    """The k-core by definition: drop any vertex with fewer than k entries to the
    vertices still present (a self loop is two entries) until none is left to drop."""
    alive = np.ones(n, dtype=bool)
    pairs = list(zip(np.asarray(src).tolist(), np.asarray(dst).tolist()))
    while True:
        deg = np.zeros(n, dtype=np.int64)
        for u, v in pairs:
            if alive[u] and alive[v]:
                deg[u] += 1
                deg[v] += 1
        drop = alive & (deg < k)
        if not drop.any():
            return alive
        alive &= ~drop


def brute_core(n, src, dst):
    core = np.zeros(n, dtype=np.int64)
    k = 1
    while True:
        alive = brute_kcore_set(n, src, dst, k)
        if not alive.any():
            return core
        core[alive] = k
        k += 1


def brute_kcore_value(n, src, dst, k):
    alive = brute_kcore_set(n, src, dst, k)
    val = np.zeros(n, dtype=np.int64)
    for u, v in zip(np.asarray(src).tolist(), np.asarray(dst).tolist()):
        val[u] += alive[v]
        val[v] += alive[u]
    return val


@pytest.mark.parametrize("seed", range(8))
def test_oracle_matches_the_definition_on_random_multigraphs(seed):
    n, src, dst = random_multigraph(seed)
    core, rounds = CO.core_decomposition(n, src, dst)
    assert np.array_equal(core, brute_core(n, src, dst))
    assert rounds >= (1 if len(src) else 0)
    for k in sorted({0, 1, 2, 3, int(core.max()), int(core.max()) + 1}):
        val = CO.kcore(n, src, dst, k)
        assert np.array_equal(val, brute_kcore_value(n, src, dst, k)), k
        assert np.array_equal(val >= k, core >= k) if k > 0 else np.all(val >= 0)


@pytest.mark.parametrize("k", [2, 3, 5, 17])
def test_clique(k):
    n, s, d, _ = S.clique(k)
    assert np.all(CO.core_decomposition(n, s, d)[0] == k - 1)


@pytest.mark.parametrize("n,k", [(7, 1), (9, 2), (50, 3), (1000, 5)])
def test_ring_lattice(n, k):
    nn, s, d, _ = S.ring_lattice(n, k)
    assert np.all(CO.core_decomposition(nn, s, d)[0] == 2 * k)


@pytest.mark.parametrize("shape", [S.star(1), S.star(5000), S.star(1025, centre_last=True), S.path(2), S.path(259)])
def test_star_and_path(shape):
    n, s, d, _ = shape
    core, rounds = CO.core_decomposition(n, s, d)
    assert np.all(core == 1)
    assert rounds >= 1


@pytest.mark.parametrize("a,b", [(1, 1), (3, 7), (40, 40), (2, 1500)])
def test_complete_bipartite(a, b):
    n, s, d, _ = S.complete_bipartite(a, b)
    assert np.all(CO.core_decomposition(n, s, d)[0] == min(a, b))


@pytest.mark.parametrize("n", [1, 33, 1025])
def test_empty(n):
    nn, s, d, _ = S.empty(n)
    core, rounds = CO.core_decomposition(nn, s, d)
    assert np.all(core == 0) and rounds == 0
    assert np.all(CO.kcore(nn, s, d, 3) == 0)


@pytest.mark.parametrize("j", [1, 2, 5])
def test_self_loop_only_vertex(j):
    # vertex 0: j self loops and nothing else; vertex 1 isolated; 2-3 an edge
    src = np.array([0] * j + [2], dtype=np.int64)
    dst = np.array([0] * j + [3], dtype=np.int64)
    core, _ = CO.core_decomposition(4, src, dst)
    assert core.tolist() == [2 * j, 0, 1, 1]
    # k-core: the loops survive up to k = 2j; once removed, a vertex's own entries no longer count
    assert CO.kcore(4, src, dst, 2 * j).tolist() == [2 * j, 0, 0, 0]
    assert CO.kcore(4, src, dst, 2 * j + 1).tolist() == [0, 0, 0, 0]


def test_multi_loop_shape():
    n, s, d, _ = S.multi_loop(copies=60, loops=3)
    core, _ = CO.core_decomposition(n, s, d)
    assert core[0] == core[1] == 60   # the 60 copies of 0-1 outlive vertex 2's 4 entries
    assert np.array_equal(core, brute_core(n, s, d))
