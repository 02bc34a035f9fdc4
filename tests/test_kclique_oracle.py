"""The k-clique oracle (oracle/kclique_oracle.py) against brute force on small
random multigraphs and against closed forms."""
import itertools
from math import comb

import numpy as np
import pytest

from oracle import kclique_oracle as KO
from tests import shapes as S
from tests.core_cases import random_multigraph


def brute(n, src, dst, k):
    adj = set()
    for a, b in zip(np.asarray(src).tolist(), np.asarray(dst).tolist()):
        if a != b:
            adj.add((min(a, b), max(a, b)))
    return sum(all(p in adj for p in itertools.combinations(c, 2)) for c in itertools.combinations(range(n), k))


@pytest.mark.parametrize("seed", range(12))
def test_random_small_graphs_against_combinations(seed):
    rng = np.random.RandomState(100 + seed)
    n = int(rng.randint(2, 13))
    m = int(rng.randint(0, n * (n - 1) // 2 + 1))
    src, dst = rng.randint(0, n, size=m), rng.randint(0, n, size=m)
    for k in (3, 4, 5, 6):
        assert KO.count(n, src, dst, k) == brute(n, src, dst, k), k


@pytest.mark.parametrize("n", [1, 3, 7, 12])
def test_clique(n):
    _, s, d, _ = S.clique(n)
    for k in range(3, n + 2):
        assert KO.count(n, s, d, k) == comb(n, k), k


@pytest.mark.parametrize("r,a", [(3, 2), (4, 3), (5, 2)])
def test_complete_multipartite(r, a):
    n = r * a
    part = np.arange(n) // a
    i, j = np.triu_indices(n, 1)
    keep = part[i] != part[j]
    for k in range(3, r + 2):
        assert KO.count(n, i[keep], j[keep], k) == comb(r, k) * a ** k, k


def test_triangle_free_graphs_give_zero():
    for n, s, d, _ in (S.complete_bipartite(5, 9), S.star(50), S.path(40), S.empty(10)):
        for k in (3, 4, 5):
            assert KO.count(n, s, d, k) == 0


@pytest.mark.parametrize("seed", range(8))
def test_multigraph_equals_its_simplification(seed):
    n, s, d = random_multigraph(seed)
    a, b = KO.simple_edges(n, s, d)
    for k in (3, 4, 5):
        assert KO.count(n, s, d, k) == KO.count(n, a, b, k)
