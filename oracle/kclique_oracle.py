"""Exact k-clique counter — TEST INFRASTRUCTURE ONLY.

Counts the k-cliques of the simple graph underneath an edge list: every edge
becomes the pair (min, max), self loops and repeated pairs are dropped.  k = 3
is trace(A^3) / 6 computed on scipy's sparse matrices as the number of
transitive triples of the orientation O of A (sum of (O O) * O, which equals
trace(A^3) / 6 without forming the dense A^2 of a star); larger k recurse vertex
by vertex on Python sets of out-neighbours of the same orientation.  Every edge
points towards the endpoint of higher (degree, index).  The count is an exact Python int (the library
wraps modulo 2^64; the test inputs stay far below that).
"""
import numpy as np
import scipy.sparse as sp


def simple_edges(n, src, dst):
    """(a, b) with a < b: the unique non-loop pairs of the edge list."""
    s = np.asarray(src, dtype=np.int64)
    d = np.asarray(dst, dtype=np.int64)
    keep = s != d
    a, b = np.minimum(s, d)[keep], np.maximum(s, d)[keep]
    key = np.unique(a * max(n, 1) + b)
    return key // max(n, 1), key % max(n, 1)


def _orient(n, a, b):
    deg = np.bincount(a, minlength=n) + np.bincount(b, minlength=n)
    rank = np.empty(n, dtype=np.int64)
    rank[np.lexsort((np.arange(n), deg))] = np.arange(n)
    low = rank[a] < rank[b]
    return np.where(low, a, b), np.where(low, b, a)


def _triangles(n, lo, hi):
    if len(lo) == 0:
        return 0
    O = sp.csr_matrix((np.ones(len(lo), dtype=np.int64), (lo, hi)), shape=(n, n))
    return int((O @ O).multiply(O).sum())


def _count(cand, r, out):
    """r-cliques inside cand, each listed once through the out-sets."""
    if r == 1:
        return len(cand)
    if len(cand) < r:
        return 0
    return sum(_count(cand & out[w], r - 1, out) for w in cand)


def count(n, src, dst, k):
    """Number of k-cliques (k >= 1) of the simple graph on vertices 0..n-1."""
    if k < 1:
        raise ValueError("k must be >= 1")
    a, b = simple_edges(n, src, dst)
    if k == 1:
        return int(n)
    if k == 2:
        return int(len(a))
    lo, hi = _orient(n, a, b)
    if k == 3:
        return _triangles(n, lo, hi)
    out = [set() for _ in range(n)]
    for u, v in zip(lo.tolist(), hi.tolist()):
        out[u].add(v)
    return sum(_count(out[v], k - 1, out) for v in range(n) if len(out[v]) >= k - 1)


def clique_number(n, src, dst, cap=None):
    """Largest k with a k-clique (0 for no vertex), searched up to cap."""
    k = 0
    while (cap is None or k < cap) and count(n, src, dst, k + 1) > 0:
        k += 1
    return k
