"""Inputs on which k-clique counting is compared with the reference CPU app
(counts in tests/golden/ref_kclique_outputs.json, written by
golden/make_ref_kclique_fixtures.py from the reference run on the simplified
input).  Each case: (n, src, dst, oids or None); src / dst are oids when oids is
given, vertex indices otherwise.

Besides p2p-31, R-MAT, the random multigraphs and the threshold graphs of
tests/core_cases.py, the threshold graphs here put the candidate set
I = N+(v) ∩ N+(u) of one oriented edge (v, u) exactly at and one above each
tier limit of csrc/app_kclique.cu, and one graph leaves the first fragments of
a 2- or 3-fragment cut without any vertex of a clique."""
import json
import os

import numpy as np
import scipy.sparse as sp

from tests import shapes as S
from tests.core_cases import SHAPES, random_multigraph
from tests.golden_io import GOLDEN, load_p2p31
from tests.util import rmat_graph

# the kernel's tier limits (kKcWarpMax, kKcCtaMax) and its largest k (GL_KCLIQUE_MAX_K)
WARP_MAX = 32
CTA_MAX = 1024
MAX_K = 32


def common_block(m):
    """D (m vertices) x C (m vertices) complete bipartite, a ring lattice with two neighbours on each
    side on C, and an edge (u, v) whose endpoints are joined to all of C.  Degrees: D m, u and v m + 1,
    C m + 6, so the oriented edge u -> v has the candidate set C (s = m); every other edge has s <= 4.
    The clique number is 5 (u, v and a triangle of the ring lattice)."""
    D = np.arange(m)
    C = np.arange(m, 2 * m)
    u, v = 2 * m, 2 * m + 1
    s = [np.repeat(D, m), C, C, np.full(m, u), np.full(m, v), [u]]
    d = [np.tile(C, m), m + (D + 1) % m, m + (D + 2) % m, C, C, [v]]
    return S._out(2 * m + 2, np.concatenate(s).astype(np.int64), np.concatenate(d).astype(np.int64))


def nested_block(m=CTA_MAX + 76, path=10):
    """An edge (u, v) whose candidate set C (m > CTA_MAX vertices) holds a vertex w0 whose own
    out-neighbours inside C are the other m - 1 > CTA_MAX members: from k = 5 on the list tier pushes a
    second list above the limit.  ids: u = 0, v = 1, w0 = 2, C' = 3 .. m + 1, P = the next m vertices.
    u, v and w0 are joined to each other and to all of C'; P x C' is complete bipartite and a path joins
    the first `path` members of C'.  Degrees: P m - 1, u, v and w0 m + 1 (ties broken by id), C' at
    least m + 3."""
    Cp = np.arange(3, m + 2)
    P = np.arange(m + 2, 2 * m + 2)
    s = [[0, 0, 1], np.zeros(m - 1), np.ones(m - 1), np.full(m - 1, 2), np.repeat(P, m - 1), Cp[:path - 1]]
    d = [[1, 2, 2], Cp, Cp, Cp, np.tile(Cp, m), Cp[1:path]]
    return S._out(2 * m + 2, np.concatenate(s).astype(np.int64), np.concatenate(d).astype(np.int64))


def clique_in_last_block(n=300, k=10):
    """A path over the first two thirds of the ids and a k-clique on the last k: with 2 or 3 contiguous
    fragments the first ones own no vertex of any triangle."""
    p = np.arange(2 * n // 3 - 1)
    i, j = np.triu_indices(k, 1)
    return S._out(n, np.concatenate([p, n - k + i]), np.concatenate([p + 1, n - k + j]))


THRESHOLDS = {
    "clique34": S.clique(WARP_MAX + 2), "clique35": S.clique(WARP_MAX + 3),
    "block32": common_block(WARP_MAX), "block33": common_block(WARP_MAX + 1),
    "block1024": common_block(CTA_MAX), "block1025": common_block(CTA_MAX + 1), "nested1100": nested_block(),
    "last_block": clique_in_last_block(),
}


# cases whose k also runs over 3 .. the given value, so that every depth-first stack pushes: a clique of
# 34 (warp tier) and of 35 vertices (one edge in the CTA bitmap tier) at k = 6 .. 8
K_UP_TO = {"tier_clique34": 8, "tier_clique35": 8}


def kclique_cases(big=True):
    """name -> (n, src, dst, oids).  big=False leaves out R-MAT scale 16."""
    cases = {}
    oids, s, d, _ = load_p2p31()
    cases["p2p31"] = (len(oids), s, d, oids)
    n, s, d, _ = rmat_graph(12, seed=1)
    cases["rmat12"] = (n, s, d, None)
    if big:
        n, s, d, _ = rmat_graph(16, seed=1)
        cases["rmat16"] = (n, s, d, None)
    for seed in range(8):
        n, s, d = random_multigraph(seed)
        cases["random%d" % seed] = (n, s, d, None)
    for name, (n, s, d, _) in SHAPES.items():
        cases["shape_" + name] = (n, s, d, None)
    for name, (n, s, d, _) in THRESHOLDS.items():
        cases["tier_" + name] = (n, s, d, None)
    return cases


def ks_for(omega):
    """k = 3, 4, 5 and, on graphs whose clique number is small, every k up to omega + 1 (count 0)."""
    top = omega + 1 if omega + 1 <= 9 else 5
    return sorted(set([3, 4, 5]) | set(range(3, top + 1)))


def as_indices(n, src, dst, oids):
    """Vertex indices in ascending-oid order (what the oracle and the fragment use)."""
    if oids is None:
        return np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    o = np.sort(np.asarray(oids, dtype=np.int64))
    return np.searchsorted(o, src), np.searchsorted(o, dst)


def candidate_sizes(n, src, dst):
    """s = |N+(v) ∩ N+(u)| of every oriented edge (v, u) by the kernel's rule: simple edges oriented from
    the lower to the higher (CSR row length, vertex index) on one fragment."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    deg = np.bincount(src, minlength=n) + np.bincount(dst, minlength=n)   # a self loop is two entries
    keep = src != dst
    a, b = np.minimum(src, dst)[keep], np.maximum(src, dst)[keep]
    key = np.unique(a * max(n, 1) + b)
    a, b = key // max(n, 1), key % max(n, 1)
    a_low = (deg[a] < deg[b]) | ((deg[a] == deg[b]) & (a < b))
    lo, hi = np.where(a_low, a, b), np.where(a_low, b, a)
    O = sp.csr_matrix((np.ones(len(lo), dtype=np.int64), (lo, hi)), shape=(n, n))
    common = (O @ O.T).tocsr()
    return np.asarray(common[lo, hi]).ravel().astype(np.int64)


def tier_items(s, k):
    """(largest s, items of the warp, CTA bitmap and CTA list tiers) for k >= 4."""
    s = np.asarray(s, dtype=np.int64)
    live = s >= k - 2
    return (int(s.max()) if len(s) else 0, int(np.sum(live & (s <= WARP_MAX))),
            int(np.sum(live & (s > WARP_MAX) & (s <= CTA_MAX))), int(np.sum(live & (s > CTA_MAX))))


def ref_kclique_outputs():
    """name -> {k: count} of the reference app on the simplified input."""
    with open(os.path.join(GOLDEN, "ref_kclique_outputs.json")) as f:
        return {name: {int(k): int(c) for k, c in v.items()} for name, v in json.load(f).items()}
