"""Inputs on which the directed local clustering coefficient (GL_APP_LCC_DIRECTED) is compared with
the reference's LCCDirected (digests of its tri and deduplicated-degree arrays in
tests/golden/ref_lcc_directed_outputs.json, written by golden/make_ref_lcc_directed_fixtures.py) and
with the oracle (oracle/lcc_directed_oracle.py).

Each case: (n, src, dst, oids or None); src / dst are oids when oids is given, vertex indices
otherwise.  Edges are directed.  The cases reach: self loops and duplicates (R-MAT), pairs joined in
both directions (reciprocal, multigraphs), in- and out-rows longer than the kernel's warp and CTA row
cuts (the stars), a graph where every degree ties (clique), a vertex with only in-edges, isolated
vertices, no edges at all, and pairs with 255, 256 and 300 parallel entries, where the reference's
uint8_t weights wrap (256 -> 0, 300 -> 44)."""
import json
import os

import numpy as np

from tests import directed_cases as D
from tests import golden_io as G
from tests import shapes as S
from tests.golden_io import GOLDEN

# the uint8_t weight of lcc_directed.h:205 wraps from this many entries per pair on
WRAP = 256


def multigraph(n, m, seed):
    """m random directed edges over n vertices, with repeated pairs, reversed pairs and self loops."""
    rng = np.random.default_rng([seed, n, m])
    s = rng.integers(0, n, m)
    d = rng.integers(0, n, m)
    k = m // 4    # a quarter of the edges again, a quarter reversed
    return n, np.concatenate([s, s[:k], d[k:2 * k]]), np.concatenate([d, d[:k], s[k:2 * k]])


def reciprocal(n, p, seed):
    """A simple undirected random graph, every edge in both directions and no self loop."""
    rng = np.random.default_rng([seed, n])
    i, j = np.triu_indices(n, 1)
    keep = rng.random(len(i)) < p
    i, j = i[keep], j[keep]
    return n, np.concatenate([i, j]), np.concatenate([j, i])


def parallel_pair(copies):
    """Triangle 0, 1, 2 plus vertex 3 joined to 0 and 1; the pair {0, 1} has `copies` entries, split over
    both directions (0 -> 1 gets the larger half)."""
    a = (copies + 1) // 2
    s = [0] * a + [1] * (copies - a) + [1, 2, 3, 1]
    d = [1] * a + [0] * (copies - a) + [2, 0, 0, 3]
    return 4, np.array(s, dtype=np.int64), np.array(d, dtype=np.int64)


def only_in():
    """Vertex 0 has only in-edges, from a ring 1 .. 40 whose neighbours also point at each other."""
    v = np.arange(1, 41)
    nxt = np.where(v == 40, 1, v + 1)
    return 41, np.concatenate([v, v]), np.concatenate([np.zeros(40, np.int64), nxt])


def star_ring(k, inward):
    """Centre 0 with an edge to (outward) or from (inward) each of the leaves 1 .. k, and a ring of edges
    i -> i + 1 among the leaves: the centre's merged row has k entries, with a triangle on every ring
    edge."""
    n, s, d, _ = (S.sink_heavy if inward else S.source_heavy)(k)
    v = np.arange(1, k + 1)
    return n, np.concatenate([s, v]), np.concatenate([d, np.where(v == k, 1, v + 1)])


def _strip(shape):
    n, s, d = shape[:3]
    return n, np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64), None


def lcc_directed_cases():
    """name -> (n, src, dst, oids or None)."""
    oids, src, dst, _ = G.load_p2p31()
    cases = {"p2p31": (len(oids), src, dst, oids)}
    for name in ("rmat12", "rmat14"):
        cases[name] = _strip(D.build(name))
    for seed in (1, 2):
        cases["multigraph%d" % seed] = _strip(multigraph(300, 3000, seed))
    cases["reciprocal"] = _strip(reciprocal(120, 0.1, 3))
    cases["in_star4097"] = _strip(star_ring(4097, True))
    cases["out_star4097"] = _strip(star_ring(4097, False))
    cases["clique40"] = _strip(S.clique(40))
    cases["only_in"] = _strip(only_in())
    cases["isolated"] = _strip(S.pad_to(S.path(50), 200))
    cases["empty"] = _strip(S.empty(33))
    for c in (255, 256, 300):
        cases["pair%d" % c] = _strip(parallel_pair(c))
    return cases


def as_indices(n, src, dst, oids):
    """src / dst as vertex indices (positions in the ascending oid list)."""
    if oids is None:
        return np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    o = np.sort(np.asarray(oids, dtype=np.int64))
    return np.searchsorted(o, src), np.searchsorted(o, dst)


def ref_lcc_directed_outputs():
    """name -> {"tri", "d": digests, "tri_sum": int} of the reference app's run."""
    with open(os.path.join(GOLDEN, "ref_lcc_directed_outputs.json")) as f:
        return json.load(f)
