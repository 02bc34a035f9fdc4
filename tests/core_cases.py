"""Inputs on which core decomposition / k-core are compared with the reference
CPU apps (digests in tests/golden/ref_core_outputs.json, written by
golden/make_ref_core_fixtures.py).  Each case: (n, src, dst, oids or None, k
values for kcore besides max core and max core + 1); src / dst are oids when
oids is given, vertex indices otherwise."""
import json
import os

import numpy as np

from tests import shapes as S
from tests.golden_io import GOLDEN, load_p2p31
from tests.util import rmat_graph

# the threshold graphs of tests/shapes.py the core apps run on
SHAPES = {
    "empty1": S.empty(1), "empty1025": S.empty(1025),
    "star1023": S.star(1023), "star1025_last": S.star(1025, centre_last=True), "star70000": S.star(70000),
    "hub33": S.hub_block(33), "hub64": S.hub_block(64), "path300": S.path(300),
    "clique40": S.clique(40), "ring_lattice": S.ring_lattice(5000, 7), "bipartite": S.complete_bipartite(30, 2000),
    "multi_loop": S.multi_loop(), "chorded": S.chorded_ring(45057, seed=3),
    "pad65537": S.pad_to(S.path(1000), 65537),
    "union": S.union([S.star(2000), S.clique(20), S.path(50), S.empty(7), S.hub_block(40)], seed=5),
}


def random_multigraph(seed):
    """Up to 40 vertices, multi-edges and self loops."""
    rng = np.random.RandomState(seed)
    n = int(rng.randint(1, 40))
    m = int(rng.randint(0, 4 * n + 1))
    src = rng.randint(0, n, size=m)
    dst = rng.randint(0, n, size=m)
    k = m // 4
    src = np.concatenate([src, src[:k], rng.randint(0, n, size=3)])
    dst = np.concatenate([dst, dst[:k], src[-3:]])
    return n, src.astype(np.int64), dst.astype(np.int64)


def core_cases(big=True):
    """name -> (n, src, dst, oids, ks).  big=False leaves out R-MAT scale 20."""
    cases = {}
    oids, s, d, _ = load_p2p31()
    cases["p2p31"] = (len(oids), s, d, oids, [0, 3, 6, 7])
    n, s, d, _ = rmat_graph(12, seed=21)
    cases["rmat12"] = (n, s, d, None, [0, 2, 16])
    for seed in range(8):
        n, s, d = random_multigraph(seed)
        cases["random%d" % seed] = (n, s, d, None, [0, 1, 2, 3])
    for name, (n, s, d, _) in SHAPES.items():
        cases["shape_" + name] = (n, s, d, None, [0, 1, 2])
    if big:
        n, s, d, _ = rmat_graph(20, seed=1)
        cases["rmat20"] = (n, s, d, None, [16])
    return cases


def as_indices(n, src, dst, oids):
    """Vertex indices in ascending-oid order (what the oracle and the fragment use)."""
    if oids is None:
        return src, dst
    o = np.sort(np.asarray(oids, dtype=np.int64))
    return np.searchsorted(o, src), np.searchsorted(o, dst)


def ref_core_outputs():
    """name -> {"core": digest, "max_core": int, "kcore": {k: digest}} of the reference apps."""
    with open(os.path.join(GOLDEN, "ref_core_outputs.json")) as f:
        return json.load(f)
