"""Small graphs for GL_APP_PAGERANK_VC: each returns (n, src, dst) with vertices 0..n-1."""
import numpy as np


def pagerank_vc_cases():
    rng = np.random.default_rng(12)
    cases = {}
    # self loops (counted twice in the degree) and duplicate edges
    cases["loops_dups"] = (6, [0, 0, 1, 1, 1, 2, 3, 3, 5], [0, 1, 2, 2, 1, 3, 4, 4, 5])
    # no edge at all: every vertex is dangling
    cases["all_dangling"] = (7, [], [])
    # fewer vertices than fragments at F = 9 and 4: tail fragments own no masters
    cases["n_below_f"] = (3, [0, 1, 2], [1, 2, 2])
    # n not divisible by 4 or 9, random multigraph with isolated vertices
    n = 103
    s = rng.integers(0, n - 5, 400)
    d = rng.integers(0, n - 5, 400)
    cases["n_103"] = (n, s.tolist(), d.tolist())
    # a star whose hub row spans several 4096-entry chunks, plus a ring over the leaves
    n = 9000
    leaves = np.arange(1, n)
    src = np.concatenate([np.zeros(n - 1, dtype=np.int64), leaves])
    dst = np.concatenate([leaves, np.roll(leaves, 1)])
    cases["star_9000"] = (n, src.tolist(), dst.tolist())
    # a row between the one-thread and the chunked tiers (33..4096 entries)
    n = 700
    src = np.concatenate([np.full(600, 5), rng.integers(0, n, 300)])
    dst = np.concatenate([rng.integers(0, n, 600), rng.integers(0, n, 300)])
    cases["mid_row"] = (n, src.tolist(), dst.tolist())
    return {k: (n, np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64)) for k, (n, s, d) in cases.items()}


# The fixtures of the reference's PageRankVC (tests/golden/ref_pagerank_vc_outputs.{json,npz}, written by
# tests/golden/make_ref_pagerank_vc_fixtures.py): every case above plus p2p-31 and R-MAT 12, at these
# rounds, damping factors and fragment counts.  For the two large graphs the fixtures keep the values of
# SAMPLE vertices (and the sum over all), to stay small.
REF_ROUNDS = (0, 1, 10)
REF_DELTAS = (0.85, 0.5)
REF_FNUMS = (1, 4, 9)
LARGE = ("p2p31", "rmat12")
SAMPLE = 1024


def ref_cases():
    """The fixture inputs: pagerank_vc_cases() plus p2p-31 (the dataset's ids start at 1, so with
    n = max id + 1 oid 0 is an isolated vertex) and R-MAT 12 (edge factor 16, seed 7)."""
    from tests import golden_io as G
    cases = pagerank_vc_cases()
    oids, s, d, _ = G.load_p2p31()
    cases["p2p31"] = (int(oids.max()) + 1, s, d)
    from tests.util import pkg
    s12, d12, _ = pkg().rmat_edges_host(12, 16, seed=7)
    cases["rmat12"] = (1 << 12, s12, d12)
    return cases


def sample_index(n):
    """The vertices a large case keeps: oid 0, then SAMPLE - 1 evenly spaced ids."""
    if n <= SAMPLE:
        return np.arange(n)
    return np.unique(np.concatenate([[0], np.linspace(0, n - 1, SAMPLE - 1).astype(np.int64)]))


def ref_key(name, R, delta, fnum):
    return "%s|R%d|d%g|F%d" % (name, R, delta, fnum)


def ref_pagerank_vc_outputs():
    """(meta, arrays): meta = the JSON file (sums, the runs the reference aborted), arrays = the npz."""
    import json
    import os
    from tests import golden_io as G
    meta = json.load(open(os.path.join(G.GOLDEN, "ref_pagerank_vc_outputs.json")))
    arrays = dict(np.load(os.path.join(G.GOLDEN, "ref_pagerank_vc_outputs.npz")))
    return meta, arrays
