"""Inputs and the f64 oracle of directed PageRank (GL_APP_PAGERANK_DIRECTED, the LDBC Graphalytics
directed PageRank, the reference's PageRankDirected).

Each case: (n, src, dst), vertex indices 0..n-1, directed edges.
  mixed        sinks with in-edges, isolated vertices, a vertex whose only out-edge is a self loop,
               duplicate edges and a 2-cycle;
  no_edges     every vertex dangling;  single / single_loop  one vertex, without and with a self loop;
  tier_rows    in-rows of exactly 32 and 33 entries (the one-thread / warp cut of csrc/row_tiers.cuh)
               and of kTierChunk and kTierChunk + 1 entries (the warp / chunk cut);
  long_rows    an in-row longer than two chunks and a source whose out-row is longer than a chunk;
  random       a sparse random multigraph with self loops;
  p2p31        dataset/p2p-31 (in index space: position in the ascending oid list), 46 199 of its
               62 586 vertices are sinks with in-edges.

The oracle follows the semantics block of GL_APP_PAGERANK_DIRECTED in include/grape_b200.h.  Fixtures of
the reference's own PageRankDirected (tests/golden/ref_pagerank_directed_outputs.{json,npz}) are written by
tests/golden/make_ref_pagerank_directed_fixtures.py."""
import json
import os

import numpy as np

from tests.golden_io import GOLDEN

CHUNK = 4096                   # csrc/row_tiers.cuh kTierChunk
DELTAS = (0.85, 0.5, 0.0, 1.0)
ROUNDS = (0, 1, 2, 10)
REF_DELTAS = (0.85, 0.5)       # the fixtures: every case at these d and ROUNDS, p2p-31 at (0.85, 10)
P2P = ("p2p31", 0.85, 10)


def _case(n, s, d):
    return n, np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64)


def mixed():
    """0 -> 1 twice; 1 <-> 2; 3 -> 3 only; 0 -> 4 and 5 -> 4 (4 a sink); 2 -> 5; 8 -> 9 (9 a sink);
    6 and 7 isolated."""
    s = [0, 0, 1, 2, 3, 0, 5, 2, 8]
    d = [1, 1, 2, 1, 3, 4, 4, 5, 9]
    return _case(10, s, d)


def tier_rows(seed=3):
    """Targets 0..3 with in-rows of 32, 33, CHUNK and CHUNK + 1 entries, drawn with repetition from
    sources 10..299, which also carry a random multigraph of their own; 4 is a sink fed by all of them."""
    rng = np.random.default_rng(seed)
    n = 300
    srcs, dsts = [rng.integers(10, n, 1500)], [rng.integers(5, n, 1500)]
    for t, k in enumerate((32, 33, CHUNK, CHUNK + 1)):
        srcs.append(rng.integers(10, n, k))
        dsts.append(np.full(k, t))
    srcs.append(np.arange(10, n))
    dsts.append(np.full(n - 10, 4))
    return _case(n, np.concatenate(srcs), np.concatenate(dsts))


def long_rows(seed=4):
    """Vertex 0's in-row holds 2 * CHUNK + 808 entries; vertex 1's out-row holds CHUNK + 904 entries
    (its share of rank is divided over that many edges)."""
    rng = np.random.default_rng(seed)
    n = 200
    k0, k1 = 2 * CHUNK + 808, CHUNK + 904
    s = np.concatenate([rng.integers(2, n, k0), np.ones(k1, np.int64), rng.integers(0, n, 600)])
    d = np.concatenate([np.zeros(k0, np.int64), rng.integers(0, n, k1), rng.integers(2, n, 600)])
    return _case(n, s, d)


def random_graph(seed=5):
    rng = np.random.default_rng(seed)
    n = 150
    return _case(n, rng.integers(0, n, 300), rng.integers(0, n - 20, 300))


def p2p31():
    from tests import golden_io as G
    oids, src, dst, _ = G.load_p2p31()
    return _case(len(oids), np.searchsorted(oids, src), np.searchsorted(oids, dst))


def pagerank_directed_cases(with_p2p=True):
    """name -> (n, src, dst)."""
    cases = {"mixed": mixed(), "no_edges": _case(7, [], []), "single": _case(1, [], []),
             "single_loop": _case(1, [0], [0]), "tier_rows": tier_rows(), "long_rows": long_rows(),
             "random": random_graph()}
    if with_p2p:
        cases["p2p31"] = p2p31()
    return cases


def pagerank_directed(n, s, d, delta, rounds):
    """The definition in numpy f64: one value per vertex index."""
    s = np.asarray(s, dtype=np.int64)
    d = np.asarray(d, dtype=np.int64)
    if rounds <= 0:
        return np.zeros(n)
    deg = np.bincount(s, minlength=n).astype(np.float64)
    dang = deg == 0
    safe = np.where(dang, 1.0, deg)
    p = 1.0 / n
    x = np.where(dang, p, p / safe)
    S = p * float(dang.sum())
    for k in range(1, rounds + 1):
        base = (1.0 - delta) / n + delta * S / n
        c = delta * np.bincount(d, weights=x[s], minlength=n) + base
        x = np.where(dang, c, c / safe)
        if k < rounds:
            S = float(c[dang].sum())
    return np.where(dang, x, x * deg)


def plain_loop(n, s, d, delta, rounds):
    """The same definition one vertex and one edge at a time, as the reference's PEval / IncEval read."""
    res = [0.0] * n
    if rounds <= 0:
        return np.array(res)
    out_deg = [0] * n
    in_rows = [[] for _ in range(n)]
    for a, b in zip(np.asarray(s).tolist(), np.asarray(d).tolist()):
        out_deg[a] += 1
        in_rows[b].append(a)
    p = 1.0 / n
    x = [p / out_deg[v] if out_deg[v] else p for v in range(n)]
    S = p * sum(1 for v in range(n) if out_deg[v] == 0)
    for k in range(1, rounds + 1):
        base = (1.0 - delta) / n + delta * S / n
        nx, S_next = [0.0] * n, 0.0
        for v in range(n):
            cur = 0.0
            for w in in_rows[v]:
                cur += x[w]
            cur = delta * cur + base
            if out_deg[v] == 0:
                nx[v] = cur
                S_next += cur
            else:
                nx[v] = cur / out_deg[v]
        x = nx
        if k < rounds:
            S = S_next
    return np.array([x[v] * out_deg[v] if out_deg[v] else x[v] for v in range(n)])


def ref_key(name, delta, rounds):
    return "%s|d%g|R%d" % (name, delta, rounds)


def ref_runs():
    """(name, delta, rounds) of every fixture run."""
    runs = [(name, dl, r) for name in sorted(pagerank_directed_cases(with_p2p=False))
            for dl in REF_DELTAS for r in ROUNDS]
    return runs + [P2P]


def ref_pagerank_directed_outputs():
    """(meta, arrays): meta = the JSON file (the sum of every run), arrays = the npz (values in index
    order)."""
    meta = json.load(open(os.path.join(GOLDEN, "ref_pagerank_directed_outputs.json")))
    arrays = dict(np.load(os.path.join(GOLDEN, "ref_pagerank_directed_outputs.npz")))
    return meta, arrays


# the reference's PageRankDirected (run_app_opt --application pagerank --directed) through
# oracle/_ref/ref_pagerank_directed_driver, built by __graft_entry__.build() from oracle/ref/pagerank_directed.mk
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_EXE = os.path.join(ROOT, "oracle", "_ref", "ref_pagerank_directed_driver")


def run_ref(n, s, d, delta, rounds, threads=1):
    """The reference's output in vertex-index order (float64)."""
    import subprocess
    import tempfile
    from oracle import refdriver
    with tempfile.TemporaryDirectory() as tmp:
        g, out = os.path.join(tmp, "g.bin"), os.path.join(tmp, "out.txt")
        refdriver.write_graph(g, n, s, d)
        cmd = [REF_EXE, "--graph", g, "--pr_d", repr(float(delta)), "--mr", str(int(rounds)),
               "--threads", str(int(threads)), "--out", out]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
        if p.returncode != 0:
            raise RuntimeError("ref_pagerank_directed_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
        oids, vals = refdriver.parse_output(open(out).read())
    assert np.array_equal(oids, np.arange(n))
    return vals
