"""Inputs and the f64 oracle of un-normalised PageRank (GL_APP_PAGERANK_LOCAL, the reference's
PageRankLocal, run_app --application pagerank_local).

Each case: (n, src, dst), vertex indices 0..n-1.  Every case runs on an undirected fragment (each edge
in both rows, a self loop twice in its row) and on a directed one (the out-rows only).
  mixed        isolated vertices (6, 7), a vertex whose only edge is a self loop (3), a vertex with a
               self loop and other edges (5), a duplicate edge (0 -> 1 twice) and, directed, sinks that
               are someone's out-neighbour (4, 9: their undivided x is read);
  empty        seven vertices, no edges;  single / single_loop  one vertex, without and with a self loop;
  tier_rows    out-rows of exactly 32 and 33 entries (the one-thread / warp cut of csrc/row_tiers.cuh)
               and of kTierChunk and kTierChunk + 1 entries (the warp / chunk cut), in a graph sparse
               enough that the reference's one-fragment run takes its dividing branch;
  long_rows    an out-row longer than two chunks and one longer than a chunk;
  random       a sparse random multigraph with self loops;
  dense        average degree above 10 on one fragment (the reference's non-dividing branch there);
  p2p31        dataset/p2p-31 (in index space: position in the ascending oid list).

The oracle follows the semantics block of GL_APP_PAGERANK_LOCAL in include/grape_b200.h.  Fixtures of
the reference's own PageRankLocal (tests/golden/ref_pagerank_local_outputs.{json,npz}) are written by
tests/golden/make_ref_pagerank_local_fixtures.py."""
import json
import os

import numpy as np

from tests.golden_io import GOLDEN

CHUNK = 4096                   # csrc/row_tiers.cuh kTierChunk
DELTAS = (0.85, 0.5, 0.0, 1.0)
ROUNDS = (1, 2, 10)
DIRS = ("undirected", "directed")
REF_DELTAS = (0.85, 0.5)       # the fixtures: these d x ROUNDS, on 1 rank where avg_degree <= 10 and on
REF_RANKS = (1, 2, 3)          # 2 and 3 ranks for every case but p2p31
P2P = (0.85, 10)               # p2p31 (both directions, 1 rank)
DENSE = ("dense", 0.85, 10)    # the one 1-rank run with avg_degree > 10 (both directions)


def _case(n, s, d):
    return n, np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64)


def mixed():
    """0 -> 1 twice; 1 <-> 2; 3 -> 3 only; 0 -> 4 and 5 -> 4 (4 a sink); 2 -> 5; 5 -> 5; 8 -> 9 (9 a
    sink); 6 and 7 isolated."""
    s = [0, 0, 1, 2, 3, 0, 5, 2, 5, 8]
    d = [1, 1, 2, 1, 3, 4, 4, 5, 5, 9]
    return _case(10, s, d)


def _padded(n_active, s, d, n):
    """Vertices n_active..n-1 added, mostly isolated, so that one fragment's avg_degree stays at most 10:
    10 of them spread over the range, each fed by an active vertex and chained both ways, the last one
    back to vertex 10, link every ordered pair of fragments at 2 and 3 ranks."""
    hops = n_active + (n - n_active) // 10 * np.arange(10, dtype=np.int64)
    s = np.concatenate([s, np.arange(10, 20), hops[:-1], hops[1:], hops[-1:]])
    d = np.concatenate([d, hops, hops[1:], hops[:-1], [10]])
    return _case(n, s, d)


def tier_rows(seed=3):
    """Sources 0..3 with out-rows of 32, 33, CHUNK and CHUNK + 1 entries, drawn with repetition from
    targets 10..299, which also carry a random multigraph of their own; padded to 2400 vertices."""
    rng = np.random.default_rng(seed)
    n = 300
    srcs, dsts = [rng.integers(10, n, 1500)], [rng.integers(10, n, 1500)]
    for t, k in enumerate((32, 33, CHUNK, CHUNK + 1)):
        srcs.append(np.full(k, t))
        dsts.append(rng.integers(10, n, k))
    return _padded(n, np.concatenate(srcs), np.concatenate(dsts), 2400)


def long_rows(seed=4):
    """Vertex 0's out-row holds 2 * CHUNK + 808 entries, vertex 1's CHUNK + 904; padded to 3200
    vertices."""
    rng = np.random.default_rng(seed)
    n = 200
    k0, k1 = 2 * CHUNK + 808, CHUNK + 904
    s = np.concatenate([np.zeros(k0, np.int64), np.ones(k1, np.int64), rng.integers(2, n, 600)])
    d = np.concatenate([rng.integers(2, n, k0), rng.integers(2, n, k1), rng.integers(0, n, 600)])
    return _padded(n, s, d, 3200)


def random_graph(seed=5):
    rng = np.random.default_rng(seed)
    n = 150
    return _case(n, rng.integers(0, n, 300), rng.integers(0, n - 20, 300))


def dense(seed=6):
    rng = np.random.default_rng(seed)
    n = 64
    return _case(n, rng.integers(0, n, 1200), rng.integers(0, n, 1200))


def p2p31():
    from tests import golden_io as G
    oids, src, dst, _ = G.load_p2p31()
    return _case(len(oids), np.searchsorted(oids, src), np.searchsorted(oids, dst))


def pagerank_local_cases(with_p2p=True):
    """name -> (n, src, dst)."""
    cases = {"mixed": mixed(), "empty": _case(7, [], []), "single": _case(1, [], []),
             "single_loop": _case(1, [0], [0]), "tier_rows": tier_rows(), "long_rows": long_rows(),
             "random": random_graph(), "dense": dense()}
    if with_p2p:
        cases["p2p31"] = p2p31()
    return cases


def rows(n, s, d, directed):
    """The out-rows as (row of each entry, column of each entry): directed, the edges; undirected, each
    edge in both rows (a self loop twice in its row)."""
    s = np.asarray(s, dtype=np.int64)
    d = np.asarray(d, dtype=np.int64)
    if directed:
        return s, d
    return np.concatenate([s, d]), np.concatenate([d, s])


def avg_degree(n, s, d, directed):
    """The reference's PageRankLocalContext::avg_degree on one fragment: out-row entries / vertices."""
    return len(rows(n, s, d, directed)[0]) / float(n)


def pagerank_local(n, s, d, delta, rounds, directed, divide=True):
    """The definition in numpy f64: one value per vertex index.  divide=False is the reference's
    one-fragment branch for avg_degree > 10, which never divides by the degree after PEval."""
    assert rounds >= 1
    r, c = rows(n, s, d, directed)
    deg = np.bincount(r, minlength=n).astype(np.float64)
    safe = np.where(deg == 0, 1.0, deg)
    x = 1.0 / safe
    for k in range(1, rounds + 1):
        cur = (1.0 - delta) + delta * np.bincount(r, weights=x[c], minlength=n)
        if k == rounds:
            return cur
        x = cur / safe if divide else cur


def plain_loop(n, s, d, delta, rounds, directed):
    """The same definition one vertex and one row entry at a time, as the reference's PEval / IncEval
    read."""
    r, c = rows(n, s, d, directed)
    out_rows = [[] for _ in range(n)]
    for a, b in zip(r.tolist(), c.tolist()):
        out_rows[a].append(b)
    x = [1.0 / len(out_rows[v]) if out_rows[v] else 1.0 for v in range(n)]
    for k in range(1, rounds + 1):
        nx = [0.0] * n
        for v in range(n):
            cur = 0.0
            for u in out_rows[v]:
                cur += x[u]
            cur = 1 - delta + delta * cur
            nx[v] = cur if k == rounds or not out_rows[v] else cur / len(out_rows[v])
        x = nx
    return np.array(x)


def ref_key(name, directed, delta, rounds, ranks):
    return "%s|%s|d%g|R%d|np%d" % (name, directed, delta, rounds, ranks)


def ref_runs(cases=None):
    """(name, "undirected" | "directed", delta, rounds, ranks) of every fixture run."""
    cases = cases or pagerank_local_cases()
    runs = []
    for name in sorted(cases):
        n, s, d = cases[name]
        for dr in DIRS:
            if name == "p2p31":
                runs.append((name, dr) + P2P + (1,))
                continue
            for ranks in REF_RANKS:
                if ranks == 1 and avg_degree(n, s, d, dr == "directed") > 10:
                    if name == DENSE[0]:
                        runs.append((name, dr) + DENSE[1:] + (1,))
                    continue
                runs += [(name, dr, dl, R, ranks) for dl in REF_DELTAS for R in ROUNDS]
    return runs


def ref_pagerank_local_outputs():
    """(meta, arrays): meta = the JSON file (each recorded run's sum and, on one rank, the reference's
    avg_degree; the runs the reference did not complete), arrays = the npz (values in index order)."""
    meta = json.load(open(os.path.join(GOLDEN, "ref_pagerank_local_outputs.json")))
    arrays = dict(np.load(os.path.join(GOLDEN, "ref_pagerank_local_outputs.npz")))
    return meta, arrays


def segment_owner(n, ranks):
    """The fragment of each vertex under the reference's segment partitioner (ascending oid blocks of
    ceil(n / ranks)) and the library's block partition."""
    chunk = -(-n // ranks)
    return np.arange(n, dtype=np.int64) // max(chunk, 1)


def every_pair_linked(n, s, d, ranks, directed):
    """True when every fragment holds an outer copy of some vertex of every other fragment: an edge
    joins them (directed: an edge from the holder to the owner, the fragment keeps its out-rows
    only).  The reference's BatchShuffleMessageManager
    waits for a message from every peer in UpdatePartialOuterVertices but posts no receive for a peer
    it holds no outer copy of, so PageRankLocal does not complete on several fragments otherwise."""
    if ranks == 1:
        return True
    owner = segment_owner(n, ranks)
    linked = np.zeros((ranks, ranks), dtype=bool)
    a, b = owner[np.asarray(s, dtype=np.int64)], owner[np.asarray(d, dtype=np.int64)]
    linked[a, b] = True
    if not directed:
        linked[b, a] = True
    np.fill_diagonal(linked, True)
    return bool(linked.all())


# the reference's PageRankLocal (run_app --application pagerank_local) through
# oracle/_ref/ref_pagerank_local_driver, built by __graft_entry__.build() from oracle/ref/pagerank_local.mk
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_EXE = os.path.join(ROOT, "oracle", "_ref", "ref_pagerank_local_driver")


def run_ref(n, s, d, delta, rounds, directed, ranks=1, threads=1):
    """-> (the reference's output in vertex-index order (float64), rank 0's avg_degree)."""
    import subprocess
    import tempfile
    from oracle import refdriver
    with tempfile.TemporaryDirectory() as tmp:
        g, out = os.path.join(tmp, "g.bin"), os.path.join(tmp, "out")
        refdriver.write_graph(g, n, s, d)
        cmd = [REF_EXE, "--graph", g, "--directed", "1" if directed else "0", "--pr_d", repr(float(delta)),
               "--mr", str(int(rounds)), "--threads", str(int(threads)), "--out", out]
        env = dict(os.environ, GL_MPI_NP=str(int(ranks)), GL_MPI_TIMEOUT_S="300")
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900, env=env)
        if p.returncode != 0:
            raise RuntimeError("ref_pagerank_local_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
        info = json.loads(p.stdout.strip().splitlines()[-1])
        text = "".join(open("%s.%d" % (out, f)).read() for f in range(int(ranks)))
        oids, vals = refdriver.parse_output(text)
    assert np.array_equal(oids, np.arange(n))
    return vals, info["avg_degree"]
