"""CPU checks of oracle/pagerank_vc_oracle.py: the scipy definition against a dense restatement,
closed forms, the edge-cut PageRank oracle, and the statistics model's per-fragment shares."""
import numpy as np
import pytest

from oracle import pagerank_vc_oracle as V
from tests.pagerank_vc_cases import pagerank_vc_cases


def dense(n, src, dst, delta, R):
    """Loop-by-loop restatement of pagerank_vc.h on a dense matrix."""
    if R <= 0:
        return np.zeros(n)
    W = np.zeros((n, n))
    deg = np.zeros(n)
    for a, b in zip(src, dst):
        W[a, b] += 1
        W[b, a] += 1
        deg[a] += 1
        deg[b] += 1
    D = int((deg == 0).sum())
    p = 1.0 / n
    mr = np.array([p if deg[v] == 0 else p / deg[v] for v in range(n)])
    ds = p * D
    for k in range(1, R + 1):
        base = (1 - delta) / n + delta * ds / n
        ds = base * D
        s = W @ mr
        if k == R:
            return s * delta + base
        mr = np.array([base if deg[v] == 0 else (base + delta * s[v]) / deg[v] for v in range(n)])


CASES = pagerank_vc_cases()


@pytest.mark.parametrize("name", sorted(k for k in CASES if CASES[k][0] <= 1000))
@pytest.mark.parametrize("R", [0, 1, 10])
@pytest.mark.parametrize("delta", [0.85, 0.5])
def test_oracle_matches_dense_restatement(name, R, delta):
    n, s, d = CASES[name]
    np.testing.assert_allclose(V.pagerank_vc(n, s, d, delta, R), dense(n, s, d, delta, R), rtol=1e-12, atol=0)


def test_closed_forms():
    # cycle: every vertex has degree 2, the uniform vector is a fixed point
    n = 11
    s = np.arange(n)
    got = V.pagerank_vc(n, s, (s + 1) % n, 0.85, 10)
    np.testing.assert_allclose(got, np.full(n, 1.0 / n), rtol=1e-14)
    # only isolated vertices: base = 1/n every round
    np.testing.assert_allclose(V.pagerank_vc(5, [], [], 0.85, 7), np.full(5, 0.2), rtol=1e-14)
    # star with k leaves, one round: hub = d * k * (1/n) / 1 + base; leaf = d * (1/n) / k + base
    k = 6
    n = k + 1
    got = V.pagerank_vc(n, np.zeros(k, dtype=np.int64), np.arange(1, n), 0.85, 1)
    base = 0.15 / n
    np.testing.assert_allclose(got[0], 0.85 * k * (1.0 / n) + base, rtol=1e-14)
    np.testing.assert_allclose(got[1:], 0.85 * (1.0 / n / k) + base, rtol=1e-14)
    # R <= 0: nothing runs
    assert not V.pagerank_vc(4, [0], [1], 0.85, -3).any()


@pytest.mark.parametrize("name", ["loops_dups", "n_103", "mid_row"])
@pytest.mark.parametrize("R", [1, 10])
def test_equals_edge_cut_pagerank_oracle(name, R):
    """GL_APP_PAGERANK's oracle on the undirected edge-cut graph counts rounds the same way."""
    from oracle import pyoracle
    n, s, d = CASES[name]
    g = pyoracle.Graph(n, s, d, directed=False)
    np.testing.assert_allclose(V.pagerank_vc(n, s, d, 0.85, R), g.pagerank(0.85, R), rtol=1e-12)


@pytest.mark.parametrize("fnum", [1, 4, 9, 16])
def test_partition_covers_every_vertex_and_edge(fnum):
    n, s, d = CASES["n_103"]
    parts = V.partition(n, fnum)
    masters = np.concatenate([np.arange(*p["master"]) for p in parts])
    assert np.array_equal(masters, np.arange(n))
    for p in parts:
        assert p["src"][0] <= p["master"][0] and p["master"][1] <= max(p["src"][1], p["master"][0])
    blk = V.block_of(n, fnum, s, d)
    for p, f in zip(parts, range(fnum)):
        mine = blk == f
        assert np.all((s[mine] >= p["src"][0]) & (s[mine] < p["src"][1]))
        assert np.all((d[mine] >= p["dst"][0]) & (d[mine] < p["dst"][1]))


@pytest.mark.parametrize("fnum", [4, 9])
@pytest.mark.parametrize("name", sorted(CASES))
def test_stats_shares_add_up(fnum, name):
    n, s, d = CASES[name]
    one = V.stats(n, s, d, 1, 10)[0]
    many = V.stats(n, s, d, fnum, 10)
    assert sum(x["entries_scanned"] for x in many) == one["entries_scanned"] == 20 * len(s)
    assert sum(x["touched_vertices"] for x in many) == one["touched_vertices"] == 10 * n
    assert sum(x["masters"] for x in many) == n
    assert one["msg_bytes_sent"] == 0
    # every byte a fragment scatters is one a holder receives; every gathered byte reaches an owner
    side = int(round(fnum ** 0.5))
    parts = V.partition(n, fnum)
    sent = sum(x["msg_bytes_sent"] for x in many)
    pairs = sum(8 * (q["master"][1] - q["master"][0])
                for q in parts for f in range(fnum)
                if f != q["fid"] and (f // side == q["fid"] // side or f % side == q["fid"] // side))
    assert sent == 11 * pairs + 10 * pairs
