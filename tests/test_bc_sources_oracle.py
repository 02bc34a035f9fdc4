"""The CPU oracle of betweenness centrality over a list of sources (oracle/bc_sources_oracle.py):
against networkx's exact BC on simple graphs, against a plain per-vertex Brandes loop on multigraphs,
and against the reference app's c summed over each list (tests/golden/ref_bc_sources_outputs.npz, and
the live driver when oracle/_ref is built)."""
from collections import deque

import numpy as np
import pytest

from oracle import bc_oracle as BO
from oracle import bc_sources_oracle as BSO
from oracle import refbc
from tests import shapes as S
from tests.bc_cases import bc_cases, source_index
from tests.bc_sources_cases import ref_bc_sources_outputs, ref_cases
from tests.core_cases import as_indices

CASES = bc_cases()


def graph(n, src, dst, oids):
    """(n, rp, col) on vertex indices in ascending-oid order."""
    s, d = as_indices(n, src, dst, oids)
    rp, col = BO.sorted_csr(n, s, d)
    return rp, col


def brandes(n, rp, col, sources):
    """Per-vertex Brandes with the multigraph rules: every row entry is a path step (a parallel edge counts
    once per copy, a self loop never qualifies), sigma 1 at depth 1, sums in row order, list order fold."""
    bc = [0.0] * n
    for s in sources:
        if s is None:
            continue
        depth = [-1] * n
        depth[s] = 0
        order, q = [s], deque([s])
        while q:
            v = q.popleft()
            for j in range(rp[v], rp[v + 1]):
                w = int(col[j])
                if depth[w] < 0:
                    depth[w] = depth[v] + 1
                    order.append(w)
                    q.append(w)
        sigma = [0.0] * n
        sigma[s] = 1.0
        for v in order[1:]:
            if depth[v] == 1:
                sigma[v] = 1.0
                continue
            acc = 0.0
            for j in range(rp[v], rp[v + 1]):
                if depth[int(col[j])] == depth[v] - 1:
                    acc += sigma[int(col[j])]
            sigma[v] = acc
        t = [0.0] * n
        for v in reversed(order[1:]):
            acc = 0.0
            for j in range(rp[v], rp[v + 1]):
                if depth[int(col[j])] == depth[v] + 1:
                    acc += t[int(col[j])]
            dl = acc * sigma[v]
            t[v] = (1.0 / sigma[v]) * (1.0 + dl)
            bc[v] += dl
    return np.array(bc)


def simple_graphs():
    out = {}
    for name, (n, src, dst, oids, _) in CASES.items():
        s, d = as_indices(n, src, dst, oids)
        keys = set()
        simple = True
        for a, b in zip(s.tolist(), d.tolist()):
            k = (min(a, b), max(a, b))
            if a == b or k in keys:
                simple = False
                break
            keys.add(k)
        if simple and n <= 2100 and len(s) <= 40000 and name not in ("rmat12_deg1", "rmat12_absent"):
            out[name] = (n, s, d)
    for name, (n, s, d, _) in {"path": S.path(30), "star": S.star(40), "clique": S.clique(12),
                               "bipartite": S.complete_bipartite(5, 7)}.items():
        out[name] = (n, s, d)
    side = 6
    grid = [(r * side + c, r * side + c + 1) for r in range(side) for c in range(side - 1)] + \
           [(r * side + c, (r + 1) * side + c) for r in range(side - 1) for c in range(side)]
    out["grid"] = (side * side, np.array([a for a, _ in grid]), np.array([b for _, b in grid]))
    return out


SIMPLE = simple_graphs()


@pytest.mark.parametrize("name", sorted(SIMPLE) + ["karate"])
def test_networkx_exact(name):
    nx = pytest.importorskip("networkx")
    if name == "karate":
        G = nx.karate_club_graph()
        n = G.number_of_nodes()
        e = np.array(G.edges(), dtype=np.int64)
        s, d = e[:, 0], e[:, 1]
    else:
        n, s, d = SIMPLE[name]
        G = nx.Graph()
        G.add_nodes_from(range(n))
        G.add_edges_from(zip(np.asarray(s).tolist(), np.asarray(d).tolist()))
    rp, col = BO.sorted_csr(n, s, d)
    got, _ = BSO.bc_sources(n, rp, col, list(range(n)))
    w = nx.betweenness_centrality(G, normalized=False)
    want = 2.0 * np.array([w[v] for v in range(n)])
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)


MULTI = ["random%d" % i for i in range(8)] + ["shape_multi_loop", "shape_empty1", "diamond_chain40", "shape_union"]


@pytest.mark.parametrize("name", MULTI)
def test_plain_brandes_on_multigraphs(name):
    n, src, dst, oids, _ = CASES[name]
    rp, col = graph(n, src, dst, oids)
    lids = list(range(n)) if n <= 300 else list(range(0, n, max(n // 60, 1)))
    got, st = BSO.bc_sources(n, rp, col, lids + [None, lids[0]])
    want = brandes(n, rp, col, lids + [None, lids[0]])
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)
    assert st["touched_vertices"] == st["frontier_vertices"] - len(lids) - 1


def _ref_check(name, got_sources, sums):
    n, src, dst, oids, sources = ref_cases()[name]
    assert list(got_sources) == list(sources)
    rp, col = graph(n, src, dst, oids)
    want, _ = BSO.bc_sources(n, rp, col, [source_index(n, oids, s) for s in sources])
    assert np.allclose(want, sums, rtol=1e-5, atol=1e-6 * max(1.0, float(np.max(np.abs(want)))))


@pytest.mark.parametrize("name", sorted(ref_cases()))
def test_reference_fixtures(name):
    z = ref_bc_sources_outputs()
    _ref_check(name, z[name + "_sources"], z[name])


@pytest.mark.skipif(not refbc.available(), reason="oracle/_ref/ref_bc_driver is not built")
def test_live_reference():
    name = "rmat12"
    n, src, dst, oids, sources = ref_cases()[name]
    sources = sources[:4]
    acc = np.zeros(n)
    for s in sources:
        c, _, _ = refbc.run_app(n, src, dst, s, oids=oids, threads=1)
        c = c.astype(np.float64)
        c[s] = 0.0
        acc += c
    rp, col = graph(n, src, dst, oids)
    want, _ = BSO.bc_sources(n, rp, col, sources)
    assert np.allclose(want, acc, rtol=1e-5, atol=1e-6 * float(np.max(want)))
