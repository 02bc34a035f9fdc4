"""The betweenness oracle (oracle/bc_oracle.py) against a brute-force
restatement in exact rational arithmetic on random multigraphs, and against
closed forms on paths, stars, cliques, complete bipartite graphs and cycles."""
from collections import deque
from fractions import Fraction

import numpy as np
import pytest

from oracle import bc_oracle as BO
from tests import shapes as S
from tests.core_cases import random_multigraph

INF = BO.INF


def brute_force(n, src, dst, source):
    """depth, sigma and c by the rules of the reference app, per CSR entry, with Fractions."""
    adj = [[] for _ in range(n)]
    for a, b in zip(src.tolist(), dst.tolist()):
        adj[a].append(b)
        adj[b].append(a)
    depth = [None] * n
    depth[source] = 0
    q = deque([source])
    while q:
        v = q.popleft()
        for u in adj[v]:
            if depth[u] is None:
                depth[u] = depth[v] + 1
                q.append(u)
    order = sorted((v for v in range(n) if depth[v] is not None), key=lambda v: depth[v])
    sigma = [Fraction(0)] * n
    for v in order:
        if depth[v] <= 1:
            sigma[v] = Fraction(1)   # the source, and every depth-1 vertex whatever its parallel edges
        else:
            sigma[v] = sum((sigma[u] for u in adj[v] if depth[u] == depth[v] - 1), Fraction(0))
    c = [Fraction(0)] * n
    for v in reversed(order):
        acc = sum(((1 + c[u]) / sigma[u] for u in adj[v] if depth[u] == depth[v] + 1), Fraction(0))
        c[v] = acc if v == source else acc * sigma[v]
    return depth, sigma, c


@pytest.mark.parametrize("seed", range(24))
def test_f64_oracle_equals_brute_force(seed):
    n, s, d = random_multigraph(seed)
    rng = np.random.RandomState(1000 + seed)
    source = int(rng.randint(0, n))
    depth, sigma, c = brute_force(n, s, d, source)
    gc, gs, gd = BO.bc(n, s, d, source, "f64")
    for v in range(n):
        if depth[v] is None:
            assert gd[v] == INF and gs[v] == 0 and gc[v] == 0
            continue
        assert gd[v] == depth[v]
        assert gs[v] == float(sigma[v])
        assert abs(float(gc[v]) - float(c[v])) <= 1e-6 * max(1.0, abs(float(c[v]))), v


def test_absent_and_isolated_sources():
    n, s, d, _ = S.union([S.path(5), S.empty(3)], seed=0)
    for source in (None, n, -1):
        c, sigma, depth = BO.bc(n, s, d, source)
        assert (depth == INF).all() and not sigma.any() and not c.any()
    iso = [v for v in range(n) if v not in set(s.tolist()) | set(d.tolist())][0]
    c, sigma, depth = BO.bc(n, s, d, iso)
    assert depth[iso] == 0 and sigma[iso] == 1 and c[iso] == 0
    assert (np.delete(depth, iso) == INF).all()


def test_parallel_edges_to_the_source_keep_sigma_one():
    # source 0 joined twice to 1 and 2; 3 hangs off both: sigma(3) = 2, not 4
    src = np.array([0, 0, 0, 0, 1, 2])
    dst = np.array([1, 1, 2, 2, 3, 3])
    for mode in ("f64", "replay"):
        c, sigma, depth = BO.bc(4, src, dst, 0, mode)
        assert depth.tolist() == [0, 1, 1, 2]
        assert sigma.tolist() == [1, 1, 1, 2]
        # t(3) = 1/2 reaches 1 and 2 once each; each copy of a source edge adds 1.5
        assert c.tolist() == [6.0, 0.5, 0.5, 0.0]


def closed_form_cases():
    out = []
    n = 12
    out.append(("path", n, np.arange(n - 1), np.arange(1, n), 0, [n - 1 - v for v in range(n)]))
    k = 9
    star_s, star_d = np.zeros(k, dtype=np.int64), np.arange(1, k + 1)
    out.append(("star_centre", k + 1, star_s, star_d, 0, [k] + [0] * k))
    out.append(("star_leaf", k + 1, star_s, star_d, 1, [k - 1, k] + [0] * (k - 1)))
    m = 7
    iu = np.triu_indices(m, 1)
    out.append(("clique", m, iu[0], iu[1], 0, [m - 1] + [0] * (m - 1)))
    a, b = 4, 5
    ka = np.repeat(np.arange(a), b)
    kb = np.tile(np.arange(a, a + b), a)
    out.append(("bipartite", a + b, ka, kb, 0, [a + b - 1] + [0] * (a - 1) + [Fraction(a - 1, b)] * b))
    for n in (10, 11):
        cs, cd = np.arange(n), (np.arange(n) + 1) % n
        half = n // 2
        want = [n - 1]
        for v in range(1, n):
            dv = min(v, n - v)
            want.append(0 if (n % 2 == 1 and dv == half) else (half - dv - Fraction(1, 2) if n % 2 == 0 else half - dv))
        if n % 2 == 0:
            want[half] = 0
        out.append(("cycle%d" % n, n, cs, cd, 0, want))
    return out


@pytest.mark.parametrize("case", closed_form_cases(), ids=lambda c: c[0])
@pytest.mark.parametrize("mode", ["f64", "replay"])
def test_closed_forms(case, mode):
    _, n, s, d, source, want = case
    c, _, _ = BO.bc(n, np.asarray(s), np.asarray(d), source, mode)
    # exact up to the f32 rounding of fractional values such as (a - 1) / b
    assert np.allclose(c, [float(x) for x in want], rtol=2 ** -22, atol=0)


@pytest.mark.parametrize("seed", range(8))
def test_source_is_reached_minus_one_on_simple_graphs(seed):
    rng = np.random.RandomState(seed)
    n = 200
    pairs = {(int(min(a, b)), int(max(a, b))) for a, b in rng.randint(0, n, size=(600, 2)) if a != b}
    s = np.array([p[0] for p in pairs])
    d = np.array([p[1] for p in pairs])
    source = int(s[0])
    for mode in ("f64", "replay"):
        c, _, depth = BO.bc(n, s, d, source, mode)
        reached = int(np.count_nonzero(depth != INF))
        assert abs(float(c[source]) - (reached - 1)) <= 1e-5 * reached


@pytest.mark.parametrize("seed", range(8))
def test_replay_and_f64_agree(seed):
    from tests.util import rmat_graph
    n, s, d, _ = rmat_graph(10, seed=seed + 3)
    source = int(np.argmax(np.bincount(np.concatenate([s, d]), minlength=n)))
    cf, sf, df = BO.bc(n, s, d, source, "f64")
    cr, sr, dr = BO.bc(n, s, d, source, "replay")
    assert np.array_equal(df, dr) and np.array_equal(sf, sr)
    assert np.all(np.abs(cf.astype(np.float64) - cr) <= 1e-3 * np.abs(cr.astype(np.float64)))
