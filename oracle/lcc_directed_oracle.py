"""Directed local clustering coefficient (the reference's LCCDirected,
examples/analytical_apps/lcc/lcc_directed.h) as sparse linear algebra — TEST
INFRASTRUCTURE ONLY.

An independent formulation, not the oriented triangle walk of the reference or of
csrc/app_lcc_directed.cu.  With A the directed adjacency counted with multiplicity
(A[u, v] = number of edges u -> v), W = A + A^T holds the weight of every pair:
W[v, u] = #(v->u) + #(u->v), the CSR entries of u in oe(v) + ie(v); W[v, v] = 2 #(v->v).
P is the off-diagonal pattern of W and W_off its off-diagonal part.  Then

    d(v)   = nnz of row v of W        (distinct neighbours, v itself with a self loop)
    tri(v) = rowsum((P W_off) o P)[v] / 2
           = sum of W[u, x] over unordered pairs {u, x} of N(v) \\ {v}, u != x
    lcc(v) = tri / (d (d - 1)), 0 when d < 2.

reference=True applies the reference's uint8_t weights (lcc_directed.h:205): every
W[u, x] that enters tri is taken modulo 256 (d is unchanged), which reproduces the
reference bit for bit.  Counts are int64 (the reference's LCCDirected64)."""
import numpy as np
import scipy.sparse as sp

from .stats_model import DENSE, Stats

# rows of P per sparse product, chosen so that one product stays around this many partial products
_FLOPS_PER_BLOCK = 1 << 26


def weights(n, src, dst):
    """W = A + A^T (CSR, int64, duplicates summed)."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    ones = np.ones(len(src), dtype=np.int64)
    a = sp.coo_matrix((ones, (src, dst)), shape=(n, n)).tocsr()
    w = (a + a.T).tocsr()
    w.sum_duplicates()
    w.sort_indices()
    return w


def lcc_directed(n, src, dst, reference=False):
    """-> (lcc float64, tri int64, d int64), one value per vertex index 0..n-1."""
    w = weights(n, src, dst)
    d = np.diff(w.indptr).astype(np.int64)
    w_off = w.copy()
    w_off.setdiag(0)
    w_off.eliminate_zeros()
    p = w_off.copy()
    p.data = np.ones_like(p.data)
    if reference:
        w_off.data = w_off.data % 256   # zeros that stay explicit add nothing
    tri2 = np.zeros(n, dtype=np.int64)
    # row blocks: the partial products of row v are sum over u in N(v) of |N(u)|
    plen = np.diff(p.indptr).astype(np.int64)
    rows = np.repeat(np.arange(n, dtype=np.int64), plen)
    flops = np.bincount(rows, weights=plen[p.indices], minlength=n).astype(np.int64)
    lo = 0
    cum = np.cumsum(flops)
    while lo < n:
        base = cum[lo - 1] if lo else 0
        hi = int(np.searchsorted(cum, base + _FLOPS_PER_BLOCK, side="right"))
        hi = min(max(hi, lo + 1), n)
        pb = p[lo:hi]
        tri2[lo:hi] = np.asarray((pb @ w_off).multiply(pb).sum(axis=1), dtype=np.int64).ravel()
        lo = hi
    tri = tri2 // 2
    lcc = np.zeros(n, dtype=np.float64)
    ok = d >= 2
    lcc[ok] = tri[ok].astype(np.float64) / (d[ok] * (d[ok] - 1)).astype(np.float64)
    return lcc, tri, d


def lcc_directed_fast(n, src, dst, reference=False):
    """The same values through an orientation, for graphs where the row products of lcc_directed are too
    many: rank the vertices by (d, index) and let U hold the pairs of P from a vertex to a lower-ranked
    one.  A triangle a > b > c (in rank) is U[a,b] U[a,c] U[b,c], and it adds W[b,c] to a, W[a,c] to b
    and W[a,b] to c:
        tri = rowsum((U (U o W)) o U) + colsum(((U o W) U^T) o U) + colsum(((U o W) U) o U).
    -> (lcc, tri, d) as lcc_directed."""
    w = weights(n, src, dst)
    d = np.diff(w.indptr).astype(np.int64)
    w_off = w.tocoo()
    off = w_off.row != w_off.col
    r, c, x = w_off.row[off].astype(np.int64), w_off.col[off].astype(np.int64), w_off.data[off].astype(np.int64)
    if reference:
        x = x % 256
    rank = np.empty(n, dtype=np.int64)
    rank[np.lexsort((np.arange(n), d))] = np.arange(n)
    low = rank[c] < rank[r]
    u = sp.csr_matrix((np.ones(int(low.sum()), dtype=np.int64), (r[low], c[low])), shape=(n, n))
    uw = sp.csr_matrix((x[low], (r[low], c[low])), shape=(n, n))
    tri = np.asarray((u @ uw).multiply(u).sum(axis=1), dtype=np.int64).ravel()
    tri += np.asarray((uw @ u.T).multiply(u).sum(axis=0), dtype=np.int64).ravel()
    tri += np.asarray((uw @ u).multiply(u).sum(axis=0), dtype=np.int64).ravel()
    lcc = np.zeros(n, dtype=np.float64)
    ok = d >= 2
    lcc[ok] = tri[ok].astype(np.float64) / (d[ok] * (d[ok] - 1)).astype(np.float64)
    return lcc, tri, d


def stats(n, src, dst, rank=None, owned=None):
    """Query statistics (gl_query_stats, the step layout of oracle/stats_model.py) of GL_APP_LCC_DIRECTED
    on the directed edge list (src, dst) over vertices 0..n-1.  PEval builds N+(v), the distinct
    neighbours u != v of v over its out- and in-edges with (deg u, rank u) < (deg v, rank v), deg =
    out-edges + in-edges counted with multiplicity and rank = the gid order (default: the vertex index);
    step 1 reads N+(u) for every oriented entry (v, u) of the fragment's vertices (`owned`, a boolean
    mask; default all); step 2 ends the query."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    rank = np.arange(n, dtype=np.int64) if rank is None else np.asarray(rank, dtype=np.int64)
    owned = np.ones(n, dtype=bool) if owned is None else np.asarray(owned, dtype=bool)
    deg = np.bincount(src, minlength=n) + np.bincount(dst, minlength=n)
    a = np.concatenate([src, dst])
    b = np.concatenate([dst, src])
    pairs = np.unique(a * max(n, 1) + b)
    v, u = pairs // max(n, 1), pairs % max(n, 1)
    keep = (v != u) & ((deg[u] < deg[v]) | ((deg[u] == deg[v]) & (rank[u] < rank[v])))
    v, u = v[keep], u[keep]
    out_deg = np.bincount(v, minlength=n)
    entries = int(out_deg[u[owned[v]]].sum())
    iv = int(owned.sum())
    return Stats(3, [0, entries, 0], [0, iv, 0], [0, DENSE, 0], iv)


def brute_force(n, src, dst):
    """Pair enumeration straight from the definition (small graphs): -> (tri, d)."""
    w = {}
    for a, b in zip(np.asarray(src, np.int64).tolist(), np.asarray(dst, np.int64).tolist()):
        w[(a, b)] = w.get((a, b), 0) + 1
        w[(b, a)] = w.get((b, a), 0) + 1
    nbr = [set() for _ in range(n)]
    for (a, b) in w:
        nbr[a].add(b)
    tri = np.zeros(n, dtype=np.int64)
    d = np.array([len(s) for s in nbr], dtype=np.int64)
    for v in range(n):
        others = sorted(nbr[v] - {v})
        for i, u in enumerate(others):
            for x in others[i + 1:]:
                tri[v] += w.get((u, x), 0)
    return tri, d
