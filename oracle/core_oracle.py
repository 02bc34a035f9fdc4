"""CPU oracle for core decomposition and k-core (numpy) — TEST INFRASTRUCTURE ONLY.

A plain level-synchronous restatement of the reference CPU apps
(examples/analytical_apps/core_decomposition/core_decomposition.h,
kcore/kcore.h) on the undirected CSR the fragment builder makes: every input
edge (u, v) is an entry in u's row and one in v's row, so a multi-edge counts
once per copy and a self loop counts twice.

* core_decomposition: a vertex is peeled at level L once its count of entries
  to unpeeled vertices is <= L; isolated vertices get core 0.  Levels jump to
  max(L + 1, smallest remaining count), which peels exactly what stepping L by
  one would.  Also returns the number of sub-rounds (frontier scans).
* kcore: one peel at L = k - 1 that counts down every entry of a peeled row;
  the value is the number of a vertex's entries whose other endpoint survives.
"""
import numpy as np


def undirected_csr(n, src, dst):
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    rows = np.concatenate([src, dst])
    cols = np.concatenate([dst, src])
    order = np.argsort(rows, kind="stable")
    rp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=rp[1:])
    return rp, cols[order]


def _row_entries(rp, col, vs):
    """Concatenated rows of the vertices vs."""
    b, e = rp[vs], rp[vs + 1]
    lens = e - b
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, dtype=np.int64)
    starts = np.repeat(b - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    return col[starts + np.arange(total, dtype=np.int64)]


def _peel(rp, col, cnt, front, L, peeled, count_peeled):
    """Sub-rounds of one level from the frontier `front` (already peeled).
    Returns (vertices peeled, in order of their sub-round; sub-rounds run)."""
    got, rounds = [], 0
    while len(front):
        rounds += 1
        got.append(front)
        nb = _row_entries(rp, col, front)
        if not count_peeled:
            nb = nb[~peeled[nb]]
        u, c = np.unique(nb, return_counts=True)
        old = cnt[u]
        cnt[u] = old - c
        cross = (old > L) & (old - c <= L)
        front = u[cross]
        peeled[front] = True
    return (np.concatenate(got) if got else np.zeros(0, dtype=np.int64)), rounds


def core_decomposition(n, src, dst):
    """(core number per vertex as int64, sub-rounds of the level-synchronous peel)."""
    rp, col = undirected_csr(n, src, dst)
    cnt = np.diff(rp)
    core = np.zeros(n, dtype=np.int64)
    peeled = cnt == 0
    L, rounds = -1, 0
    while not peeled.all():
        rem = np.flatnonzero(~peeled)
        L = max(L + 1, int(cnt[rem].min()))
        front = rem[cnt[rem] <= L]
        peeled[front] = True
        got, r = _peel(rp, col, cnt, front, L, peeled, False)
        core[got] = L
        rounds += r
    return core, rounds


def kcore(n, src, dst, k):
    """Count of entries to surviving endpoints per vertex (int64); the k-core is value >= k."""
    rp, col = undirected_csr(n, src, dst)
    cnt = np.diff(rp)
    L = int(k) - 1
    front = np.flatnonzero(cnt <= L)
    peeled = np.zeros(n, dtype=bool)
    peeled[front] = True
    _peel(rp, col, cnt, front, L, peeled, True)
    return cnt.astype(np.int64)
