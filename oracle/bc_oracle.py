"""CPU oracle for single-source betweenness centrality (numpy) — TEST INFRASTRUCTURE ONLY.

A level-synchronous restatement of the reference CPU app `bc`
(examples/analytical_apps/bc/staged_bc_bfs.h, then bc/staged_bc.h) on the
undirected CSR the fragment builder makes: every input edge (u, v) is an entry
in u's row and one in v's row (a multi-edge once per copy, a self loop twice),
rows sorted by neighbour, vertices in ascending-lid order.

Returns (c float32, sigma float64, depth int64) per vertex; an unreached
vertex has depth INT64_MAX, sigma 0 and c 0.
* sigma(source) = 1; a depth-1 vertex has sigma 1 however many parallel edges
  join it to the source; a vertex at depth d >= 2 sums sigma(u) over the
  entries (v, u) of its row with depth(u) = d - 1.
* Backward, levels L .. 0: a vertex v at depth d > 0 takes
  c = f32(double(cacc) * sigma), t = f32((1 / sigma) * (1 + double(c))), where
  cacc is the sum of t over its entries to depth d + 1; the source keeps cacc.

Two arithmetics:
* mode="f64": what the GPU app computes: each sum taken in f64 over the
  vertex's own row, rounded to f32 once.
* mode="replay": the reference's one-thread order: sigma by sequential f64
  additions in (v ascending, row order), c as a running f32 sum in the same
  order (np.add.at on float32).  It reproduces the reference bit for bit.

bc_rows() is the GPU app exactly: the same rules on the fragment's own CSR,
with every sum taken in the order of the kernel's gathers.  The f64 mode
differs from it only where a sum rounds (sigma past 2^53, or t values far
apart in magnitude), which is why both are kept.
"""
import numpy as np

INF = np.iinfo(np.int64).max


def sorted_csr(n, src, dst):
    """(rp, col) of the undirected multigraph with every row sorted ascending."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    rows = np.concatenate([src, dst])
    cols = np.concatenate([dst, src])
    order = np.lexsort((cols, rows))
    rp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=rp[1:])
    return rp, cols[order]


def _entries(rp, col, vs):
    """(owner, neighbour) of the concatenated rows of vs, in order."""
    b, e = rp[vs], rp[vs + 1]
    lens = e - b
    total = int(lens.sum())
    if total == 0:
        z = np.zeros(0, dtype=np.int64)
        return z, z
    starts = np.repeat(b - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    return np.repeat(vs, lens), col[starts + np.arange(total, dtype=np.int64)]


def _segment_sum(owner, vals, vs):
    """f64 sum of vals per owner in vs (vs ascending, owner grouped in that order)."""
    out = np.zeros(len(vs), dtype=np.float64)
    if len(owner):
        idx = np.searchsorted(vs, owner)
        np.add.at(out, idx, vals)   # unbuffered: one addition per entry, in entry order
    return out


def levels_of(n, rp, col, source):
    """BFS levels (list of ascending lid arrays) and the depth array."""
    depth = np.full(n, INF, dtype=np.int64)
    if source is None or not 0 <= source < n:
        return [], depth
    depth[source] = 0
    levels = [np.array([source], dtype=np.int64)]
    while True:
        _, nb = _entries(rp, col, levels[-1])
        nb = np.unique(nb[depth[nb] == INF])
        if len(nb) == 0:
            break
        depth[nb] = len(levels)
        levels.append(nb)
    return levels, depth


def bc(n, src, dst, source, mode="f64"):
    """-> (c float32, sigma float64, depth int64) in lid order.  source: a lid, or None / out of range
    for a source oid that is not in the graph."""
    assert mode in ("f64", "replay")
    rp, col = sorted_csr(n, src, dst)
    levels, depth = levels_of(n, rp, col, source)
    sigma = np.zeros(n, dtype=np.float64)
    c = np.zeros(n, dtype=np.float32)
    if not levels:
        return c, sigma, depth
    sigma[levels[0]] = 1.0
    if len(levels) > 1:
        sigma[levels[1]] = 1.0
    for d in range(2, len(levels)):
        if mode == "f64":
            # gather over the level's own rows
            own, nb = _entries(rp, col, levels[d])
            keep = depth[nb] == d - 1
            sigma[levels[d]] = _segment_sum(own[keep], sigma[nb[keep]], levels[d])
        else:
            # the reference's scatter from the previous level, v ascending, row order
            v, u = _entries(rp, col, levels[d - 1])
            keep = depth[u] == d
            np.add.at(sigma, u[keep], sigma[v[keep]])
    t = np.zeros(n, dtype=np.float32)
    L = len(levels) - 1
    if mode == "f64":
        for d in range(L, -1, -1):
            vs = levels[d]
            own, nb = _entries(rp, col, vs)
            keep = depth[nb] == d + 1
            cacc = _segment_sum(own[keep], t[nb[keep]].astype(np.float64), vs).astype(np.float32)
            if d == 0:
                c[vs] = cacc
                break
            cv = (cacc.astype(np.float64) * sigma[vs]).astype(np.float32)
            c[vs] = cv
            t[vs] = ((1.0 / sigma[vs]) * (1.0 + cv.astype(np.float64))).astype(np.float32)
        return c, sigma, depth
    for d in range(L, 0, -1):
        vs = levels[d]
        c[vs] = (c[vs].astype(np.float64) * sigma[vs]).astype(np.float32)
        t[vs] = ((1.0 / sigma[vs]) * (1.0 + c[vs].astype(np.float64))).astype(np.float32)
        v, u = _entries(rp, col, vs)
        keep = depth[u] == d - 1
        np.add.at(c, u[keep], t[v[keep]])   # float32 running sums in the reference's thread-0 order
    return c, sigma, depth


def warp_fold(a):
    """The xor butterfly of warp_sum (engine.cuh) on the last axis (32 lanes): lane i += lane i ^ o for
    o = 16, 8, 4, 2, 1.  Lanes i and i ^ o add the same two values, so every lane ends with lane 0's
    value, which is a[:h] + a[h:] folded down to one."""
    a = np.asarray(a, dtype=np.float64)
    assert a.shape[-1] == 32
    h = 16
    while h:
        a = a[..., :h] + a[..., h:]
        h //= 2
    return a[..., 0]


def ordered_row_sums(rp, col, vs, term, short=32, chunk=1024):
    """f64 sum of term[col[j]] over the row of every vertex in vs, in the order of the gathers of
    app_bc.cu: a row of up to `short` entries is summed sequentially from 0.0; a longer row is cut into
    `chunk`-entry chunks, lane l of a chunk sums the chunk's entries l, l + 32, .. sequentially, the 32
    lane partials are folded by warp_fold, and the chunk sums are added in chunk order from 0.0.
    short=None: one sequential sum over every row (k_bc_pull_multi / k_bc_back_multi).
    term: f64 per vertex, 0.0 where an entry does not qualify (the kernels add 0.0 then too)."""
    vs = np.asarray(vs, dtype=np.int64)
    out = np.zeros(len(vs), dtype=np.float64)
    if len(vs) == 0:
        return out
    deg = (rp[vs + 1] - rp[vs]).astype(np.int64)
    total = int(deg.sum())
    if total == 0:
        return out
    row = np.repeat(np.arange(len(vs), dtype=np.int64), deg)
    first = np.concatenate([[0], np.cumsum(deg)[:-1]])
    j = np.arange(total, dtype=np.int64) - np.repeat(first, deg)   # position within the row
    vals = term[col[np.repeat(rp[vs].astype(np.int64), deg) + j].astype(np.int64)]
    seq = np.ones(total, dtype=bool) if short is None else (deg <= short)[row]
    # np.add.at is unbuffered: repeated indices are added one at a time, in entry order
    np.add.at(out, row[seq], vals[seq])
    lng = ~seq
    if lng.any():
        nch = (deg + chunk - 1) // chunk
        nch[deg <= short] = 0
        cbase = np.concatenate([[0], np.cumsum(nch)[:-1]])
        ck = cbase[row[lng]] + j[lng] // chunk             # global chunk index, chunks in row / chunk order
        lanes = np.zeros((int(nch.sum()), 32), dtype=np.float64)
        np.add.at(lanes, (ck, (j[lng] % chunk) % 32), vals[lng])
        np.add.at(out, np.repeat(np.arange(len(vs), dtype=np.int64), nch), warp_fold(lanes))
    return out


def bc_rows(n, rp, col, source, short=32, chunk=1024):
    """What k_bc_fused computes, bit for bit, on the CSR (rp, col) in the kernel's own row order (global
    vertex indices; a fragment's csr(0) when it is the only one).  Same rules as bc(): sigma(source) =
    1, sigma = 1 at depth 1, the source keeps cacc, c = f32(f64(cacc) * sigma), t = f32((1 / sigma) *
    (1 + f64(c))); every sum in the order of ordered_row_sums (short=None: the multi-fragment
    kernels' sequential rows).  -> (c float32, sigma float64, depth int64)."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    levels, depth = levels_of(n, rp, col, source)
    sigma = np.zeros(n, dtype=np.float64)
    c = np.zeros(n, dtype=np.float32)
    if not levels:
        return c, sigma, depth
    sigma[levels[0]] = 1.0
    if len(levels) > 1:
        sigma[levels[1]] = 1.0
    for d in range(2, len(levels)):
        term = np.where(depth == d - 1, sigma, 0.0)
        sigma[levels[d]] = ordered_row_sums(rp, col, levels[d], term, short, chunk)
    t = np.zeros(n, dtype=np.float32)
    for d in range(len(levels) - 1, -1, -1):
        vs = levels[d]
        term = np.where(depth == d + 1, t.astype(np.float64), 0.0)
        cacc = ordered_row_sums(rp, col, vs, term, short, chunk).astype(np.float32)
        if d == 0:
            c[vs] = cacc
            break
        cv = (cacc.astype(np.float64) * sigma[vs]).astype(np.float32)
        c[vs] = cv
        t[vs] = ((1.0 / sigma[vs]) * (1.0 + cv.astype(np.float64))).astype(np.float32)
    return c, sigma, depth
