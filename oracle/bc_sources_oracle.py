"""CPU oracle for betweenness centrality summed over a list of sources (numpy) — TEST INFRASTRUCTURE ONLY.

For every source s of the list, on the CSR (rp, col) in its own row order (a fragment's csr(0) when it
is the only one): depth_s and sigma_s as bc_oracle.bc_rows (sigma 1 at depth 1 however many parallel
edges); backward from the deepest level, cacc = the sum of t_s(w) over the entries (v, w) of v's row
with depth_s(w) = depth_s(v) + 1, delta_s(v) = cacc * sigma_s(v), t_s(v) = (1 / sigma_s(v)) *
(1 + delta_s(v)), all f64; bc(v) = (((0.0 + delta_s1(v)) + delta_s2(v)) + ...) in list order.

Every row sum is taken in the order of app_bc_sources.cu: a row of up to `chunk` entries sequentially
from 0.0, a longer row as sequential chunk sums added in chunk order from 0.0.  Entries that do not
qualify add nothing (the kernel skips them; every qualifying term is positive, so adding 0.0 instead
would not change a bit).
"""
import numpy as np

from oracle.bc_oracle import INF, levels_of

CHUNK = 1024


def chunk_row_sums(rp, col, vs, term, chunk=CHUNK):
    """f64 sum of term[col[j]] over the row of every vertex in vs, in the kernel's order."""
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
    j = np.arange(total, dtype=np.int64) - np.repeat(first, deg)
    vals = term[col[np.repeat(rp[vs].astype(np.int64), deg) + j]]
    nz = vals != 0.0
    seq = (deg <= chunk)[row] & nz
    np.add.at(out, row[seq], vals[seq])   # unbuffered: one addition per entry, in entry order
    lng = (deg > chunk)[row] & nz
    if lng.any():
        nch = np.where(deg > chunk, (deg + chunk - 1) // chunk, 0)
        cbase = np.concatenate([[0], np.cumsum(nch)[:-1]])
        part = np.zeros(int(nch.sum()), dtype=np.float64)
        np.add.at(part, cbase[row[lng]] + j[lng] // chunk, vals[lng])
        np.add.at(out, np.repeat(np.arange(len(vs), dtype=np.int64), nch), part)
    return out


def deltas(n, rp, col, source, chunk=CHUNK):
    """-> (delta float64, depth int64) of one source lid (None: not in the graph); delta is 0 at the
    source and at unreached vertices."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    levels, depth = levels_of(n, rp, col, source)
    delta = np.zeros(n, dtype=np.float64)
    if not levels:
        return delta, depth
    sigma = np.zeros(n, dtype=np.float64)
    sigma[levels[0]] = 1.0
    if len(levels) > 1:
        sigma[levels[1]] = 1.0
    for d in range(2, len(levels)):
        term = np.where(depth == d - 1, sigma, 0.0)
        sigma[levels[d]] = chunk_row_sums(rp, col, levels[d], term, chunk)
    t = np.zeros(n, dtype=np.float64)
    for d in range(len(levels) - 1, 0, -1):
        vs = levels[d]
        term = np.where(depth == d + 1, t, 0.0)
        cacc = chunk_row_sums(rp, col, vs, term, chunk)
        dv = cacc * sigma[vs]
        delta[vs] = dv
        t[vs] = (1.0 / sigma[vs]) * (1.0 + dv)
    return delta, depth


def bc_sources(n, rp, col, sources, chunk=CHUNK):
    """-> (bc float64 [n], stats) for the list of source lids (None: an entry not in the graph), folded in
    list order.  stats: frontier_vertices (reached vertices summed over the list, sources included),
    touched_vertices (that minus the entries found in the graph) and per_source (each entry's reached
    count)."""
    bc = np.zeros(n, dtype=np.float64)
    per = []
    for s in sources:
        dl, depth = deltas(n, rp, col, s, chunk)
        bc += dl
        per.append(int(np.count_nonzero(depth != INF)))
    present = sum(1 for s in sources if s is not None and 0 <= s < n)
    return bc, {"frontier_vertices": sum(per), "touched_vertices": sum(per) - present, "per_source": per}


def source_lids(frag_oids, oids):
    """List entries (oids) -> lids of a one-fragment graph whose inner oids are frag_oids in lid order
    (None for an oid that is not a vertex)."""
    frag_oids = np.asarray(frag_oids, dtype=np.int64)
    order = np.argsort(frag_oids, kind="stable")
    so = frag_oids[order]
    out = []
    for o in oids:
        i = int(np.searchsorted(so, o))
        out.append(int(order[i]) if i < len(so) and so[i] == o else None)
    return out
