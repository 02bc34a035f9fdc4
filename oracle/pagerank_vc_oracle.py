"""PageRankVC (the reference's pagerank_vc.h, run_app --vc) as plain scipy: the definition
GL_APP_PAGERANK_VC is checked against, and a host model of its query statistics.

Vertices are 0..n-1 and every edge is undirected for the app; deg(v) counts edge endpoints
equal to v (a self loop twice, every duplicate).  See GL_APP_PAGERANK_VC in include/grape_b200.h."""
import math

import numpy as np
import scipy.sparse as sp


def adjacency(n, src, dst):
    """W = A + A^T with multiplicity: W[v, u] = number of local CSR entries (v, u)."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    a = sp.csr_matrix((np.ones(len(src)), (src, dst)), shape=(n, n))
    return (a + a.T).tocsr()


def pagerank_vc(n, src, dst, delta=0.85, max_round=10):
    """One f64 value per vertex 0..n-1 after max_round rounds (all 0.0 when max_round <= 0)."""
    if max_round <= 0:
        return np.zeros(n, dtype=np.float64)
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    deg = (np.bincount(src, minlength=n) + np.bincount(dst, minlength=n)).astype(np.float64)
    dangling = deg == 0
    D = float(dangling.sum())
    W = adjacency(n, src, dst)
    p = 1.0 / n
    safe = np.where(dangling, 1.0, deg)
    mr = np.where(dangling, p, p / safe)
    dangling_sum = p * D
    for k in range(1, max_round + 1):
        base = (1.0 - delta) / n + delta * dangling_sum / n
        dangling_sum = base * D
        s = W @ mr
        if k < max_round:
            mr = np.where(dangling, base, (base + delta * s) / safe)
        else:
            return s * delta + base
    raise AssertionError("unreachable")


def partition(n, fnum):
    """The VCPartitioner layout: per fid a dict of master / source / destination ranges."""
    side = int(round(math.sqrt(fnum)))
    assert side * side == fnum, "fnum must be a perfect square"
    mvc = -(-n // fnum)
    vchunk = mvc * side

    def chunk(c):
        return (min(c * vchunk, n), min((c + 1) * vchunk, n))

    out = []
    for f in range(fnum):
        s, d = chunk(f // side), chunk(f % side)
        local = (s[1] - s[0]) + (0 if f // side == f % side else d[1] - d[0])
        out.append({"fid": f, "side": side, "mvc": mvc, "vchunk": vchunk,
                    "master": (min(f * mvc, n), min((f + 1) * mvc, n)),
                    "src": s, "dst": d, "local_vnum": local})
    return out


def block_of(n, fnum, src, dst):
    """Fragment of every edge: (a / vchunk) * s + b / vchunk."""
    p = partition(n, fnum)[0]
    return (np.asarray(src, dtype=np.int64) // p["vchunk"]) * p["side"] + np.asarray(dst, dtype=np.int64) // p["vchunk"]


def stats(n, src, dst, fnum=1, max_round=10):
    """Per fid, what gl_app_query reports: supersteps, the per-round step_entries / step_frontier,
    entries_scanned, frontier_vertices, touched_vertices and msg_bytes_sent."""
    parts = partition(n, fnum)
    blk = np.bincount(block_of(n, fnum, src, dst), minlength=fnum) if len(src) else np.zeros(fnum, dtype=np.int64)
    side = parts[0]["side"]
    out = []
    for p in parts:
        f = p["fid"]
        nm = p["master"][1] - p["master"][0]
        holds = lambda g, c: g // side == c or g % side == c   # noqa: E731
        gather = sum(8 * (q["master"][1] - q["master"][0]) for q in parts
                     if q["fid"] != f and holds(f, q["fid"] // side))
        scatter = 8 * nm * sum(1 for g in range(fnum) if g != f and holds(g, f // side))
        R = max(max_round, 0)
        entries = 2 * int(blk[f])
        out.append({"fid": f, "supersteps": R + 1, "block_edges": int(blk[f]), "entries": entries,
                    "local_vnum": p["local_vnum"], "masters": nm,
                    "step_entries": [entries] * R, "step_frontier": [p["local_vnum"]] * R,
                    "entries_scanned": entries * R, "frontier_vertices": p["local_vnum"] * R,
                    "touched_vertices": nm * R,
                    "msg_bytes_sent": 0 if (fnum == 1 or R == 0) else (R + 1) * gather + R * scatter})
    return out
