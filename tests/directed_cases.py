"""Directed graphs split into several fragments: the case table of the
several-fragment directed tests and the fragment geometry each case is chosen for.

On a directed fragment the outer vertex set is the union of the outer columns of
`oe` and `ie`, so a fragment can hold outer copies that it sees only through an
in-edge.  Those copies, the dangling vertices fed across the cut and the deep
paths that run against fid order take code paths (BFS pull levels over `ie`,
WCC labels travelling against edge direction, the dangling rule of directed
PageRank) that no undirected case reaches.  Every case here is listed with the
geometry it must reach (`claims`), which tests/test_directed_cases.py checks on
the CPU and tests/mgpu_directed_worker.py checks again on the fragments the
library built.

Every builder returns (n, src, dst, w): vertex ids 0..n-1 (int64) and float64
weights.  The library splits ids into blocks of ceil(n / fnum) ascending ids.
"""
import numpy as np

from tests import golden_io as G
from tests import shapes as S

# p2p-31 is loaded with its own oids; the edge list below is in index space
# (position in the ascending oid list), which is also the library's id order.
P2P_SOURCE_OID = 6


def p2p31_oids():
    return G.load_p2p31()[0]


def _p2p31():
    oids, src, dst, w = G.load_p2p31()
    return len(oids), np.searchsorted(oids, src), np.searchsorted(oids, dst), w


def _rmat(scale, seed, weight_mode):
    import importlib
    src, dst, w = importlib.import_module("libgrape-lite_b200").rmat_edges_host(scale, 16, seed, weight_mode)
    return 1 << scale, src, dst, w.astype(np.float64)


def reversed_path(L):
    """Edges i+1 -> i: BFS from the last vertex walks against fid order to vertex 0."""
    n, src, dst, w = S.path(L)
    return n, dst, src, w


def cycle(n):
    """Edges i -> i+1 (mod n): each fragment's only in-edge from outside comes
    from the previous fragment (fragment 0's from the last one)."""
    v = np.arange(n, dtype=np.int64)
    return n, v, (v + 1) % n, S._weights(n)


PATH_L = 400                    # BFS depth from the last vertex: > BFS_U8_MAX_LEVELS

# name -> (builder, real weights).  Real weights (R-MAT weight mode 2) are
# multiples of 2^-24: f64 sums are exact, f32 sums are not.
CASES = {
    "p2p31": (_p2p31, False),
    "rmat12": (lambda: _rmat(12, 21, 1), False),
    "rmat14": (lambda: _rmat(14, 23, 1), False),
    "rmat12_real": (lambda: _rmat(12, 25, 2), True),
    "rmat14_real": (lambda: _rmat(14, 27, 2), True),
    "sink4097": (lambda: S.sink_heavy(4097), False),
    "source4097": (lambda: S.source_heavy(4097), False),
    "reversed_path": (lambda: reversed_path(PATH_L), False),
    "cycle": (lambda: cycle(300), False),
    "star_last": (lambda: S.star(4097, True), False),
    "hub_block": (lambda: S.hub_block(33), False),
    "union": (lambda: S.union([S.star(1500), S.clique(30), S.path(40), S.empty(5)], seed=5), False),
    "empty": (lambda: S.empty(33), False),
    "path_then_isolated": (lambda: S.pad_to(S.path(300), 1000), False),
}

FNUMS = (2, 3)


def build(name):
    n, src, dst, w = CASES[name][0]()
    return n, np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64), np.asarray(w, dtype=np.float64)


def chunk_of(n, fnum):
    return (n + fnum - 1) // fnum


def geometry(n, src, dst, fnum):
    """Per fid: the inner range [lo, hi), the outer vertices the fragment sees
    through its out-edges (`oe_outer`) and through its in-edges (`ie_outer`),
    the ones seen only through in-edges (`ie_only`), the fids those in-edges come
    from (`in_from`), and the inner vertices with out-degree 0 that have in-edges
    from another fragment (`dangling_cross`).  All ids global, ascending."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    chunk = chunk_of(n, fnum)
    outdeg = np.bincount(src, minlength=n)
    out = []
    for fid in range(fnum):
        lo, hi = min(n, fid * chunk), min(n, (fid + 1) * chunk)
        s_in = (src >= lo) & (src < hi)
        d_in = (dst >= lo) & (dst < hi)
        oe_outer = np.unique(dst[s_in & ~d_in])
        ie_outer = np.unique(src[d_in & ~s_in])
        cross = np.unique(dst[d_in & ~s_in])
        out.append(dict(fid=fid, lo=lo, hi=hi, oe_outer=oe_outer, ie_outer=ie_outer,
                        outer=np.union1d(oe_outer, ie_outer),
                        ie_only=np.setdiff1d(ie_outer, oe_outer),
                        in_from=np.unique(ie_outer // chunk) if len(ie_outer) else np.zeros(0, np.int64),
                        dangling_cross=cross[outdeg[cross] == 0]))
    return out


def claims(name, n, src, dst, fnum):
    """(what, holds) pairs: the geometry case `name` is listed for at `fnum`."""
    geo = geometry(n, src, dst, fnum)
    chunk = chunk_of(n, fnum)
    outdeg = np.bincount(src, minlength=n)
    indeg = np.bincount(dst, minlength=n)
    some_ie_only = any(len(g["ie_only"]) for g in geo)
    some_dangling = any(len(g["dangling_cross"]) for g in geo)
    c = []
    if name in ("p2p31", "rmat12", "rmat14", "rmat12_real", "rmat14_real"):
        c.append(("every fragment has outer vertices seen only through in-edges", all(len(g["ie_only"]) for g in geo)))
        c.append(("every fragment has a dangling vertex fed across the cut", all(len(g["dangling_cross"]) for g in geo)))
    if name == "sink4097":
        c.append(("fid 0 sees more than K_HUB_DEG outer vertices only through in-edges",
                  len(geo[0]["ie_only"]) > S.K_HUB_DEG))
        c.append(("the centre's in-row is longer than a dense tile", indeg[0] > S.K_DENSE_TILE))
        c.append(("the dangling centre is fed across the cut", 0 in geo[0]["dangling_cross"]))
    if name == "source4097":
        c.append(("the centre pushes more than K_HUB_DEG entries across the cut", len(geo[0]["oe_outer"]) > S.K_HUB_DEG))
        c.append(("every other fragment sees the centre only as an in-neighbour",
                  all(list(g["ie_only"]) == [0] for g in geo[1:])))
    if name == "reversed_path":
        last = geo[-1]["hi"] - 1
        c.append(("BFS from the last vertex is deeper than BFS_U8_MAX_LEVELS", last > S.BFS_U8_MAX_LEVELS))
        c.append(("every fragment but the last sees its successor's first vertex only through an in-edge",
                  all(list(g["ie_only"]) == [g["hi"]] for g in geo[:-1])))
        c.append(("in-edges cross every boundary against fid order",
                  all(list(g["in_from"]) == [g["fid"] + 1] for g in geo[:-1]) and len(geo[-1]["in_from"]) == 0))
    if name == "cycle":
        c.append(("every fragment's only in-edge from outside comes from the previous fragment",
                  all(list(g["in_from"]) == [(g["fid"] - 1) % fnum] and list(g["ie_only"]) == [(g["lo"] - 1) % n]
                      for g in geo)))
        c.append(("BFS from vertex 0 is deeper than BFS_U8_MAX_LEVELS", n - 1 > S.BFS_U8_MAX_LEVELS))
    if name == "star_last":
        c.append(("the centre (last fragment) pushes more than K_HUB_DEG entries across the cut",
                  len(geo[-1]["oe_outer"]) > S.K_HUB_DEG))
        c.append(("every other fragment sees the centre only as an in-neighbour",
                  all(list(g["ie_only"]) == [n - 1] for g in geo[:-1])))
    if name == "hub_block":
        hubs = np.flatnonzero(outdeg > S.K_HUB_DEG)
        f = hubs[0] // chunk
        c.append(("more than K_MAX_TILE_HUBS long rows in one tile of one fragment",
                  len(hubs) > S.K_MAX_TILE_HUBS and np.all(hubs // chunk == f)
                  and np.all(hubs // S.K_TILE_V == hubs[0] // S.K_TILE_V)))
        c.append(("another fragment sees every hub only through in-edges",
                  any(np.array_equal(g["ie_only"], hubs) for g in geo if g["fid"] != f)))
    if name == "union":
        c.append(("outer vertices seen only through in-edges", some_ie_only))
        c.append(("a dangling vertex fed across the cut", some_dangling))
        c.append(("every fragment has edges to or from another", all(len(g["outer"]) for g in geo)))
    if name == "empty":
        c.append(("no edges, no outer vertices", len(src) == 0 and all(len(g["outer"]) == 0 for g in geo)))
    if name == "path_then_isolated":
        c.append(("an owner boundary inside a 32-bit bitmap word", chunk % 32 != 0))
        c.append(("fragments of isolated vertices only",
                  any(g["hi"] > g["lo"] and not np.any(((src >= g["lo"]) & (src < g["hi"])) | ((dst >= g["lo"]) & (dst < g["hi"])))
                      for g in geo)))
    return [(w, bool(h)) for w, h in c]


# ---------------------------------------------------------------------------
# Configurations of the several-fragment worker (tests/mgpu_directed_worker.py).
# The driver derives the number of OK lines it expects from these tables.
BFS_CONFIGS = [
    ("fused", dict(direction_opt=1)),
    ("fused_push", dict(direction_opt=0)),
    ("step", dict(direction_opt=1, fuse_supersteps=0)),
    ("step_push", dict(direction_opt=0, fuse_supersteps=0)),
    ("r1ship", dict(direction_opt=1, reserved={7: 1})),      # round-1 frontier shipment
    ("spill", dict(direction_opt=1, reserved={3: 4})),       # a ring of 4 level bitmaps: park, spill, relaunch
]
BFS_SOURCES = ("max_out", "last_frag")               # in every BFS configuration
BFS_SOURCES_FUSED = ("ie_only", "unknown")           # in the default (fused push/pull) configuration only
SSSP_SOURCES = ("last_frag",)
# (sssp_f64, sssp_prio, edge data bytes)
SSSP_INT = [(f64, prio, eb) for f64 in (0, 1) for prio in (0.0, 0.5) for eb in (4, 8)]
SSSP_REAL = [(1, 0.0, 8), (0, 0.0, 4)]       # f64: exact; f32: <= 1e-6 relative, same reached set
WCC_KINDS = ("wcc", "wcc_opt")
PR_CONFIGS = [(pull, delta, rounds) for pull in (0, 1) for delta in (0.85, 0.5) for rounds in (0, 1, 10)]
P2P_GOLDEN = ("bfs", "sssp_f32", "sssp_f64", "pagerank", "wcc")
UNDIRECTED_EXTRAS = ("sssp_f64_prio", "pr_pull32", "pr_pull32_nohub")
REFUSED = ("core_decomposition", "kcore", "kclique")
PATH_CHECKS = ("pull_fused", "pull_step")


def ok_lines_expected():
    """OK lines one worker run prints when everything matches."""
    total = 0
    for _, real in CASES.values():
        total += (len(BFS_CONFIGS) * len(BFS_SOURCES) + len(BFS_SOURCES_FUSED)
                  + len(SSSP_SOURCES) * len(SSSP_REAL if real else SSSP_INT)
                  + len(WCC_KINDS) + len(PR_CONFIGS) + 1)   # + the geometry of the built fragments
    return total + len(P2P_GOLDEN) + len(UNDIRECTED_EXTRAS) + len(REFUSED) + len(PATH_CHECKS)


def sources(n, src, dst, fnum):
    """Global ids of the BFS / SSSP sources of a case: the vertex of largest
    out-degree, the vertex of largest out-degree among those some fragment sees
    only through an in-edge (0 when there is none), the vertex of largest
    out-degree in the last fragment (highest id on ties), and an id no fragment
    holds."""
    outdeg = np.bincount(np.asarray(src, dtype=np.int64), minlength=n)
    geo = geometry(n, src, dst, fnum)
    ie_only = np.unique(np.concatenate([g["ie_only"] for g in geo]))
    last = geo[-1]
    lo, hi = last["lo"], last["hi"]
    if hi > lo:
        seg = outdeg[lo:hi]
        last_v = lo + int(np.flatnonzero(seg == seg.max())[-1])
    else:
        last_v = n - 1
    return {"max_out": int(np.argmax(outdeg)) if n else 0,
            "ie_only": int(ie_only[np.argmax(outdeg[ie_only])]) if len(ie_only) else 0,
            "last_frag": last_v,
            "unknown": n + 7}
