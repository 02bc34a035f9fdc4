"""Graphs that put the betweenness-centrality kernel (csrc/app_bc.cu) on its own
thresholds, the sources each one is run from, and host replicas of what the
kernel reports per step.

The gathers of k_bc_fused sum a row of up to K_BC_SHORT entries in one thread
and cut a longer row into K_BC_CHUNK-entry chunks; discovery is push (through
the hub phase for rows over K_HUB_DEG) or pull, chosen per level by Beamer's
rule.  Every generator returns (n, src, dst, w) like tests/shapes.py, with the
vertex the graph is built around ("root") as a separate entry of BC_SHAPES.
"""
import numpy as np

from oracle import bc_oracle as BO
from tests import shapes as S

K_BC_SHORT = 32     # app_bc.cu kBcShort: rows up to this length are summed by one thread
K_BC_CHUNK = 1024   # app_bc.cu kBcChunk: entries per chunk of a longer row
ROW_LENS = [31, 32, 33, 1023, 1024, 1025, 2048, 2049, 3073]   # both sides of each cut, and three chunks
TWO_53 = 2.0 ** 53


def _iso(n, src, dst):
    """(n + 1, src, dst, w): one isolated vertex appended, so that every graph has an isolated source."""
    return S._out(n + 1, np.concatenate([np.asarray(x, dtype=np.int64) for x in src]),
                  np.concatenate([np.asarray(x, dtype=np.int64) for x in dst]))


def fans(width=1100):
    """Root 0, a depth-1 layer 1..width, then depth-2 collectors: for every L in ROW_LENS one whose L
    entries spread over the layer (parallel edges once L > width), and for every L over 1000 one made
    of L parallel edges to three layer vertices."""
    s, d = [np.zeros(width, dtype=np.int64)], [np.arange(1, width + 1)]
    v = width + 1
    for L in ROW_LENS:
        s.append(np.full(L, v))
        d.append(1 + (np.arange(L) * 7 + L) % width)
        v += 1
        if L > 1000:
            s.append(np.full(L, v))
            d.append(1 + np.arange(L) % 3)
            v += 1
    return _iso(v, s, d)


def kab(a, b):
    """K(a, b) on A = 1..a and B = a+1..a+b, with root 0 joined to every vertex of A: the B rows (a
    entries) are a sigma gather at depth 2, the A rows (b + 1 entries) a backward gather at depth 1."""
    i, j = np.meshgrid(np.arange(1, a + 1), np.arange(a + 1, a + b + 1), indexing="ij")
    return _iso(1 + a + b, [np.zeros(a, dtype=np.int64), i.ravel()], [np.arange(1, a + 1), j.ravel()])


MIXED_LENS = [1, 33, 2, 1025, 5, 2049, 32, 1024, 17, 2048, 31, 3072, 100, 2000, 3000]


def mixed(width=40):
    """Root 0, a depth-1 layer of `width` vertices, and one depth-2 level whose rows (MIXED_LENS, parallel
    edges into the layer) are short and 1, 2 and 3 chunks long, interleaved in id order."""
    s, d = [np.zeros(width, dtype=np.int64)], [np.arange(1, width + 1)]
    for i, L in enumerate(MIXED_LENS):
        s.append(np.full(L, width + 1 + i))
        d.append(1 + (np.arange(L) * 3 + i) % width)
    return _iso(width + 1 + len(MIXED_LENS), s, d)


def _diamonds(k):
    """Joints 0, 4, .., 4k, each joined to the next through three middle vertices: sigma(joint i) = 3^i
    (rounded in f64 past 2^53)."""
    s, d = [], []
    for i in range(k):
        for m in (1, 2, 3):
            s += [4 * i, 4 * i + m]
            d += [4 * i + m, 4 * i + 4]
    return s, d


def order_chain(spread=1100, seed=3):
    """sigma past 2^53 summed in long rows (the forward gather): a 40-diamond chain from root 0 to joint
    J = 160 (sigma = 3^40), `spread` vertices joined to J by 1..7 parallel edges each, then three
    collectors joined to 32, 1024 and all of the spread vertices.  The collectors' sums round, so
    their sigma depends on the order of the row's additions."""
    s, d = _diamonds(40)
    J = 160
    k = np.random.RandomState(seed).randint(1, 8, size=spread)
    sp = J + 1 + np.arange(spread)
    src, dst = [np.array(s), np.repeat(sp, k)], [np.array(d), np.full(int(k.sum()), J)]
    col0 = J + 1 + spread
    for i, (lo, hi) in enumerate([(0, 32), (40, 40 + 1024), (0, spread)]):
        src.append(np.full(hi - lo, col0 + i))
        dst.append(sp[lo:hi])
    return _iso(col0 + 3, src, dst)


def _chain(first, mults):
    """Vertices first, first + 1, .. , first + len(mults): vertex first joined to root 0 once (depth 1,
    sigma 1), vertex first + i + 1 to first + i by mults[i] parallel edges (sigma times mults[i])."""
    s, d = [np.array([0])], [np.array([first])]
    for i, k in enumerate(mults):
        s.append(np.full(k, first + i + 1))
        d.append(np.full(k, first + i))
    return np.concatenate(s), np.concatenate(d)


def back_chain(eps=1021):
    """A backward gather whose f64 sum rounds: u at depth 24 with sigma 1, and three kinds of leaves at
    depth 25, each joined to u and to one vertex of sigma 2^60, 2^84 or 2^114 (chains of parallel
    edges; sigma 1 + 2^k rounds to 2^k), so that their t are 2^-60 (a), 2^-84 (b) and 2^-114 (the eps
    leaves).  u's row is [parent, a, b, eps leaves]: 1024 entries.  Summed in sequence, a + b is an f32
    tie and every 2^-114 is below half an f64 ulp, so cacc(u) rounds down to 2^-60; the chunk's lanes
    add the eps terms in groups first, and cacc(u) rounds up."""
    depth_u = 24
    plans = {"u": [1] * (depth_u - 1), "p60": [32] * 12 + [1] * 11, "p84": [32] * 16 + [16] + [1] * 6,
             "p114": [32] * 22 + [16]}
    s, d, top, v = [], [], {}, 1
    for name, mults in plans.items():
        cs, cd = _chain(v, mults)
        s.append(cs)
        d.append(cd)
        top[name] = v + len(mults)
        v += len(mults) + 1
    a, b = v, v + 1
    e = v + 2 + np.arange(eps)
    u = top["u"]
    s += [np.array([a, a, b, b]), e, e]
    d += [np.array([u, top["p60"], u, top["p84"]]), np.full(eps, u), np.full(eps, top["p114"])]
    return _iso(v + 2 + eps, s, d)


# name -> (builder, root): the root is the vertex the graph is built around (None: the max-degree vertex)
BC_SHAPES = {
    "fans": (fans, 0),
    **{"kab%d_%d" % (a, L - 1): (lambda a=a, L=L: kab(a, L - 1), 0) for a in (32, 33) for L in ROW_LENS},
    "mixed": (mixed, 0),
    "order_chain": (order_chain, 0),
    "back_chain": (back_chain, 0),
    "star70000": (lambda: S.star(70000), 0),
    "star1025_last": (lambda: S.star(1025, True), 1025),
    "hub33": (lambda: S.hub_block(33), S.K_TILE_V + 3),
    "hub64": (lambda: S.hub_block(64), S.K_TILE_V + 3),
    "multi_loop": (S.multi_loop, 0),
    "path600": (lambda: S.path(600), 0),
    "clique200": (lambda: S.clique(200), 0),
    "union": (lambda: S.union([S.star(1025, True), S.empty(7), S.path(256), S.clique(33), S.hub_block(33)],
                              seed=5), None),
    "empty1": (lambda: S.empty(1), 0),
    "empty1025": (lambda: S.empty(1025), 0),
    "pad65537": (lambda: S.pad_to(S.union([S.star(4097), S.path(300)]), S.HUB_FIRST_MIN_V + 1), 0),
}
# graphs whose sums round, so that their results depend on the order of the additions
ORDER_SENSITIVE = ["order_chain", "back_chain"]


def sources(n, rp, col, root):
    """The root, the max-degree vertex, a smallest-positive-degree vertex, an isolated vertex, a depth-1
    neighbour of the max-degree vertex and an absent oid (n + 5), without repeats."""
    rp = np.asarray(rp, dtype=np.int64)
    deg = np.diff(rp)
    out = [] if root is None else [int(root)]
    if n:
        hub = int(np.argmax(deg))
        out.append(hub)
        pos = np.flatnonzero(deg > 0)
        if len(pos):
            out.append(int(pos[np.argmin(deg[pos])]))
        iso = np.flatnonzero(deg == 0)
        if len(iso):
            out.append(int(iso[-1]))
        nb = np.asarray(col[rp[hub]:rp[hub + 1]], dtype=np.int64)
        nb = nb[nb != hub]
        if len(nb):
            out.append(int(nb[len(nb) // 2]))
    out.append(n + 5)
    return list(dict.fromkeys(out))


# ---------------------------------------------------------------- host replicas of the step stats ----
def forward_steps(n, rp, col, depth, direction_opt):
    """(mode, entries) of forward levels 0..L as k_bc_fused records them.  Discovery of level d + 1 is
    chosen as at app_bc.cu:252-256: the first pull is taken when the entries of level d exceed the
    unvisited entries / 14 (integer division), and the pull is kept while (|level d| + 1) * 24 > n.
    Entries: a push reads every row of level d; a pull probes each unvisited row up to its first
    level-d neighbour (the whole row when there is none); levels d + 1 >= 2 add their sigma gather,
    which reads every row of the new level."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    deg = np.diff(rp)
    m = int(rp[-1])
    reached = depth != BO.INF
    if not reached.any():
        return []
    L = int(depth[reached].max())
    levels = [np.flatnonzero(depth == d) for d in range(L + 1)]
    msum = [int(deg[lv].sum()) for lv in levels]
    out = [(0, 0)]
    phase, m_f = 0, msum[0]
    visited = m_f
    for d in range(L):
        if direction_opt:
            phase = int(m_f > (m - visited) // 14) if phase == 0 else int((len(levels[d]) + 1) * 24 > n)
        e = msum[d] if phase == 0 else pull_probes(rp, col, depth, d)
        if d + 1 >= 2:
            e += msum[d + 1]
        out.append((phase, e))
        m_f = msum[d + 1]
        visited += m_f
    return out


def pull_probes(rp, col, depth, d):
    """Entries the pull discovery of level d + 1 reads: every vertex deeper than d (or unreached) scans
    its row up to and including its first neighbour at depth d."""
    u = np.flatnonzero(depth > d)
    if len(u) == 0:
        return 0
    deg = rp[u + 1] - rp[u]
    own, nb = BO._entries(rp, col, u)
    if len(own) == 0:
        return 0
    row = np.repeat(np.arange(len(u)), deg)
    pos = np.arange(len(own)) - np.repeat(np.concatenate([[0], np.cumsum(deg)[:-1]]), deg)
    hit = depth[nb] == d
    first = deg.copy()
    np.minimum.at(first, row[hit], pos[hit] + 1)
    return int(first.sum())


def backward_entries(rp, depth):
    """Entries of the backward gather of levels 0..L: every row of the level."""
    deg = np.diff(np.asarray(rp, dtype=np.int64))
    reached = depth != BO.INF
    if not reached.any():
        return []
    return np.bincount(depth[reached], weights=deg[reached], minlength=int(depth[reached].max()) + 1) \
        .astype(np.int64).tolist()


# --------------------------------------------------------------------------- path-taken checks ----
def reach_checks(name, n, rp, col, root):
    """(what, reached) pairs: on the CSR (rp, col) -- the fragment's own -- from `root`, the graph has the
    geometry it is there for."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    deg = np.diff(rp)
    _, depth = BO.levels_of(n, rp, col, root)
    out = []

    def rows_at(d):
        return deg[depth == d]

    if name == "fans":
        for L in ROW_LENS:
            out.append(("a depth-2 row of %d entries" % L, bool(np.any(rows_at(2) == L))))
        few = [v for v in np.flatnonzero((depth == 2) & (deg > K_BC_CHUNK))
               if len(np.unique(col[rp[v]:rp[v + 1]])) <= 3]
        out.append(("long depth-2 rows of parallel edges to three vertices", len(few) >= 3))
        out.append(("a long depth-1 row (backward gather)", bool(np.any(rows_at(1) > K_BC_CHUNK))))
    if name.startswith("kab"):
        a, b = (int(x) for x in name[3:].split("_"))
        out.append(("depth-2 rows of %d entries" % a, bool(np.all(rows_at(2) == a)) and len(rows_at(2)) == b))
        out.append(("depth-1 rows of %d entries" % (b + 1), bool(np.all(rows_at(1) == b + 1))))
    if name == "mixed":
        r = rows_at(2)
        nch = (r + K_BC_CHUNK - 1) // K_BC_CHUNK
        out.append(("short depth-2 rows", bool(np.any(r <= K_BC_SHORT))))
        for k in (1, 2, 3):
            out.append(("depth-2 long rows of %d chunks" % k, bool(np.any((r > K_BC_SHORT) & (nch == k)))))
    if name in ORDER_SENSITIVE:
        c, sigma, depth = BO.bc_rows(n, rp, col, root)
        big = sigma > TWO_53
        if name == "order_chain":
            for L in (K_BC_SHORT, K_BC_CHUNK):
                v = np.flatnonzero((deg == L) & (depth >= 2) & (depth != BO.INF))
                ok = any(bool(np.all(big[col[rp[x]:rp[x + 1]]])) for x in v)
                out.append(("a sigma gather of %d entries past 2^53" % L, ok))
        else:
            out.append(("a backward row of %d entries" % K_BC_CHUNK, bool(np.any(rows_at(24) == K_BC_CHUNK))))
            out.append(("sigma past 2^100 at depth 25", bool(np.any(sigma[depth == 25] > 2.0 ** 100))))
    if name == "star70000":
        out.append(("a pull level from the centre", any(m == 1 for m, _ in forward_steps(n, rp, col, depth, 1))))
        leaf = BO.levels_of(n, rp, col, 1)[1]
        out.append(("a pull level from a leaf", any(m == 1 for m, _ in forward_steps(n, rp, col, leaf, 1))))
    if name in ("hub33", "hub64"):
        # push only: every level with a row over kHubDeg goes through the hub phase
        pushed = [np.flatnonzero(depth == d) for d in range(int(depth[depth != BO.INF].max()))]
        longest = max(int(np.sum(deg[lv] > S.K_HUB_DEG)) for lv in pushed)
        out.append(("a push level with a row over kHubDeg", longest >= 1))
        if name == "hub64":
            # a level of at most K_TILE_V vertices is one queue tile whatever order discovery listed it in
            crowded = [lv for lv in pushed if len(lv) <= S.K_TILE_V and np.sum(deg[lv] > S.K_HUB_DEG) > S.K_MAX_TILE_HUBS]
            out.append(("a push level (one tile) with more than kMaxTileHubs rows over kHubDeg", len(crowded) > 0))
    if name == "path600":
        out.append(("2 (L + 1) steps past GL_MAX_STEP_STATS", 2 * (int(depth[depth != BO.INF].max()) + 1) > 512))
    if name.startswith("empty"):
        out.append(("no edges", int(rp[-1]) == 0))
    if name == "pad65537":
        out.append(("more than 65536 vertices", n > S.HUB_FIRST_MIN_V))
    return out
