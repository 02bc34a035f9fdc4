"""Constructed graphs that sit exactly on the size thresholds of the CUDA kernels.

R-MAT inputs find wrong answers on average graphs but never put a kernel on one
of its own boundaries (tile sizes, long-row cuts, shared-memory table sizes,
the one-byte BFS depth result).  Every generator here targets one of them; the
sizes are written relative to the constants below, which
tests/test_shapes_oracle.py checks against the `constexpr` lines of csrc/.

Every generator returns (n, src, dst, w): vertex ids 0..n-1 (int64 arrays) and
small integer weights as float64, zeros included, so that shortest-path sums
are exact in f32 and f64 alike.
"""
import numpy as np

K_HUB_DEG = 1024           # engine.cuh kHubDeg: rows longer than this go to the hub phase
K_HUB_DEG_CM = 8192        # primitives.cu kHubDegCm: the long-row cut of the queue scan's cm / cmold modes
K_HUB_CHUNK = 1024         # engine.cuh kHubChunk: entries per hub work item
K_TILE_V = 1024            # engine.cuh kTileV: vertices per frontier tile
K_MAX_TILE_HUBS = 32       # engine.cuh kMaxTileHubs: long rows a tile emits cooperatively
K_DENSE_TILE = 4096        # dense.cuh kDenseTile: CSR entries per dense-sweep tile
K_DENSE_ROWS = 1024        # dense.cuh kDenseRows: row pointers a dense tile stages
K_PR_HUB = 45056           # app_pagerank.cu kPrHub: f32 contributions kept in shared memory
HUB_FIRST_MIN_V = 1 << 16  # app_bfs.cu: one-fragment BFS takes the hub-first order from here on
BFS_U8_MAX_LEVELS = 254    # app_bfs.cu Result(): level counts up to this return one byte per vertex


def _weights(m, seed=0):
    """Integer weights 0..4 (a fifth of them 0.0), deterministic in the edge index."""
    return ((np.arange(m, dtype=np.int64) * 7 + seed) % 5).astype(np.float64)


def _out(n, src, dst):
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    return n, src, dst, _weights(len(src))


def empty(n):
    """No edges at all: m = 0, no dense tiles, every app's `if (m)` guard."""
    return _out(n, [], [])


def star(k, centre_last=False):
    """One centre with k leaves (undirected).  The leaves are rows of degree 1,
    so a 4096-entry dense tile spans about 4096 rows (> K_DENSE_ROWS: the
    global-search branch), and the centre row crosses the hub cut (k > K_HUB_DEG)
    and many dense tiles.  The centre is id 0, or the largest id."""
    n = k + 1
    c = n - 1 if centre_last else 0
    return _out(n, np.full(k, c), np.delete(np.arange(n), c))


def hub_block(h, base=K_TILE_V + 3, pool=1200, cut=K_HUB_DEG):
    """h consecutive ids base..base+h-1 inside one K_TILE_V-aligned block, hub i
    with the odd degree cut + 1 + 2i into a shared pool of vertices after
    the block.  h > K_MAX_TILE_HUBS overflows the per-tile hub slots (the
    single-thread hub_push fallback), and the odd degrees make the hub rows --
    and so their work items -- start at offsets that are not multiples of 4.
    cut = K_HUB_DEG_CM puts the rows over the cut of the queue scan's cm mode."""
    assert base // K_TILE_V == (base + h - 1) // K_TILE_V, "hubs must share one tile"
    pool0 = (base // K_TILE_V + 1) * K_TILE_V
    n = pool0 + pool
    s, d = [], []
    for i in range(h):
        deg = cut + 1 + 2 * i
        s.append(np.full(deg, base + i))
        d.append(pool0 + (np.arange(deg) * (i + 1) + i) % pool)   # repeats within a row when deg > pool
    return _out(n, np.concatenate(s), np.concatenate(d))


def path(L):
    """A path of L vertices 0 - 1 - ... - L-1: BFS from an end reaches depth
    L - 1, so L around BFS_U8_MAX_LEVELS puts the level count on both sides of
    the one-byte result.  The degree-2 rows make dense tiles span about 2048
    rows (> K_DENSE_ROWS)."""
    v = np.arange(L - 1)
    return _out(L, v, v + 1)


def clique(k):
    """K_k: every degree ties (LCC orientation tie-break on the id, CDLP
    smallest-label rule); LCC = 1 for k >= 3 with C(k-1, 2) triangles per vertex."""
    i, j = np.triu_indices(k, 1)
    return _out(k, i, j)


def ring_lattice(n, k):
    """Vertex i joined to i+1..i+k (mod n): every degree is 2k, LCC =
    3(k-1) / (2(2k-1)) with 3k(k-1)/2 triangles per vertex when n > 3k."""
    v = np.repeat(np.arange(n), k)
    off = np.tile(np.arange(1, k + 1), n)
    return _out(n, v, (v + off) % n)


def complete_bipartite(a, b):
    """K_{a,b} on ids [0, a) x [a, a+b): no triangles (LCC 0), BFS depths 1 and
    2, and CDLP swaps the two sides' labels every round."""
    i, j = np.meshgrid(np.arange(a), np.arange(a, a + b), indexing="ij")
    return _out(a + b, i.ravel(), j.ravel())


def multi_loop(copies=5000, loops=3):
    """Vertex 0 with `copies` copies of the edge 0-1 (a row far longer than
    K_HUB_DEG made of one neighbour), `loops` self loops, and a few more edges
    that close triangles through the multi-edge: pins the multiplicity rules of
    LCC, CDLP and PageRank on a long row."""
    s = [np.zeros(copies, dtype=np.int64), np.zeros(loops, dtype=np.int64), [0, 1, 2, 2, 4, 4]]
    d = [np.ones(copies, dtype=np.int64), np.zeros(loops, dtype=np.int64), [2, 2, 3, 3, 5, 0]]
    return _out(8, np.concatenate(s), np.concatenate(d))


def chorded_ring(n, seed=0, hubs=(0,), hub_deg=3000):
    """Every vertex on a ring plus one random chord, and a few hubs of degree
    about `hub_deg`: no isolated vertex, so when n > K_PR_HUB the pull gathers
    non-zero contributions both from the shared-memory table and from global
    memory.  `hubs` places the highest-degree ids on both sides of K_PR_HUB."""
    rng = np.random.RandomState(seed)
    v = np.arange(n)
    s = [v, v]
    d =[(v + 1) % n, rng.randint(0, n, size=n)]
    for h in hubs:
        s.append(np.full(hub_deg, h))
        d.append(rng.randint(0, n, size=hub_deg))
    return _out(n, np.concatenate(s), np.concatenate(d))


def pad_to(shape, n):
    """The same edges with isolated vertices appended up to n vertices."""
    n0, src, dst, w = shape
    assert n >= n0
    return n, src, dst, w


def sink_heavy(k):
    """Directed: k sources each with one edge into vertex 0 (in-edges only at the
    centre, which has no out-edge: the dangling rule of directed PageRank)."""
    return _out(k + 1, np.arange(1, k + 1), np.zeros(k))


def source_heavy(k):
    """Directed: vertex 0 with k out-edges and no in-edge; the leaves are sinks."""
    return _out(k + 1, np.zeros(k), np.arange(1, k + 1))


def rows_of_degree(degs, pool=600):
    """Row i has degs[i] entries into a pool of `pool` vertices after the rows
    (cycling, so a row longer than the pool repeats neighbours).  Degrees on both
    sides of a cut (K_HUB_DEG, K_HUB_DEG + 1, K_HUB_DEG_CM, K_HUB_DEG_CM + 1) put
    rows exactly on it; odd degrees before them shift the next row's first entry
    off a multiple of 4."""
    r = len(degs)
    s = [np.full(d, i) for i, d in enumerate(degs)]
    d = [r + (np.arange(k) + 7 * i) % pool for i, k in enumerate(degs)]
    return _out(r + pool, np.concatenate(s), np.concatenate(d))


def bipartite_cover(shape, directed=False):
    """Bipartite double cover: vertex u becomes 2u (side A) and 2u + 1 (side B),
    and every edge u - v becomes 2u - 2v+1 and 2v - 2u+1 (directed: u -> v
    becomes 2u -> 2v+1 only).  Row 2u has the degree (out-degree) of row u, and
    every row of side A points into side B: a queue drawn from side A never
    changes its own sources, so one relaxation step over it is exactly the
    Jacobi step in any order."""
    n, src, dst, w = shape
    if directed:
        return 2 * n, 2 * src, 2 * dst + 1, w
    return 2 * n, np.concatenate([2 * src, 2 * dst]), np.concatenate([2 * dst + 1, 2 * src + 1]), np.concatenate([w, w])


def union(shapes, seed=None):
    """Disjoint union with contiguous id ranges, or (seed given) with the ids
    shuffled by a seeded permutation."""
    offs, s, d, w = [], [], [], []
    n = 0
    for (pn, ps, pd, pw) in shapes:
        offs.append(n)
        s.append(ps + n)
        d.append(pd + n)
        w.append(pw)
        n += pn
    src, dst, ww = np.concatenate(s), np.concatenate(d), np.concatenate(w)
    if seed is not None:
        perm = np.random.RandomState(seed).permutation(n).astype(np.int64)
        src, dst = perm[src], perm[dst]
    return n, src, dst, ww


# ----------------------------------------------------------------------------
# Path-taken checks on a CSR (row pointers of the fragment's own layout)
def long_rows_per_block(rp, block=K_TILE_V, cut=K_HUB_DEG):
    """Most rows longer than `cut` entries in one `block`-aligned id block."""
    deg = np.diff(np.asarray(rp, dtype=np.int64))
    long_ids = np.flatnonzero(deg > cut)
    if len(long_ids) == 0:
        return 0
    return int(np.bincount(long_ids // block).max())


def max_dense_tile_rows(rp, tile=K_DENSE_TILE):
    """Most rows one `tile`-entry tile of the CSR can touch, computed the way
    k_dense_tile_rows / k_dense_pull do (nr = r1 - r0 + 1)."""
    rp = np.asarray(rp, dtype=np.int64)
    nrows, m = len(rp) - 1, int(rp[-1])
    ntiles = (m + tile - 1) // tile
    if ntiles == 0:
        return 0
    e = np.arange(ntiles, dtype=np.int64) * tile
    first = np.searchsorted(rp, e, side="right") - 1       # largest r with rp[r] <= e
    tile_row = np.concatenate([first, [nrows]])
    r1 = np.minimum(tile_row[1:], nrows - 1)
    return int((r1 - tile_row[:-1] + 1).max())


def hub_rows_unaligned(rp, cut=K_HUB_DEG):
    """Number of rows longer than `cut` whose first entry is not 4-aligned."""
    rp = np.asarray(rp, dtype=np.int64)
    deg = np.diff(rp)
    return int(np.sum((deg > cut) & (rp[:-1] % 4 != 0)))


# Path-taken checks of the queue scan (gl_edge_scan_queue, modes cta / cm / cmold): a CTA
# takes K_TILE_V consecutive queue entries; a row longer than the cut becomes ceil(deg /
# K_HUB_CHUNK) hub work items, counted once per queue entry.
def hub_cap(m):
    """Hub work items the queue scan has room for on a fragment of m CSR entries
    (primitives.cu ensure_scratch: m / kHubChunk + m / kHubDeg + 1024)."""
    m = max(int(m), 1)
    return m // K_HUB_CHUNK + m // K_HUB_DEG + 1024


def queue_hub_pieces(rp, q, cut):
    """Hub work items a queue emits: pieces of every long row, per entry."""
    rp = np.asarray(rp, dtype=np.int64)
    deg = (rp[1:] - rp[:-1])[np.asarray(q, dtype=np.int64)]
    return int(np.sum(np.where(deg > cut, (deg + K_HUB_CHUNK - 1) // K_HUB_CHUNK, 0)))


def long_rows_per_queue_tile(rp, q, cut):
    """Most queue entries with a row longer than `cut` in one K_TILE_V-entry queue tile."""
    rp = np.asarray(rp, dtype=np.int64)
    deg = (rp[1:] - rp[:-1])[np.asarray(q, dtype=np.int64)]
    pos = np.flatnonzero(deg > cut)
    return 0 if len(pos) == 0 else int(np.bincount(pos // K_TILE_V).max())


ROW_DEGREES = [3, K_HUB_DEG, K_HUB_DEG + 1, 1, K_HUB_DEG_CM, K_HUB_DEG_CM + 1, 5, K_HUB_DEG + 1, K_HUB_DEG_CM + 1]

# The graphs of the engine-primitive tests (tests/test_gpu_engine.py), all bipartite covers so that
# one relaxation step over a side-A queue is exact.  "degrees" is padded with isolated vertices:
# rows of degree 0.
ENGINE_SHAPES = {
    "star": lambda: bipartite_cover(star(70000)),
    "hub_block": lambda: bipartite_cover(hub_block(33)),
    "hub_block_cm": lambda: bipartite_cover(hub_block(33, cut=K_HUB_DEG_CM)),
    "multi_loop": lambda: bipartite_cover(multi_loop()),
    "degrees": lambda: bipartite_cover(pad_to(rows_of_degree(ROW_DEGREES), len(ROW_DEGREES) + 600 + 40)),
}


def engine_path_checks(name, rp, side_a):
    """(branch, reached) pairs for the engine-primitive case `name`: on CSR rp,
    the sorted side-A queue `side_a` -- or 32 copies of its longest row -- takes
    the queue scan through the branch."""
    rp = np.asarray(rp, dtype=np.int64)
    side_a = np.asarray(side_a, dtype=np.int64)
    deg = rp[1:] - rp[:-1]
    out = []
    if name == "star":
        q = np.full(32, side_a[np.argmax(deg[side_a])])
        for cut in (K_HUB_DEG, K_HUB_DEG_CM):
            out.append(("32 copies of the centre: hub items above hub_cap at cut %d" % cut,
                        queue_hub_pieces(rp, q, cut) > hub_cap(rp[-1])))
    if name in ("hub_block", "hub_block_cm"):
        cut = K_HUB_DEG if name == "hub_block" else K_HUB_DEG_CM
        out.append(("more than %d long rows in one queue tile at cut %d" % (K_MAX_TILE_HUBS, cut),
                    long_rows_per_queue_tile(rp, side_a, cut) > K_MAX_TILE_HUBS))
        out.append(("long rows starting off a 4-aligned entry at cut %d" % cut,
                    queue_hub_rows_unaligned(rp, side_a, cut) > 0))
    if name == "multi_loop":
        out.append(("the 5000-fold multi-edge is one long row", deg[side_a].max() > 5000))
    if name == "degrees":
        for d in (K_HUB_DEG, K_HUB_DEG + 1, K_HUB_DEG_CM, K_HUB_DEG_CM + 1, 0):
            out.append(("a row of degree %d" % d, bool(np.any(deg[side_a] == d))))
        for cut in (K_HUB_DEG, K_HUB_DEG_CM):
            out.append(("long rows starting off a 4-aligned entry at cut %d" % cut,
                        queue_hub_rows_unaligned(rp, side_a, cut) > 0))
    return out


def queue_hub_rows_unaligned(rp, q, cut):
    """Queue entries with a row longer than `cut` whose first entry is not
    4-aligned: their hub items make the TMA hub phase copy from the enclosing
    16-byte boundary."""
    rp = np.asarray(rp, dtype=np.int64)
    q = np.asarray(q, dtype=np.int64)
    deg = rp[q + 1] - rp[q]
    return int(np.sum((deg > cut) & (rp[q] % 4 != 0)))
