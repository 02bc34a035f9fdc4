"""Every app on the constructed threshold graphs of tests/shapes.py, through the C
ABI, against the CPU oracle on the same edge list.

Each test first checks on the CPU, from the fragment's own CSR, that its input
really reaches the kernel branch it is there for (more than kMaxTileHubs long
rows in one tile, a dense tile spanning more than kDenseRows rows, more than
kPrHub vertices, ...), so a shape that stops covering its branch fails instead
of passing quietly."""
import numpy as np
import pytest

from oracle import pyoracle
from tests import shapes as S
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu

INT64_MAX = np.iinfo(np.int64).max

# name -> shape builder; every one of them runs undirected, the ones in DIRECTED also directed
SHAPES = {
    "empty1": lambda: S.empty(1), "empty33": lambda: S.empty(33), "empty1025": lambda: S.empty(1025),
    **{"star%d" % k: (lambda k=k: S.star(k)) for k in (1023, 1024, 1025, 4095, 4096, 4097, 70000)},
    **{"star%d_last" % k: (lambda k=k: S.star(k, True)) for k in (1023, 1024, 1025, 4095, 4096, 4097, 70000)},
    "hub33": lambda: S.hub_block(33), "hub64": lambda: S.hub_block(64),
    **{"path%d" % L: (lambda L=L: S.path(L)) for L in (251, 254, 255, 256, 257, 259)},
    "path5000": lambda: S.path(5000),
    **{"clique%d" % k: (lambda k=k: S.clique(k)) for k in (2, 3, 32, 33, 200)},
    "ring2048_16": lambda: S.ring_lattice(2048, 16), "ring1000_5": lambda: S.ring_lattice(1000, 5),
    "bipartite40_70": lambda: S.complete_bipartite(40, 70),
    "multi_loop": S.multi_loop,
    **{"pad%d" % n: (lambda n=n: S.pad_to(S.union([S.star(4097), S.path(300)]), n))
       for n in (S.HUB_FIRST_MIN_V - 1, S.HUB_FIRST_MIN_V, S.HUB_FIRST_MIN_V + 1)},
    **{"pr%d" % n: (lambda n=n: S.chorded_ring(n, seed=n, hubs=(0, n // 2, n - 1)))
       for n in (S.K_PR_HUB - 1, S.K_PR_HUB, S.K_PR_HUB + 1)},
    "union": lambda: S.union([S.star(1025, True), S.empty(7), S.path(256), S.clique(33), S.hub_block(33)]),
    "union_perm": lambda: S.union([S.star(1025, True), S.empty(7), S.path(256), S.clique(33), S.hub_block(33)],
                                  seed=5),
    "sink4097": lambda: S.sink_heavy(4097), "source4097": lambda: S.source_heavy(4097),
}
DIRECTED = ["star4097", "star4097_last", "hub33", "path256", "union_perm", "sink4097", "source4097", "empty33"]
UNDIRECTED = [k for k in SHAPES if k not in ("sink4097", "source4097")]
PATHS = [k for k in SHAPES if k.startswith("path") and k != "path5000"]


class Built:
    def __init__(self, name, directed, w_dtype):
        self.name, self.directed = name, directed
        self.n, self.src, self.dst, self.w = SHAPES[name]()
        self.frag = pkg().Fragment.from_edges(self.n, self.src, self.dst, self.w, directed=directed,
                                              w_dtype=w_dtype)
        self.g = pyoracle.Graph(self.n, self.src, self.dst, self.w, directed=directed)
        self.rp, _, _ = self.frag.csr(0)
        self.deg = np.diff(self.rp.astype(np.int64))
        assert self.frag.ivnum == self.n

    def sources(self):
        """the largest-degree vertex, a leaf (smallest positive degree) and an isolated vertex"""
        out = [int(self.g.max_degree_vertex())]
        pos = np.flatnonzero(self.deg > 0)
        if len(pos):
            out.append(int(pos[np.argmin(self.deg[pos])]))
        iso = np.flatnonzero(self.deg == 0)
        if len(iso):
            out.append(int(iso[-1]))
        return list(dict.fromkeys(out))


@pytest.fixture(scope="module")
def built():
    cache = {}

    def get(name, directed=False, w_dtype=np.float32):
        key = (name, directed, np.dtype(w_dtype).name)
        if key not in cache:
            cache[key] = Built(name, directed, w_dtype)
        return cache[key]

    yield get
    for b in cache.values():
        b.frag.close()


def _app(kind, frag, **cfg):
    return pkg().App(kind, frag, **cfg)


# ------------------------------------------------------------ path-taken ----
def test_shapes_reach_their_thresholds(built):
    """The fragment's own CSR has the geometry each shape is there for."""
    for name in ("hub33", "hub64", "union"):
        rp = built(name).rp
        assert S.long_rows_per_block(rp) > S.K_MAX_TILE_HUBS, name
        assert S.hub_rows_unaligned(rp) > 0, name
    for name in ("star4095", "star4096", "star4097", "star4097_last", "star70000", "star70000_last", "path5000",
                 "pad65536"):
        assert S.max_dense_tile_rows(built(name).rp) > S.K_DENSE_ROWS, name
    for k in (1023, 1024, 1025, 4095, 4096, 4097, 70000):
        assert built("star%d" % k).deg.max() == k
    assert built("star1024").deg.max() == S.K_HUB_DEG and built("star1025").deg.max() == S.K_HUB_DEG + 1
    assert built("multi_loop").deg.max() > S.K_HUB_DEG
    for n in (S.K_PR_HUB - 1, S.K_PR_HUB, S.K_PR_HUB + 1):
        b = built("pr%d" % n)
        assert b.frag.ivnum == n and np.all(b.deg > 0)
    assert built("pr%d" % (S.K_PR_HUB + 1)).frag.ivnum > S.K_PR_HUB
    for n in (S.HUB_FIRST_MIN_V - 1, S.HUB_FIRST_MIN_V, S.HUB_FIRST_MIN_V + 1):
        assert built("pad%d" % n).frag.ivnum == n
    for n in (1, 33, 1025):
        b = built("empty%d" % n)
        assert b.frag.oe_num == 0 and b.frag.ivnum == n
    # the one-byte BFS result limit: the path depths fall on both sides of it
    depths = [int(built(p).g.bfs(0)[0].max()) for p in PATHS]
    assert min(depths) < S.BFS_U8_MAX_LEVELS - 1 and max(depths) > S.BFS_U8_MAX_LEVELS + 1, depths


# ------------------------------------------------------------------- BFS ----
BFS_CFGS = [(fuse, dopt, order, r6) for fuse in (0, 1) for dopt in (0, 1) for order in (0, 1, 2) for r6 in (0, 1)]


def _bfs_check(b, cfgs):
    pulled = False
    for source in b.sources():
        want, _ = b.g.bfs(source)
        for fuse, dopt, order, r6 in cfgs:
            app = _app("bfs", b.frag, source_oid=source, fuse_supersteps=fuse, direction_opt=dopt,
                       reserved={1: order, 6: r6})
            st = app.query()
            got = app.result()
            assert np.array_equal(got, want), (b.name, source, fuse, dopt, order, r6,
                                               np.flatnonzero(got != want)[:8])
            pulled |= dopt == 1 and any(st.step_mode[i] == 1 for i in range(st.n_steps))
            if r6 == 0 and order == 0:
                app.query()                       # a second query on the same app
                assert np.array_equal(app.result(), want), (b.name, source, fuse, dopt, "second query")
            app.close()
    return pulled


@pytest.mark.parametrize("name", UNDIRECTED)
def test_bfs(built, name):
    b = built(name)
    pulled = _bfs_check(b, BFS_CFGS)
    if name.startswith("star") and b.deg.max() >= 4095:
        assert pulled, "no pull level ran on %s with direction_opt = 1" % name


@pytest.mark.parametrize("name", DIRECTED)
def test_bfs_directed(built, name):
    _bfs_check(built(name, True), [c for c in BFS_CFGS if c[2] != 2])


# ------------------------------------------------------------------ SSSP ----
SSSP_SHAPES = ["star1025", "star1025_last", "star4097", "star70000_last", "hub33", "hub64", "path255", "multi_loop",
               "clique200", "union_perm", "empty33", "pad65537"]


@pytest.mark.parametrize("wdt", [np.float32, np.float64])
@pytest.mark.parametrize("directed,name", [(False, s) for s in SSSP_SHAPES] +
                         [(True, s) for s in ("hub33", "union_perm", "source4097", "star4097_last")])
def test_sssp(built, name, directed, wdt):
    """Integer weights (zeros included): every sum is exact in f32 and f64.  f64 edge data
    is what runs the plain-load hub phase (the TMA phase takes 4-byte weights only)."""
    b = built(name, directed, wdt)
    assert b.frag.edata_bytes == np.dtype(wdt).itemsize
    if name in ("hub33", "hub64"):
        assert S.long_rows_per_block(b.rp) > S.K_MAX_TILE_HUBS and S.hub_rows_unaligned(b.rp) > 0
    for source in b.sources()[:2]:
        want, _ = b.g.sssp(source)
        for f64 in (0, 1):
            for prio in (0.0, 0.5, 1e9):
                app = _app("sssp", b.frag, source_oid=source, sssp_f64=f64, sssp_prio=prio)
                app.query()
                got = app.result()
                assert np.array_equal(got, want), (name, source, f64, prio, np.flatnonzero(got != want)[:8])
                app.close()


@pytest.mark.parametrize("wdt", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["star4097", "hub33", "path255"])
def test_sssp_all_zero_weights(name, wdt):
    """Every weight 0.0: the bucket-width heuristic (32 x mean weight / mean degree) is 0, so
    every relaxation lands in the far bucket and the width never grows; all distances are 0."""
    n, src, dst, w = SHAPES[name]()
    w = np.zeros_like(w)
    frag = pkg().Fragment.from_edges(n, src, dst, w, w_dtype=wdt)
    want, _ = pyoracle.Graph(n, src, dst, w).sssp(int(src[0]))
    for f64 in (0, 1):
        for prio in (0.0, 0.5):
            app = _app("sssp", frag, source_oid=int(src[0]), sssp_f64=f64, sssp_prio=prio)
            app.query()
            assert np.array_equal(app.result(), want), (name, f64, prio)
            app.close()
    frag.close()


# ------------------------------------------------------------------- WCC ----
@pytest.mark.parametrize("name", UNDIRECTED + ["d:" + s for s in DIRECTED])
def test_wcc(built, name):
    directed = name.startswith("d:")
    b = built(name[2:] if directed else name, directed)
    want = b.g.wcc()[0].astype(np.int64)
    for kind, res in (("wcc", {}), ("wcc_opt", {}), ("wcc", {0: 1})):
        app = _app(kind, b.frag, reserved=res)
        app.query()
        got = app.result()
        assert np.array_equal(got, want), (b.name, kind, res, np.flatnonzero(got != want)[:8])
        app.close()


# -------------------------------------------------------------- PageRank ----
PR_VARIANTS = {"push": dict(pr_pull=0), "pull64": dict(pr_pull=1),
               "pull32_hub": dict(pr_pull=1, reserved={5: 1}), "pull32": dict(pr_pull=1, reserved={4: 1, 5: 1})}
PR_SHAPES = ["empty1", "empty33", "empty1025", "star1025", "star4097", "star4097_last", "star70000",
             "star70000_last", "hub33", "hub64", "path5000", "clique33", "bipartite40_70", "multi_loop", "union_perm",
             "pad65536", "pr45055", "pr45056", "pr45057"]


def _pr_check(b, got, delta, rounds, directed):
    if rounds == 0:
        # zero rounds: the initial 1/N, as the reference's GPU app and its
        # pagerank_parallel CPU app return (oracle modes 1 and 2)
        want = np.full(b.n, 1.0 / b.n)
    else:
        want = b.g.pagerank(delta, rounds, 2 if directed else 0)
    assert np.max(np.abs(got - want) / want) < 1e-6, (b.name, delta, rounds)
    if not directed:
        assert abs(got.sum() - 1.0) < 1e-6, (b.name, delta, rounds)


@pytest.mark.parametrize("variant", list(PR_VARIANTS))
@pytest.mark.parametrize("name", PR_SHAPES)
def test_pagerank(built, name, variant):
    b = built(name)
    if name == "pr45057":
        assert b.frag.ivnum > S.K_PR_HUB and np.count_nonzero(b.deg) > S.K_PR_HUB
    if name in ("star4097", "star70000", "path5000"):
        assert S.max_dense_tile_rows(b.rp) > S.K_DENSE_ROWS
    for delta in (0.85, 0.5):
        for rounds in (0, 1, 10):
            app = _app("pagerank", b.frag, pr_delta=delta, max_round=rounds, **PR_VARIANTS[variant])
            app.query()
            _pr_check(b, app.result(), delta, rounds, False)
            app.close()


@pytest.mark.parametrize("name", ["sink4097", "source4097", "star4097_last", "hub33", "union_perm", "empty33"])
def test_pagerank_directed(built, name):
    b = built(name, True)
    for pull in (0, 1):
        for delta in (0.85, 0.5):
            for rounds in (0, 1, 10):
                app = _app("pagerank", b.frag, pr_delta=delta, max_round=rounds, pr_pull=pull)
                app.query()
                _pr_check(b, app.result(), delta, rounds, True)
                app.close()


@pytest.mark.parametrize("scale", [16, 18])
def test_pagerank_f32_hub_pull_rmat(scale):
    """R-MAT above kPrHub vertices: the f32 hub pull gathers from shared memory and global memory."""
    n, src, dst, _ = rmat_graph(scale, seed=2)
    assert n > S.K_PR_HUB
    g = pyoracle.Graph(n, src, dst, None)
    frag = pkg().Fragment.rmat(scale, 16, seed=2)
    assert np.count_nonzero(np.diff(frag.csr(0)[0].astype(np.int64))) > S.K_PR_HUB
    for delta in (0.85, 0.5):
        app = _app("pagerank", frag, pr_delta=delta, max_round=10, **PR_VARIANTS["pull32_hub"])
        app.query()
        got = app.result()
        want = g.pagerank(delta, 10, 0)
        assert np.max(np.abs(got - want) / want) < 1e-6
        assert abs(got.sum() - 1.0) < 1e-6
        app.close()
    frag.close()


# ------------------------------------------------------------------ CDLP ----
@pytest.mark.parametrize("name", UNDIRECTED)
def test_cdlp(built, name):
    b = built(name)
    for rounds in (0, 1, 2, 10):
        app = _app("cdlp", b.frag, max_round=rounds)
        app.query()
        got = app.result()
        want = b.g.cdlp(rounds)
        assert np.array_equal(got, want), (name, rounds, np.flatnonzero(got != want)[:8])
        app.close()


# ------------------------------------------------------------------- LCC ----
@pytest.mark.parametrize("name", UNDIRECTED)
def test_lcc(built, name):
    b = built(name)
    app = _app("lcc", b.frag)
    app.query()
    got = app.result()
    want, _ = b.g.lcc()
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), (name, np.flatnonzero(got != want)[:8])
    app.close()
