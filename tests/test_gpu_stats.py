"""The query statistics every bandwidth figure is computed from (gl_query_stats:
entries_scanned, frontier_vertices, touched_vertices, supersteps and the per-step
arrays), on one fragment, against the host model oracle/stats_model.py evaluated on
the oracle's CSR.  Exact where the definition in include/grape_b200.h is exact
(BFS push, PageRank, CDLP, LCC, k-core, core decomposition's entries, the first
round of WCC), bounds where a counter depends on the order in which threads win
(pull levels, SSSP, WCC, wcc_opt).  Graphs: the threshold shapes of tests/shapes.py
(rows at the tile and long-row cuts are where the tile walk hands a row to the hub
list, which counts it), R-MAT on both sides of the hub-first switch, p2p-31, and a
path deeper than the fused BFS's level table.  No time is asserted anywhere."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import core_oracle, pyoracle
from oracle import stats_model as M
from tests import golden_io as G
from tests import shapes as S
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu

GUARD = 0xA5A5A5A5A5A5A5A5


def _p2p(directed):
    oids, src, dst, w = G.load_p2p31()
    return len(oids), src, dst, w, directed, oids


GRAPHS = {
    "star1024": lambda: S.star(S.K_HUB_DEG), "star1025": lambda: S.star(S.K_HUB_DEG + 1),
    "star1025_last": lambda: S.star(S.K_HUB_DEG + 1, True), "star70000_last": lambda: S.star(70000, True),
    "hub33": lambda: S.hub_block(33), "hub64": lambda: S.hub_block(64),
    "degrees": lambda: S.rows_of_degree([3, S.K_HUB_DEG, S.K_HUB_DEG + 1, 1, 2 * S.K_HUB_CHUNK + 1, 5]),
    "multi_loop": S.multi_loop, "clique33": lambda: S.clique(33), "empty33": lambda: S.empty(33),
    "path256": lambda: S.path(256), "path1000": lambda: S.path(1000),
    "union_perm": lambda: S.union([S.star(1025, True), S.empty(7), S.path(256), S.clique(33), S.hub_block(33)],
                                  seed=5),
    "pad65536": lambda: S.pad_to(S.union([S.star(4097), S.path(300)]), S.HUB_FIRST_MIN_V),
    "rmat12": lambda: rmat_graph(12, seed=7), "rmat17": lambda: rmat_graph(17, seed=3),
    "p2p31": lambda: _p2p(False), "p2p31_directed": lambda: _p2p(True),
    "hub33_directed": lambda: S.hub_block(33) + (True,), "source4097_directed": lambda: S.source_heavy(4097) + (True,),
}
UNDIRECTED = [k for k in GRAPHS if not k.endswith("_directed")]


class Built:
    def __init__(self, name):
        t = GRAPHS[name]()
        self.name = name
        self.n, src, dst, w = t[:4]
        self.directed = len(t) > 4 and bool(t[4])
        oids = t[5] if len(t) > 5 else None
        w = None if w is None else np.asarray(w, dtype=np.float64)
        self.src, self.dst = src, dst
        self.frag = pkg().Fragment.from_edges(self.n, src, dst, w, directed=self.directed, oids=oids)
        self.g = pyoracle.Graph(self.n, src, dst, w, directed=self.directed, oids=oids)
        self.oids = np.arange(self.n, dtype=np.int64) if oids is None else self.g.oids
        if self.g.entries:
            self.rp, self.col, _ = self.g.csr()
        else:
            self.rp, self.col = np.zeros(self.n + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32)
        self.deg = np.diff(self.rp.astype(np.int64))
        self.m = int(self.deg.sum())
        assert self.frag.ivnum == self.n

    def sources(self):
        """the largest row, a smallest non-empty row, the last vertex and (if any) an isolated vertex"""
        out = [int(np.argmax(self.deg))]
        pos = np.flatnonzero(self.deg > 0)
        if len(pos):
            out.append(int(pos[np.argmin(self.deg[pos])]))
        out.append(self.n - 1)
        iso = np.flatnonzero(self.deg == 0)
        if len(iso):
            out.append(int(iso[0]))
        return list(dict.fromkeys(out))


@pytest.fixture(scope="module")
def built():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Built(name)
        return cache[name]

    yield get
    for b in cache.values():
        b.frag.close()


def _guarded_type():
    """gl_query_stats followed by guard words (built on first use: the package loads lazily)."""
    class GuardedStats(C.Structure):
        _fields_ = [("st", pkg().QueryStats), ("guard", C.c_uint64 * 8)]
    return GuardedStats


class Dev:
    """One query's statistics read out of a gl_query_stats that is followed by guard words."""

    def __init__(self, app):
        L = pkg().lib()
        buf = _guarded_type()()
        C.memset(C.byref(buf), 0xA5, C.sizeof(buf))
        before = L.gl_kernel_launch_count()
        pkg().check(L.gl_app_query(app.h, C.byref(buf.st)))
        self.launch_delta = L.gl_kernel_launch_count() - before
        assert list(buf.guard) == [GUARD] * 8, "gl_app_query wrote past gl_query_stats"
        st = buf.st
        for k in ("supersteps", "entries_scanned", "frontier_vertices", "touched_vertices", "kernel_launches",
                  "n_steps", "msg_bytes_sent"):
            setattr(self, k, int(getattr(st, k)))
        n = self.n_steps
        assert 0 <= n <= M.GL_MAX_STEP_STATS
        self.step_entries = [int(x) for x in st.step_entries[:n]]
        self.step_frontier = [int(x) for x in st.step_frontier[:n]]
        self.step_mode = [int(x) for x in st.step_mode[:n]]
        # nothing is reported past n_steps
        assert not any(st.step_entries[n:]) and not any(st.step_frontier[n:]) and not any(st.step_mode[n:])
        assert not any(st.step_ms[n:])

    def __repr__(self):
        return ("Dev(supersteps=%d n_steps=%d entries=%d frontier=%d touched=%d step_entries=%s step_frontier=%s step_mode=%s)"
                % (self.supersteps, self.n_steps, self.entries_scanned, self.frontier_vertices, self.touched_vertices,
                   self.step_entries[:12], self.step_frontier[:12], self.step_mode[:12]))


def _identities(d, max_degree, ctx):
    """What holds for every app: the totals are the sums of the steps, n_steps is capped, a step
    that is not a pull step (those read the rows of the vertices not yet reached) reads at most
    max_degree entries per vertex it expands, the launch counter agrees."""
    assert d.n_steps == min(d.supersteps, M.GL_MAX_STEP_STATS), (ctx, d)
    if d.supersteps <= M.GL_MAX_STEP_STATS:
        assert d.entries_scanned == sum(d.step_entries), (ctx, d)
        assert d.frontier_vertices == sum(d.step_frontier), (ctx, d)
    else:
        assert d.entries_scanned >= sum(d.step_entries) and d.frontier_vertices >= sum(d.step_frontier), (ctx, d)
    for i in range(d.n_steps):
        assert d.step_mode[i] == M.PULL or d.step_entries[i] <= d.step_frontier[i] * max_degree, (ctx, i, d)
    assert d.kernel_launches == d.launch_delta, (ctx, d)


def _same(d, want, ctx):
    """Exact equality with the model, values side by side on failure."""
    msg = "%s\n  model  %r\n  device %r" % (ctx, want, d)
    assert d.supersteps == want.supersteps, msg
    assert d.n_steps == want.n_steps, msg
    assert d.step_frontier == want.step_frontier[:d.n_steps], msg
    assert d.step_entries == want.step_entries[:d.n_steps], msg
    assert d.step_mode == want.step_mode[:d.n_steps], msg
    assert d.entries_scanned == want.entries_scanned, msg
    assert d.frontier_vertices == want.frontier_vertices, msg
    assert d.touched_vertices == want.touched_vertices, msg


def _depths(levels, n):
    want = np.full(n, np.iinfo(np.int64).max, dtype=np.int64)
    for d, l in enumerate(levels):
        want[l] = d
    return want


# ------------------------------------------------------------------- BFS ----
PUSH_CFGS = [dict(fuse_supersteps=f, reserved={1: o}) for f in (0, 1) for o in (0, 1, 2)]


def _bfs_push(b, source, cfgs=PUSH_CFGS, second_query=True):
    want = M.bfs_push(b.rp, b.col, source)
    depths = _depths(M.bfs_levels(b.rp, b.col, source), b.n)
    seen = []
    for cfg in cfgs:
        app = pkg().App("bfs", b.frag, source_oid=int(b.oids[source]), direction_opt=0, **cfg)
        for q in range(2 if second_query else 1):
            d = Dev(app)
            ctx = (b.name, "bfs push", source, cfg, "query %d" % q)
            _identities(d, int(b.deg.max(initial=0)), ctx)
            _same(d, want, ctx)
            assert np.array_equal(app.result(), depths), ctx
        seen.append(d)
        app.close()
    return seen


@pytest.mark.parametrize("name", list(GRAPHS))
def test_bfs_push(built, name):
    b = built(name)
    for source in b.sources():
        _bfs_push(b, source)


def test_bfs_hub_rows_are_counted_once(built):
    """The path-taken side of the hub graphs: their BFS expands rows longer than kHubDeg (counted by
    the hub phase, not by the tile that met them), more than kMaxTileHubs of them in one tile, and a
    row of exactly kHubDeg entries (counted by its tile)."""
    assert built("star1024").deg.max() == S.K_HUB_DEG and built("star1025").deg.max() == S.K_HUB_DEG + 1
    for name in ("hub33", "hub64"):
        assert S.long_rows_per_block(built(name).rp) > S.K_MAX_TILE_HUBS
    d = built("degrees").deg
    assert S.K_HUB_DEG in d and S.K_HUB_DEG + 1 in d and 2 * S.K_HUB_CHUNK + 1 in d
    # from a hub, level 1 is the pool and level 2 every other hub: one tile with more long rows than slots
    b = built("hub64")
    lv = M.bfs_levels(b.rp, b.col, b.sources()[0])
    assert np.count_nonzero(b.deg[lv[2]] > S.K_HUB_DEG) > S.K_MAX_TILE_HUBS
    _bfs_push(b, b.sources()[0], second_query=False)


def test_bfs_absent_source(built):
    b = built("rmat12")
    for fuse in (0, 1):
        app = pkg().App("bfs", b.frag, source_oid=b.n + 5, direction_opt=0, fuse_supersteps=fuse)
        d = Dev(app)
        _identities(d, int(b.deg.max()), ("absent source", fuse))
        # the stepwise query runs one expansion of the empty frontier, the fused kernel none
        assert d.supersteps == (1 if fuse else 2) and d.n_steps == d.supersteps, d
        assert d.entries_scanned == 0 and d.frontier_vertices == 0 and d.touched_vertices == 0, d
        assert not any(d.step_entries) and not any(d.step_frontier) and not any(d.step_mode), d
        app.close()


@pytest.mark.parametrize("source", [0, 500])
def test_bfs_path_deeper_than_the_step_arrays(built, source):
    """1000 levels from the end, 501 from the middle: the per-step arrays stop at
    GL_MAX_STEP_STATS, the totals and supersteps cover the whole query, fused and stepwise agree."""
    b = built("path1000")
    want = M.bfs_push(b.rp, b.col, source)
    assert want.supersteps == (1001 if source == 0 else 502)
    fused, stepwise = [_bfs_push(b, source, [dict(fuse_supersteps=f, reserved={1: 1})])[0] for f in (1, 0)]
    for k in ("supersteps", "n_steps", "entries_scanned", "frontier_vertices", "touched_vertices", "step_entries",
              "step_frontier", "step_mode"):
        assert getattr(fused, k) == getattr(stepwise, k), (k, fused, stepwise)
    if source == 0:
        assert fused.n_steps == M.GL_MAX_STEP_STATS and fused.entries_scanned == 1998 and fused.frontier_vertices == 1000


@pytest.mark.parametrize("name", ["path256", "rmat12", "union_perm"])
def test_bfs_spilled_level_ring(built, name):
    """Four level bitmaps: the fused kernel parks and is relaunched every three levels."""
    b = built(name)
    source = max(range(0, b.n, max(b.n // 16, 1)), key=lambda v: len(M.bfs_levels(b.rp, b.col, v)))
    assert len(M.bfs_levels(b.rp, b.col, source)) > 4
    for d in _bfs_push(b, source, [dict(fuse_supersteps=1, reserved={1: o, 3: 4}) for o in (1, 2)]):
        assert d.launch_delta >= 2, d
    _bfs_push(b, source, [dict(fuse_supersteps=0, reserved={3: 4})])


@pytest.mark.parametrize("name", UNDIRECTED)
def test_bfs_direction_optimising(built, name):
    """direction_opt = 1: the levels' sizes whatever the direction, a push step's entries exactly, a
    pull step's within its bounds; the stepwise query's push / pull sequence equals the rule
    evaluated on the host (the fused kernel estimates the frontier's entries from degree classes, so
    only its choice for level 0, where it knows the source's row, is pinned)."""
    b = built(name)
    nz = int(np.count_nonzero(b.deg))
    pulled = False
    for source in b.sources():
        want = M.bfs_push(b.rp, b.col, source)
        bounds = M.bfs_pull_bounds(b.rp, b.col, source)
        for beta in (0, 3):
            rule = [0] + M.bfs_direction_modes(want.step_frontier[1:], want.step_entries[1:], b.m, b.n, nz,
                                               beta if beta else 24)
            for fuse in (0, 1):
                for order in (1, 2):
                    cfg = dict(fuse_supersteps=fuse, reserved={1: order, 2: beta})
                    app = pkg().App("bfs", b.frag, source_oid=int(b.oids[source]), direction_opt=1, **cfg)
                    d = Dev(app)
                    ctx = "%s\n  model  %r\n  rule %s\n  device %r" % ((b.name, source, cfg), want, rule[:12], d)
                    _identities(d, int(b.deg.max(initial=0)), ctx)
                    assert d.supersteps == want.supersteps and d.n_steps == want.n_steps, ctx
                    assert d.step_frontier == want.step_frontier[:d.n_steps], ctx
                    assert d.frontier_vertices == want.frontier_vertices, ctx
                    assert d.touched_vertices == want.touched_vertices, ctx
                    for i in range(1, d.n_steps):
                        if d.step_mode[i] == M.PUSH:
                            assert d.step_entries[i] == want.step_entries[i], (i, ctx)
                        else:
                            found, most = bounds[i - 1]
                            assert d.step_mode[i] == M.PULL and found <= d.step_entries[i] <= most, (i, ctx)
                    if fuse == 0:
                        assert d.step_mode == rule[:d.n_steps], ctx
                    elif d.n_steps > 1:
                        assert d.step_mode[1] == rule[1], ctx
                    pulled |= M.PULL in d.step_mode
                    app.close()
    if name in ("star70000_last", "rmat12", "rmat17", "clique33"):
        assert pulled, "no pull level on %s" % name


# ------------------------------------------------------- dense-round apps ----
PR_VARIANTS = [dict(pr_pull=0), dict(pr_pull=1), dict(pr_pull=1, reserved={5: 1}), dict(pr_pull=1, reserved={4: 1, 5: 1})]


@pytest.mark.parametrize("name", [k for k in GRAPHS if k not in ("p2p31_directed", "source4097_directed")])
def test_pagerank(built, name):
    b = built(name)
    for variant in PR_VARIANTS:
        for rounds in (0, 1, 3):
            app = pkg().App("pagerank", b.frag, max_round=rounds, **variant)
            for q in range(2):
                d = Dev(app)
                ctx = (b.name, "pagerank", variant, rounds, q)
                _identities(d, int(b.deg.max(initial=0)), ctx)
                _same(d, M.pagerank(b.rp, rounds), ctx)
            app.close()


@pytest.mark.parametrize("name", UNDIRECTED)
def test_cdlp(built, name):
    b = built(name)
    for rounds in (0, 1, 3):
        app = pkg().App("cdlp", b.frag, max_round=rounds)
        for q in range(2):
            d = Dev(app)
            ctx = (b.name, "cdlp", rounds, q)
            _identities(d, int(b.deg.max(initial=0)), ctx)
            _same(d, M.cdlp(b.rp, rounds), ctx)
        app.close()


@pytest.mark.parametrize("name", UNDIRECTED)
def test_lcc(built, name):
    b = built(name)
    app = pkg().App("lcc", b.frag)
    for q in range(2):
        d = Dev(app)
        _identities(d, b.m, (b.name, "lcc", q))
        _same(d, M.lcc(b.rp, b.col), (b.name, "lcc", q))
    app.close()


# ------------------------------------------------------------- peeling ----
@pytest.mark.parametrize("name", [k for k in UNDIRECTED if k != "p2p31"])
def test_core_and_kcore(built, name):
    """The whole peel is PEval's launch: supersteps counts its sub-rounds while n_steps stays 1 and the
    step arrays stay zero, so the counters are in the totals only: entries = the rows of the peeled
    vertices; k-core's frontier = the vertices it removes."""
    b = built(name)
    app = pkg().App("core_decomposition", b.frag)
    first = None
    for q in range(2):
        d = Dev(app)
        assert d.entries_scanned == b.m, (b.name, "core", d)
        assert np.count_nonzero(b.deg) <= d.frontier_vertices <= b.n, (b.name, "core", d)
        assert d.touched_vertices <= b.m and d.kernel_launches == d.launch_delta, (b.name, "core", d)
        assert d.n_steps == 1 and d.step_entries == [0] and d.step_frontier == [0], (b.name, "core", d)
        first = first or d
        assert (d.entries_scanned, d.frontier_vertices, d.supersteps) == \
            (first.entries_scanned, first.frontier_vertices, first.supersteps)
    app.close()
    for k in (1, 2, 3, 34):
        value = core_oracle.kcore(b.n, b.src, b.dst, k)
        app = pkg().App("kcore", b.frag, k=k)
        d = Dev(app)
        ctx = (b.name, "kcore", k, d)
        assert np.array_equal(app.result(), value), ctx
        assert d.entries_scanned == M.kcore_entries(b.rp, value, k), ctx
        assert d.frontier_vertices == int(np.sum(value < k)), ctx
        assert d.touched_vertices <= d.entries_scanned and d.kernel_launches == d.launch_delta, ctx
        assert d.n_steps == 1 and d.step_entries == [0] and d.step_frontier == [0], ctx
        app.close()


# ------------------------------------------- order-dependent apps: bounds ----
@pytest.mark.parametrize("name", ["star1025", "star70000_last", "hub33", "degrees", "multi_loop", "union_perm",
                                  "path256", "rmat12", "p2p31", "hub33_directed", "empty33"])
def test_sssp_bounds(built, name):
    """Relaxations race, so a vertex can be expanded more than once: every reached vertex is
    expanded at least once and, but for the source, written at least once."""
    b = built(name)
    for source in b.sources()[:2]:
        dist, _ = b.g.sssp(source)
        reached = np.flatnonzero(dist < 1e300)
        for f64 in (0, 1):
            for prio in (0.0, 0.5):
                app = pkg().App("sssp", b.frag, source_oid=int(b.oids[source]), sssp_f64=f64, sssp_prio=prio)
                d = Dev(app)
                ctx = (b.name, "sssp", source, f64, prio, len(reached), int(b.deg[reached].sum()), d)
                assert np.array_equal(app.result(), dist), ctx
                _identities(d, int(b.deg.max(initial=0)), ctx)
                assert d.frontier_vertices >= len(reached), ctx
                assert d.entries_scanned >= int(b.deg[reached].sum()), ctx
                assert d.touched_vertices >= len(reached) - 1, ctx
                assert d.step_frontier[1] == 1 and d.step_entries[1] == int(b.deg[source]), ctx
                app.close()
    app = pkg().App("sssp", b.frag, source_oid=b.n + 5)
    d = Dev(app)
    assert d.entries_scanned == 0 and d.frontier_vertices == 0 and d.touched_vertices == 0, d
    app.close()


@pytest.mark.parametrize("name", UNDIRECTED)
def test_wcc_bounds(built, name):
    """Label propagation: round 1 expands every vertex (exact); later rounds depend on which
    label reaches a vertex first.  A vertex that is not the smallest of its component is
    relabelled at least once.  wcc_opt: everything happens in PEval, reported as step 0: two sampled
    entries per vertex plus the rows scanned afterwards."""
    b = built(name)
    comp = b.g.wcc()[0]
    ncomp = len(np.unique(comp))
    for res in ({}, {0: 1}):
        app = pkg().App("wcc", b.frag, reserved=res)
        d = Dev(app)
        ctx = (b.name, "wcc", res, d)
        _identities(d, int(b.deg.max(initial=0)), ctx)
        assert d.supersteps >= 2 and d.step_frontier[1] == b.n and d.step_entries[1] == b.m, ctx
        assert all(f == b.n and e == b.m for f, e, m in zip(d.step_frontier, d.step_entries, d.step_mode)
                   if m == M.DENSE), ctx
        assert d.touched_vertices >= b.n - ncomp, ctx
        app.close()
    app = pkg().App("wcc_opt", b.frag)
    for q in range(2):
        d = Dev(app)
        ctx = (b.name, "wcc_opt", d)
        assert d.supersteps == 1 and d.n_steps == 1 and d.step_frontier == [b.n], ctx
        assert d.entries_scanned == d.step_entries[0] and 2 * b.n <= d.entries_scanned <= 2 * b.n + b.m, ctx
        assert d.touched_vertices == b.n and d.kernel_launches == d.launch_delta, ctx
    app.close()


# ------------------------------------------------------ several fragments ----
@pytest.mark.parametrize("nproc", [2, 3])
def test_fragment_group_one_device(nproc):
    """Two and three fragments on one device (tests/mgpu_stats_worker.py): per rank the statistics of
    push-only BFS (fused, also deeper than the level table, and stepwise), PageRank and CDLP equal the
    fragment's share in the model, the shares add up to the one-fragment values, supersteps agree on every
    rank, and the stepwise BFS sends exactly 4 bytes per outer vertex the model says it reports."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, GL_ONE_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29620 + nproc),
           os.path.join(root, "tests", "mgpu_stats_worker.py")]
    p = subprocess.run(cmd, cwd=root, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-8000:])
    assert p.returncode == 0, p.stdout[-8000:]
    runs = int(re.search(r"runs=(\d+)", p.stdout).group(1))
    assert runs >= 80 and p.stdout.count(" OK") == runs, p.stdout[-8000:]
