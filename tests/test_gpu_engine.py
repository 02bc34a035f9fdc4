"""GPU: the C-ABI engine primitives — ForEachOutgoingEdge over a
WorkSourceArray in every load-balancing mode of the reference
(--lb none|cm|wm|cta|strict, parallel_engine.h:51-70) give identical results,
equal to a numpy restatement."""
import math
import zlib

import numpy as np
import pytest

from oracle import pyoracle
from tests import shapes as S
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
LBS = ["none", "cm", "wm", "cta", "strict", "cmold"]
INF32 = np.uint32(0xFFFFFFFF)


@pytest.fixture(scope="module")
def graph():
    n, src, dst, w = rmat_graph(13, seed=4, weight_mode=1)
    g = pyoracle.Graph(n, src, dst, w.astype(np.float64))
    frag = pkg().Fragment.rmat(13, 16, seed=4, weight_mode=1)
    rp, col, ww = g.csr()
    yield n, g, frag, rp, col, ww
    frag.close()


@pytest.mark.parametrize("lb", LBS)
def test_bfs_level_by_level(graph, lb):
    """Expanding the frontier queue level by level with GL_OP_BFS_LEVEL
    reproduces the oracle's depths; scanned entries = sum of frontier degrees."""
    P = pkg()
    n, g, frag, rp, col, _ = graph
    want, _ = g.bfs(g.max_degree_vertex())
    level = np.full(n, INF32, dtype=np.uint32)
    src = g.max_degree_vertex()
    level[src] = 0
    d_level = P.DeviceArray(level)
    words = (n + 31) // 32
    d_bm = P.DeviceArray(nbytes=4 * words)
    d_q = P.DeviceArray(nbytes=4 * n)
    frontier = np.array([src], dtype=np.uint32)
    depth = 0
    while len(frontier):
        d_q.upload(frontier)
        d_bm.fill(0)
        scanned = P.edge_scan_queue(frag, d_q, len(frontier), "bfs_level", lb, state=d_level,
                                    out_bitmap=d_bm, depth=depth + 1)
        assert scanned == int((rp[frontier + 1] - rp[frontier]).sum())
        cnt = P.compact_bitmap(d_bm, n, d_q)
        frontier = np.sort(d_q.download(np.uint32, cnt))
        depth += 1
        assert np.array_equal(frontier, np.nonzero(want == depth)[0].astype(np.uint32))
    got = d_level.download(np.uint32, n).astype(np.int64)
    got[got == 0xFFFFFFFF] = np.iinfo(np.int64).max
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------
# Exact one-step results of every op on bipartite covers (tests/shapes.py): the queue is drawn
# from side A, whose rows all point into side B, so the sources never change during the step and
# the result is the Jacobi step whatever order the kernel takes the entries in.
INF_F32 = np.float32(np.finfo(np.float32).max)
EXACT_FRAGS = ["rmat14", "rmat12_directed_f64", "rmat12_unweighted", "rmat12_fid0_of_2"] + sorted(S.ENGINE_SHAPES)
HUB_LIST_M = 1 << 22
QLENS = [0, 1, 31, 32, 33, S.K_TILE_V - 1, S.K_TILE_V, S.K_TILE_V + 1, 3 * S.K_TILE_V + 5]


def _build_exact(name):
    P = pkg()
    kw = {}
    if name.startswith("rmat"):
        scale = 14 if name == "rmat14" else 12
        src, dst, w = P.rmat_edges_host(scale, 16, 9, 1)
        base = (1 << scale, src, dst, w.astype(np.float64) * 8)     # real weights 0..8
        directed = "directed" in name
        n, s, d, w = S.bipartite_cover(base, directed=directed)
        if "unweighted" in name:
            w = None
        if "f64" in name:
            kw["w_dtype"] = np.float64
        if "fid0_of_2" in name:
            kw.update(fid=0, fnum=2)
        frag = P.Fragment.from_edges(n, s, d, w, directed=directed, **kw)
    else:
        n, s, d, w = S.ENGINE_SHAPES[name]()
        frag = P.Fragment.from_edges(n, s, d, w)
    side_a = np.array([l for l in (frag.oid2lid(o) for o in range(0, n, 2)) if l is not None], dtype=np.int64)
    return frag, side_a


@pytest.fixture(scope="module")
def exact_frags():
    built = {}
    yield built
    for frag, _ in built.values():
        frag.close()


def _queues(name, rp, side_a, rng):
    deg = (rp[1:] - rp[:-1]).astype(np.int64)
    qs = {"len%d" % L: rng.choice(side_a, L, replace=L > len(side_a)) for L in QLENS}   # unsorted
    qs["side_a_sorted"] = side_a
    p = rng.permutation(side_a)
    qs["repeats"] = rng.permutation(np.concatenate([p[:500], p[:100], p[:100], p[:3]]))
    longest = side_a[np.argmax(deg[side_a])]
    qs["longest_x32"] = rng.permutation(np.concatenate([np.full(32, longest), p[:40]]))
    # the hub list only grows within a process: enough copies to overflow the list of any
    # fragment up to HUB_LIST_M entries scanned before this one
    pieces = -(-int(deg[longest]) // S.K_HUB_CHUNK)
    if deg[longest] > S.K_HUB_DEG:
        qs["longest_many"] = np.full(S.hub_cap(HUB_LIST_M) // pieces + 1, longest)
    zero = side_a[deg[side_a] == 0]
    if len(zero):
        qs["zero_rows_mixed"] = rng.permutation(np.concatenate([zero[:50], p[:50]]))
        qs["all_zero_rows"] = zero[:100]
    return qs


def _gamma(j, u):
    """Higham's gamma_j: the recursive-summation error bound factor after j roundings."""
    return j * u / (1.0 - j * u)


def _bits(d_bm, tv):
    words = (tv + 31) // 32 + 1
    b = np.unpackbits(d_bm.download(np.uint8, 4 * words), bitorder="little").astype(bool)
    return b[:tv], b[tv:]


def _check_queue(P, frag, csr, tv, q, lb, rng, fail):
    """Every op on one queue, compared exactly (ADD_SCATTER reals: with fsum within the
    recursive-summation bound).  Appends a line to `fail` per mismatch."""
    rp, col, w = csr
    qi = q.astype(np.int64)
    deg = (rp[qi + 1] - rp[qi]).astype(np.int64)
    total = int(deg.sum())
    rows = np.repeat(qi, deg)
    idx = np.repeat(rp[qi].astype(np.int64) - np.concatenate([[0], np.cumsum(deg)[:-1]]), deg) + np.arange(total)
    dst = col[idx].astype(np.int64)
    assert not np.isin(qi, dst).any(), "the queue must not reach its own sources"
    d_q = P.DeviceArray(q.astype(np.uint32)) if len(q) else P.DeviceArray(nbytes=16)
    words = (tv + 31) // 32 + 1
    d_bm = P.DeviceArray(nbytes=4 * words)
    f64w = frag.edata_bytes == 8

    def scan(op, **kw):
        d_bm.fill(0)
        sc = P.edge_scan_queue(frag, d_q, len(q), op, lb, out_bitmap=d_bm, **kw)
        if sc != total:
            fail.append("%s: scanned %d, want %d" % (op, sc, total))

    def bits_equal(op, want_bits):
        got, stray = _bits(d_bm, tv)
        if not np.array_equal(got, want_bits) or stray.any():
            fail.append("%s: out_bitmap differs at %d lids" % (op, int(np.sum(got != want_bits))))

    # COUNT
    d_bm.fill(0)
    sc = P.edge_scan_queue(frag, d_q, len(q), "count", lb)
    if sc != total:
        fail.append("count: scanned %d, want %d" % (sc, total))
    # BFS_LEVEL: unvisited destinations take the depth, exactly once
    lv0 = np.where(rng.random(tv) < 0.5, INF32, rng.integers(0, 50, tv).astype(np.uint32)).astype(np.uint32)
    want = lv0.copy()
    hit = np.unique(dst)
    want[hit[lv0[hit] == INF32]] = 77
    d_lv = P.DeviceArray(lv0)
    scan("bfs_level", state=d_lv, depth=77)
    if not np.array_equal(d_lv.download(np.uint32, tv), want):
        fail.append("bfs_level: depths differ")
    bits_equal("bfs_level", want != lv0)
    for use_w in (0, 1):
        wf = np.zeros(len(col), np.float32) if (w is None or not use_w) else w.astype(np.float32)
        if use_w and f64w:
            for op in ("min_relax_f32", "min_relax_u32"):
                with pytest.raises(P.GrapeError, match="use_weight"):
                    P.edge_scan_queue(frag, d_q, len(q), op, lb, state=d_lv, use_weight=1)
            continue
        # MIN_RELAX_F32 (a tenth of the vertices unreached, FLT_MAX: FLT_MAX + w rounds to FLT_MAX)
        st0 = np.where(rng.random(tv) < 0.1, INF_F32, rng.integers(0, 1000, tv).astype(np.float32) * 0.75)
        st0 = st0.astype(np.float32)
        want = st0.copy()
        np.minimum.at(want, dst, (st0[rows] + wf[idx]).astype(np.float32))
        d_st = P.DeviceArray(st0)
        scan("min_relax_f32", state=d_st, use_weight=use_w)
        if not np.array_equal(d_st.download(np.float32, tv).view(np.uint32), want.view(np.uint32)):
            fail.append("min_relax_f32 use_weight=%d: states differ" % use_w)
        bits_equal("min_relax_f32 use_weight=%d" % use_w, want < st0)
        # MIN_RELAX_U32: unreached (0xFFFFFFFF) sources and sums that saturate at it
        wu = wf.astype(np.uint32).astype(np.uint64)
        r = rng.random(tv)
        u0 = np.where(r < 0.1, 0xFFFFFFFF, np.where(r < 0.2, 0xFFFFFFFF - rng.integers(0, 8, tv),
                                                    rng.integers(0, 1 << 20, tv))).astype(np.uint64)
        cand = np.minimum(u0[rows] + wu[idx], 0xFFFFFFFF)
        want = u0.copy()
        np.minimum.at(want, dst, cand)
        d_u = P.DeviceArray(u0.astype(np.uint32))
        scan("min_relax_u32", state=d_u, use_weight=use_w)
        if not np.array_equal(d_u.download(np.uint32, tv), want.astype(np.uint32)):
            fail.append("min_relax_u32 use_weight=%d: states differ at %d lids"
                        % (use_w, int(np.sum(d_u.download(np.uint32, tv) != want.astype(np.uint32)))))
        bits_equal("min_relax_u32 use_weight=%d" % use_w, want < u0)
        # unreached sources relax nothing
        for op, inf, dt in (("min_relax_f32", INF_F32, np.float32), ("min_relax_u32", INF32, np.uint32)):
            s0 = (rng.integers(0, 1000, tv)).astype(dt)
            s0[qi] = inf
            d_s = P.DeviceArray(s0)
            scan(op, state=d_s, use_weight=use_w)
            got = d_s.download(dt, tv)
            if not np.array_equal(got, s0):
                fail.append("%s use_weight=%d: an unreached source changed %d lids" % (op, use_w, int(np.sum(got != s0))))
            bits_equal("%s use_weight=%d unreached" % (op, use_w), np.zeros(tv, bool))
    # ADD_SCATTER_F64, integer-valued: exact in any order, every repeated entry adds once more
    srcv = rng.integers(-1000, 1000, tv).astype(np.float64)
    dst0 = rng.integers(-50, 50, tv).astype(np.float64)
    want = dst0.copy()
    np.add.at(want, dst, srcv[rows])
    d_src, d_dst = P.DeviceArray(srcv), P.DeviceArray(dst0)
    scan("add_scatter_f64", state=d_src, state2=d_dst)
    if not np.array_equal(d_dst.download(np.float64, tv), want):
        fail.append("add_scatter_f64 integers: sums differ")
    # ADD_SCATTER_F64, reals: k addends into one destination (starting from 0.0, which adds
    # exactly) are k - 1 roundings: |err| <= gamma(k - 1) sum|x|, gamma(j) = j u / (1 - j u),
    # u = 2^-53.  err = got - exact sum, computed by fsum over got and the negated addends (a
    # comparison with the rounded fsum of the addends would add fsum's own half ulp).
    srcv = rng.standard_normal(tv) * 10.0 ** rng.uniform(-3, 3, tv)
    d_src.upload(srcv)
    d_dst.upload(np.zeros(tv))
    scan("add_scatter_f64", state=d_src, state2=d_dst)
    got = d_dst.download(np.float64, tv)
    order = np.argsort(dst, kind="stable")
    ds, xs = dst[order], srcv[rows][order]
    cuts = np.flatnonzero(np.diff(ds)) + 1
    bad = int(np.sum(got[np.setdiff1d(np.arange(tv), ds)] != 0.0))
    for v, x in zip(ds[np.concatenate([[0], cuts])] if len(ds) else [], np.split(xs, cuts) if len(ds) else []):
        err = math.fsum(np.concatenate([[got[v]], -x]))
        if abs(err) > _gamma(len(x) - 1, 2.0 ** -53) * math.fsum(np.abs(x)):
            bad += 1
    if bad:
        fail.append("add_scatter_f64 reals: %d destinations outside the summation bound" % bad)


@pytest.mark.parametrize("lb", LBS)
@pytest.mark.parametrize("name", EXACT_FRAGS)
def test_edge_ops_exact(exact_frags, name, lb):
    """gl_edge_scan_queue on bipartite covers -- R-MAT 14 with real f32 weights, R-MAT 12
    directed with f64 weights and unweighted, fid 0 of a 2-fragment edge cut (rows hold outer
    lids), the star, the hub blocks at both cuts, the multi-edge, rows of degree 1024/1025 and
    8192/8193 and of degree 0 -- with queues of the tile-boundary lengths, unsorted, repeated
    (32 copies of the star centre: more hub items than the hub list holds): every op equals
    the numpy step exactly, and every op scans sum(degree) entries with multiplicity."""
    P = pkg()
    if name not in exact_frags:
        exact_frags[name] = _build_exact(name)
    frag, side_a = exact_frags[name]
    csr = frag.csr()
    rp = csr[0].astype(np.int64)
    tv = frag.ivnum + frag.ovnum
    if name in S.ENGINE_SHAPES:
        checks = S.engine_path_checks(name, rp, side_a)
        assert checks and all(ok for _, ok in checks), [what for what, ok in checks if not ok]
    if name == "star":
        many = _queues(name, rp, side_a, np.random.default_rng(0))["longest_many"]
        assert S.queue_hub_pieces(rp, many, S.K_HUB_DEG_CM) > S.hub_cap(max(HUB_LIST_M, rp[-1]))
    if name == "rmat12_fid0_of_2":
        assert frag.ovnum > 0 and int(csr[1].max()) >= frag.ivnum      # rows hold outer lids
    if name == "rmat12_directed_f64":
        assert frag.directed and frag.edata_bytes == 8
    rng = np.random.default_rng(zlib.crc32((name + lb).encode()))
    fail = []
    for qname, q in _queues(name, rp, side_a, rng).items():
        f = []
        _check_queue(P, frag, csr, tv, np.asarray(q, dtype=np.int64), lb, rng, f)
        fail += ["%s: %s" % (qname, x) for x in f]
    assert not fail, "\n".join(fail)


@pytest.mark.parametrize("nbits", [1, 31, 32, 33, 1023, 1025])
def test_bitmap_containers_ignore_stray_bits(nbits):
    """gl_compact_bitmap, gl_queue_fill_from_bitmap and gl_bitmap_count see exactly the bits
    below n_bits: stray bits past it in the last word (and the word after) never appear."""
    import ctypes as C
    P = pkg()
    L = P.lib()
    rng = np.random.default_rng(nbits)
    bits = rng.random(nbits) < 0.4
    bits[-1] = True
    idx = np.flatnonzero(bits)
    words = np.zeros((nbits + 31) // 32 + 1, dtype=np.uint32)
    np.bitwise_or.at(words, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    if nbits % 32:
        words[nbits >> 5] |= np.uint32(~((1 << (nbits % 32)) - 1) & 0xFFFFFFFF)
    words[-1] = 0xFFFFFFFF
    d_bm = P.DeviceArray(words)
    d_out = P.DeviceArray(nbytes=4 * (nbits + 64))
    cnt = P.compact_bitmap(d_bm, nbits, d_out)
    assert cnt == len(idx)
    assert np.array_equal(np.sort(d_out.download(np.uint32, cnt)), idx.astype(np.uint32))
    c64 = C.c_uint64()
    P.check(L.gl_bitmap_count(None, C.cast(d_bm.ptr, C.POINTER(C.c_uint32)), C.c_uint64(nbits), C.byref(c64)))
    assert c64.value == len(idx)
    q = C.c_void_p()
    P.check(L.gl_queue_create(C.byref(q), C.c_uint32(nbits)))
    try:
        P.check(L.gl_queue_fill_from_bitmap(q, None, C.cast(d_bm.ptr, C.POINTER(C.c_uint32)), C.c_uint32(nbits)))
        size = C.c_uint32()
        P.check(L.gl_queue_size(q, None, C.byref(size)))
        assert size.value == len(idx)
        data, dcount = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        P.check(L.gl_queue_data(q, C.byref(data), C.byref(dcount)))
        got = np.empty(size.value, dtype=np.uint32)
        P.check(L.gl_dev_d2h(got.ctypes.data_as(C.c_void_p), data, C.c_size_t(got.nbytes)))
        assert np.array_equal(np.sort(got), idx.astype(np.uint32))
    finally:
        L.gl_queue_destroy(q)


def test_empty_queue_and_empty_bitmap(graph):
    P = pkg()
    n, g, frag, *_ = graph
    d_q = P.DeviceArray(nbytes=16)
    d_level = P.DeviceArray(np.full(n, INF32, dtype=np.uint32))
    assert P.edge_scan_queue(frag, d_q, 0, "bfs_level", "cm", state=d_level, depth=1) == 0
    d_bm = P.DeviceArray(nbytes=4 * ((n + 31) // 32))
    d_bm.fill(0)
    d_out = P.DeviceArray(nbytes=4 * n)
    assert P.compact_bitmap(d_bm, n, d_out) == 0


def test_face2_containers_queue_varray_prepare():
    """gl_queue_* (Queue), gl_varray_* (VertexArray), gl_bitmap_* (DenseVertexSet), gl_frag_prepare."""
    import ctypes as C
    P = pkg()
    L = P.lib()
    n = 100000
    rng = np.random.default_rng(5)
    bits = rng.random(n) < 0.07
    words = np.zeros((n + 31) // 32 + 1, dtype=np.uint32)
    idx = np.nonzero(bits)[0]
    np.bitwise_or.at(words, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    bm = C.POINTER(C.c_uint32)()
    P.check(L.gl_bitmap_create(C.byref(bm), C.c_uint64(n)))
    P.check(L.gl_dev_h2d(bm, words.ctypes.data_as(C.c_void_p), C.c_size_t(words.nbytes)))
    cnt = C.c_uint64()
    P.check(L.gl_bitmap_count(None, bm, C.c_uint64(n), C.byref(cnt)))
    assert cnt.value == len(idx)
    q = C.c_void_p()
    P.check(L.gl_queue_create(C.byref(q), C.c_uint32(n)))
    P.check(L.gl_queue_fill_from_bitmap(q, None, bm, C.c_uint32(n)))
    size = C.c_uint32()
    P.check(L.gl_queue_size(q, None, C.byref(size)))
    assert size.value == len(idx)
    data, dcount = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
    P.check(L.gl_queue_data(q, C.byref(data), C.byref(dcount)))
    got = np.empty(size.value, dtype=np.uint32)
    P.check(L.gl_dev_d2h(got.ctypes.data_as(C.c_void_p), data, C.c_size_t(got.nbytes)))
    assert np.array_equal(np.sort(got), idx.astype(np.uint32))
    P.check(L.gl_queue_clear(q, None))
    P.check(L.gl_queue_size(q, None, C.byref(size)))
    assert size.value == 0
    L.gl_queue_destroy(q)
    P.check(L.gl_bitmap_clear(None, bm, C.c_uint64(n)))
    P.check(L.gl_bitmap_count(None, bm, C.c_uint64(n), C.byref(cnt)))
    assert cnt.value == 0
    P.check(L.gl_bitmap_destroy(bm))
    va = C.c_void_p()
    vals = rng.random(1000)
    P.check(L.gl_varray_create(C.byref(va), C.c_uint64(1000), 8, 0))
    P.check(L.gl_varray_h2d(va, vals.ctypes.data_as(C.c_void_p), C.c_uint64(1000), 8))
    back = np.empty(1000)
    P.check(L.gl_varray_d2h(va, back.ctypes.data_as(C.c_void_p), C.c_uint64(1000), 8))
    assert np.array_equal(back, vals)
    P.check(L.gl_varray_destroy(va))
    frag = P.Fragment.rmat(8, 16, seed=3)
    P.check(L.gl_frag_prepare(frag.h, 0, 1, 0))
    frag.offload()
    assert L.gl_frag_prepare(frag.h, 0, 1, 0) != 0
    frag.reload()
    frag.close()
