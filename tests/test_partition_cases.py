"""CPU checks of tests/partition_cases.py, the host model of gl_frag_desc under any partition: every
partition covers each vertex once, every descriptor meets gl_frag_create's preconditions and gives the
edge multiset back, the block partition reproduces the oracle's CSR, and the hash / map rules restate the
reference's partitioners."""
import numpy as np
import pytest

from oracle import pyoracle
from tests import golden_io as G
from tests import partition_cases as P
from tests import shapes as S


def _graphs():
    rng = np.random.default_rng(4)
    n = 300
    src = rng.integers(0, n, 2000)
    dst = (src + rng.integers(1, 40, 2000)) % n
    src = np.concatenate([src, [5, 5, 7]])          # a self loop and a multi-edge
    dst = np.concatenate([dst, [5, 9, 9]])
    src, dst = src[::-1].copy(), dst[::-1].copy()     # first appearance is not index order
    return {"random": (n + 20, src, dst, (np.arange(len(src)) % 7).astype(np.float64)),   # 20 isolated
            "star": S.star(100), "path": S.path(50), "multi_loop": S.multi_loop(copies=50),
            "clique": S.clique(12), "empty": S.empty(9)}


GRAPHS = _graphs()
PARTS = [("blocks", 1), ("blocks", 2), ("blocks", 3), ("hash", 1), ("hash", 2), ("hash", 3), ("map", 2), ("map", 3),
         ("skew", 2), ("skew", 3), ("hollow", 3)]


def _layout(name, part, fnum, directed):
    n, src, dst, w = GRAPHS[name]
    oids = 7 * np.arange(n, dtype=np.int64) + 3
    owner, key = P.partition(part, n, src, dst, oids, fnum)
    return n, src, dst, w, oids, P.describe(n, src, dst, w, oids, directed, owner, key, fnum)


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("part,fnum", PARTS)
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_descriptors(name, part, fnum, directed):
    n, src, dst, w, oids, L = _layout(name, part, fnum, directed)
    # every vertex on exactly one fragment; lids a permutation; ranks a permutation in gid order
    inner = np.concatenate([f["inner"] for f in L.frags])
    assert np.array_equal(np.sort(inner), np.arange(n))
    for f in L.frags:
        assert np.array_equal(L.lid[f["inner"]], np.arange(f["ivnum"]))
        assert np.all(L.owner[f["inner"]] == f["fid"])
        assert np.array_equal(f["inner_oids"], oids[f["inner"]])
    assert np.array_equal(np.sort(L.rank), np.arange(n))
    assert np.array_equal(np.argsort(L.gid, kind="stable"), L.by_rank)
    fo = P.fid_offset(fnum)
    assert np.array_equal(L.gid, (L.owner << fo) | L.lid)
    got = {"oe": [], "ie": []}
    for f in L.frags:
        iv, ov = f["ivnum"], f["ovnum"]
        ovg = f["ovgid"].astype(np.int64)
        # outer lids in ascending gid order, none owned here, every one used by some entry
        assert np.all(np.diff(ovg) > 0) and np.all((ovg >> fo) != f["fid"])
        lid2v = np.concatenate([f["inner"], f["outer"]]).astype(np.int64)
        assert np.array_equal(L.gid[f["outer"]], ovg)
        used = np.zeros(iv + ov, bool)
        for k in ("oe", "ie") if directed else ("oe",):
            rp, col, ww = f[k]
            rp = rp.astype(np.int64)
            col = col.astype(np.int64)
            assert len(rp) == iv + 1 and rp[0] == 0 and np.all(np.diff(rp) >= 0) and rp[-1] == len(col)
            rows = np.repeat(np.arange(iv), np.diff(rp))
            assert np.all(np.diff(col + rows * (1 << 33)) >= 0)        # each row sorted by lid: inner first
            assert np.all(col < iv + ov)
            used[col] = True
            got[k].append(np.stack([oids[f["inner"][rows]], oids[lid2v[col]],
                                    np.zeros(len(col)) if ww is None else ww], 1))
        assert np.all(used[iv:])
        if not directed:
            assert f["ie"] is None
        # the reverse adjacency of the outer copies is the transpose of the outer part of oe
        rp, col, _ = f["oe"]
        rows = np.repeat(np.arange(iv), np.diff(rp.astype(np.int64)))
        pairs = sorted(zip(col[col >= iv].astype(np.int64) - iv, rows[col >= iv]))
        vrp, vcol = f["ovie"]
        assert np.array_equal(np.diff(vrp.astype(np.int64)), np.bincount([p[0] for p in pairs], minlength=ov))
        assert np.array_equal(vcol.astype(np.int64), np.array([p[1] for p in pairs], dtype=np.int64))
    # the rows give the edge multiset back (undirected: both endpoint rows, a self loop twice)
    w0 = np.zeros(len(src)) if w is None else w
    e = np.stack([oids[src], oids[dst], w0], 1)
    er = np.stack([oids[dst], oids[src], w0], 1)

    def ms(a):
        a = np.concatenate(a) if a else np.zeros((0, 3))
        return a[np.lexsort(a.T[::-1])]

    if directed:
        assert np.array_equal(ms(got["oe"]), ms([e]))
        assert np.array_equal(ms(got["ie"]), ms([er]))
    else:
        assert np.array_equal(ms(got["oe"]), ms([e, er]))


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("fnum", [1, 2, 3])
def test_blocks_equal_oracle_csr(fnum, directed):
    """On the block partition the rows, written as global indices, are the oracle's CSR rows (same
    neighbours, same order within the inner and within the outer part)."""
    n, src, dst, w = GRAPHS["random"]
    oids = 7 * np.arange(n, dtype=np.int64) + 3
    g = pyoracle.Graph(n, oids[src], oids[dst], w, directed=directed, oids=oids)
    owner, key = P.blocks(n, fnum)
    L = P.describe(n, src, dst, w, oids, directed, owner, key, fnum)
    assert np.array_equal(L.rank, np.arange(n))
    for k, incoming in (("oe", False), ("ie", True)) if directed else (("oe", False),):
        orp, ocol, _ = g.csr(incoming)
        for f in L.frags:
            rp, col, _ = f[k]
            lo = int(f["inner"][0]) if f["ivnum"] else 0
            hi = lo + f["ivnum"]
            assert np.array_equal(rp.astype(np.int64), orp[lo:hi + 1].astype(np.int64) - int(orp[lo]))
            lid2v = np.concatenate([f["inner"], f["outer"]]).astype(np.int64)
            mine = lid2v[col.astype(np.int64)]
            rows = np.repeat(np.arange(f["ivnum"]), np.diff(rp.astype(np.int64)))
            want = ocol[orp[lo]:orp[hi]].astype(np.int64)
            assert np.array_equal(np.sort(mine + rows * n), np.sort(want + rows * n))
            if fnum == 1:
                assert np.array_equal(col.astype(np.int64), want)
    if not directed:
        rp, col = L.global_csr()
        orp, ocol, _ = g.csr()
        assert np.array_equal(rp, orp.astype(np.int64))
        rows = np.repeat(np.arange(n), np.diff(rp))
        assert np.array_equal(np.sort(col + rows * n), np.sort(ocol.astype(np.int64) + rows * n))


def test_reference_partition_rules():
    # MapPartitioner::Init: ceil(vnum / fnum) per fid, in list order
    assert list(P.map_sizes(4, 3)) == [2, 2, 0]
    assert list(P.map_sizes(7, 3)) == [3, 3, 1]
    assert list(P.map_sizes(6, 3)) == [2, 2, 2]
    owner, key = P.map_part(4, 3)
    assert sorted(np.bincount(owner, minlength=3)) == [0, 2, 2] and np.bincount(owner, minlength=3)[2] == 0
    # the first two vertices of the permuted list on fid 0, in list order
    perm = np.argsort(key)
    assert list(owner[perm]) == [0, 0, 1, 1]
    # HashPartitioner<int64_t>: libstdc++'s std::hash is the identity, reduced as size_t
    oids = np.array([0, 1, 2, 3, 10, 11, -1, -2, (1 << 62) + 1], dtype=np.int64)
    want = [int(o) % (1 << 64) % 3 for o in oids]
    assert list(P.hash_owner(oids, 3)) == want
    # first appearance over (src0, dst0, src1, dst1, ...), vertices without edges last in index order
    src = np.array([4, 2, 4, 0])
    dst = np.array([2, 6, 0, 4])
    key = P.first_appearance(8, src, dst)
    assert list(np.argsort(key)) == [4, 2, 6, 0, 1, 3, 5, 7]
    # hash: lids inside each fid follow first appearance
    owner, key = P.hash_part(8, src, dst, np.arange(8), 2)
    L = P.describe(8, src, dst, None, np.arange(8), False, owner, key, 2)
    assert list(L.frags[0]["inner"]) == [4, 2, 6, 0] and list(L.frags[1]["inner"]) == [1, 3, 5, 7]
    # skew: the 16 largest degrees (ties to the smaller oid) alone on the last fid
    n, s, d, _ = S.star(100)
    s = np.concatenate([s, np.arange(1, 40)])
    d = np.concatenate([d, np.arange(2, 41)])
    oids = np.arange(n, dtype=np.int64)
    owner, _ = P.skew_part(n, s, d, oids, 3)
    assert list(np.flatnonzero(owner == 2)) == [0] + list(range(2, 17))
    assert np.array_equal(owner[owner != 2], oids[owner != 2] % 2)
    # hollow: nothing on fid 1
    owner, _ = P.hollow_part(50, oids[:50])
    assert not np.any(owner == 1) and np.any(owner == 0) and np.any(owner == 2)


def test_p2p31_hash_partition():
    """p2p-31's own oids under the edge-file loader's rule: the fragments are not oid blocks and the
    lids are not in oid order, so oid order, gid order and lid order all differ."""
    oids, s_oid, d_oid, w = G.load_p2p31()
    src, dst = np.searchsorted(oids, s_oid), np.searchsorted(oids, d_oid)
    owner, key = P.hash_part(len(oids), src, dst, oids, 3)
    L = P.describe(len(oids), src, dst, w, oids, False, owner, key, 3)
    assert sum(f["ivnum"] for f in L.frags) == len(oids)
    for f in L.frags:
        assert np.any(np.diff(f["inner_oids"]) < 0)
        assert len(np.unique(f["inner_oids"])) == f["ivnum"]
    assert not np.array_equal(L.rank, np.arange(len(oids)))


def wcc_tie_case():
    """Two components whose smallest oid and smallest gid are different vertices once the fragments
    hold hashed oids with lids in first-appearance order (4 vertices, 2 fragments)."""
    oids = np.array([10, 11, 20, 21], dtype=np.int64)
    src = np.array([2, 1, 3])          # 20 - 11, 11 - 10, and 21 alone with a self loop
    dst = np.array([1, 0, 3])
    owner, key = P.hash_part(4, src, dst, oids, 2)
    return 4, src, dst, oids, P.describe(4, src, dst, None, oids, False, owner, key, 2)


def test_min_gid_and_min_oid_labels_differ():
    n, src, dst, oids, L = wcc_tie_case()
    by_oid = oids[P.min_label_wcc(n, src, dst, oids)]
    by_gid = oids[P.min_label_wcc(n, src, dst, L.gid)]
    assert list(by_oid) == [10, 10, 10, 21]
    assert list(by_gid) == [20, 20, 20, 21]     # fid 0 holds 20 (lid 0, first seen) and 10 (lid 1)
    # and the ranks agree with the gids
    assert np.array_equal(oids[P.min_label_wcc(n, src, dst, L.rank)], by_gid)
    # the oracle on the graph relabelled to gid rank gives the same labels back through rank -> oid
    g = pyoracle.Graph(n, L.rank[src], L.rank[dst], None)
    lab = g.wcc()[0].astype(np.int64)
    assert np.array_equal(oids[L.by_rank[lab[L.rank]]], by_gid)
