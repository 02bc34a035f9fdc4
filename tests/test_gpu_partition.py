"""Every app on fragments handed to gl_frag_create the way a C++ host hands them over: explicit oids,
lids in any order, several fragments that are not oid blocks (tests/partition_cases.py).

* One fragment from Fragment.from_csr with its lids in a seeded permutation of R-MAT 12 and R-MAT 17
  (at 2^17 vertices the one-fragment BFS takes the hub-first order and PageRank's f32 pull its
  shared-memory hub table): oid2lid, result_oids, every app against the oracles, BFS / SSSP / BC from the
  largest row, lid 0, lid ivnum-1 and an unknown oid, and save / load.
* The model against the library's own builder on the block partition, array for array.
* 2 and 3 fragments on one device (mgpu_partition_worker.py) under the hash, map, skew and hollow
  partitions, with an exact count of OK lines."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bc_oracle as BO
from oracle import core_oracle as CO
from oracle import kclique_oracle as KO
from oracle import pyoracle
from tests import mgpu_partition_worker as W
from tests import partition_cases as P
from tests.util import pkg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT64_MAX = np.iinfo(np.int64).max
F64_MAX = np.finfo(np.float64).max


class OneFragment:
    """R-MAT `scale` (integer weights) with oids 7i + 3 on one fragment whose lids are a seeded
    permutation, plus the same fragment with real weights for the f64 SSSP."""

    def __init__(self, scale):
        self.n = n = 1 << scale
        self.src, self.dst, w = pkg().rmat_edges_host(scale, 16, 17, 1)
        w_real = pkg().rmat_edges_host(scale, 16, 17, 2)[2]
        self.oids = 7 * np.arange(n, dtype=np.int64) + 3
        self.owner = np.zeros(n, dtype=np.int64)
        self.key = np.random.default_rng([P.SEED, scale]).permutation(n)
        self.L = P.describe(n, self.src, self.dst, w, self.oids, False, self.owner, self.key, 1)
        self.L_real = P.describe(n, self.src, self.dst, w_real, self.oids, False, self.owner, self.key, 1)
        self.frag = P.from_layout(pkg(), self.L, 0, False)
        self.frag_real = P.from_layout(pkg(), self.L_real, 0, False)
        self.g = pyoracle.Graph(n, self.src, self.dst, w.astype(np.float64))
        self.g_real = pyoracle.Graph(n, self.src, self.dst, w_real.astype(np.float64))
        self.inner = self.L.frags[0]["inner"]                 # vertex index of each lid
        deg = P.degrees(n, self.src, self.dst)
        # sources as vertex indices: the largest row, lid 0, lid ivnum-1, an oid not in the graph
        self.sources = {"maxdeg": int(np.argmax(deg)), "lid0": int(self.inner[0]), "lidlast": int(self.inner[-1]),
                        "unknown": None}

    def source_oid(self, role):
        s = self.sources[role]
        return -4 if s is None else int(self.oids[s])

    def by_index(self, lid_values):
        """Values in lid order -> values in vertex-index (= oid) order."""
        out = np.empty_like(lid_values)
        out[self.inner] = lid_values
        return out

    def close(self):
        self.frag.close()
        self.frag_real.close()


_ONE = {}


@pytest.fixture(scope="module", params=[12, 17])
def one(request):
    if request.param not in _ONE:
        _ONE[request.param] = OneFragment(request.param)
    yield _ONE[request.param]


def teardown_module():
    for o in _ONE.values():
        o.close()
    _ONE.clear()


def _run(frag, kind, vm=None, **cfg):
    app = pkg().App(kind, frag, **cfg)
    if vm is not None:
        app.set_vertex_map(vm)
    app.query()
    out = app.result()
    oids = app.result_oids() if kind != "kclique" else None
    app.close()
    return out, oids


def test_one_fragment_ids(one):
    f, L = one.frag, one.L
    assert f.ivnum == one.n and f.ovnum == 0
    io = L.frags[0]["inner_oids"]
    assert np.any(np.diff(io) < 0)                         # lids are not in oid order
    assert all(f.oid2lid(o) == lid for lid, o in enumerate(io))
    for o in (-4, 0, 4, 5, int(io.max()) + 7, int(io.max()) + 1, -(1 << 62)):
        assert f.oid2lid(o) is None
    rp, col, w = f.csr(0)
    mrp, mcol, mw = L.frags[0]["oe"]
    assert np.array_equal(rp, mrp) and np.array_equal(col, mcol) and P.same_weights(rp, col, w, mw)
    assert f.max_degree_vertex()[0] == int(np.argmax(np.diff(mrp.astype(np.int64))))
    _, ro = _run(f, "bfs", source_oid=one.source_oid("maxdeg"))
    assert np.array_equal(ro, io)


def test_one_fragment_rejects_a_repeated_oid():
    n = 64
    src = np.arange(n - 1)
    dst = src + 1
    oids = np.random.default_rng(1).permutation(n).astype(np.int64) * 5
    L = P.describe(n, src, dst, None, oids, False, np.zeros(n, np.int64), np.arange(n), 1)
    d = L.frags[0]
    bad = d["inner_oids"].copy()
    bad[40] = bad[3]
    with pytest.raises(pkg().GrapeError, match="appears twice"):
        pkg().Fragment.from_csr(n, d["oe"][0], d["oe"][1], inner_oids=bad)
    f = pkg().Fragment.from_csr(n, d["oe"][0], d["oe"][1], inner_oids=d["inner_oids"])
    assert [f.oid2lid(o) for o in d["inner_oids"]] == list(range(n))
    f.close()


@pytest.mark.parametrize("role", ["maxdeg", "lid0", "lidlast", "unknown"])
@pytest.mark.parametrize("dopt,fuse", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_one_fragment_bfs(one, role, dopt, fuse):
    s = one.sources[role]
    got, _ = _run(one.frag, "bfs", source_oid=one.source_oid(role), direction_opt=dopt, fuse_supersteps=fuse)
    want = np.full(one.n, INT64_MAX) if s is None else one.g.bfs(s)[0]
    assert np.array_equal(one.by_index(got), want)


@pytest.mark.parametrize("role", ["maxdeg", "lid0", "lidlast", "unknown"])
@pytest.mark.parametrize("f64", [0, 1])
def test_one_fragment_sssp(one, role, f64):
    """f32 on integer weights and f64 on real weights: both exact against the f64 oracle."""
    s = one.sources[role]
    frag, g = (one.frag_real, one.g_real) if f64 else (one.frag, one.g)
    got, _ = _run(frag, "sssp", source_oid=one.source_oid(role), sssp_f64=f64)
    want = np.full(one.n, F64_MAX) if s is None else g.sssp(s)[0]
    assert np.array_equal(one.by_index(got), want)


@pytest.mark.parametrize("role", ["maxdeg", "lid0", "lidlast", "unknown"])
@pytest.mark.parametrize("dopt", [0, 1])
def test_one_fragment_bc(one, role, dopt):
    """Bit for bit against the kernel's summation order on the fragment's own rows (lid order)."""
    s = one.sources[role]
    got, _ = _run(one.frag, "bc", source_oid=one.source_oid(role), direction_opt=dopt)
    rp, col, _ = one.L.frags[0]["oe"]
    c, sigma, depth = BO.bc_rows(one.n, rp, col, None if s is None else int(one.L.lid[s]))
    assert np.array_equal(got["depth"], depth)
    assert got["path_num"].tobytes() == sigma.tobytes()
    assert got["centrality"].tobytes() == c.astype(np.float64).tobytes()
    if s is None:
        assert np.all(got["depth"] == BO.INF)
    else:
        assert got["depth"][one.L.lid[s]] == 0


@pytest.mark.parametrize("cfg", [dict(), dict(pr_pull=1), dict(pr_pull=1, reserved={5: 1}),
                                 dict(pr_pull=1, reserved={4: 1, 5: 1})],
                         ids=["push", "pull", "pull_f32", "pull_f32_nohub"])
def test_one_fragment_pagerank(one, cfg):
    got, _ = _run(one.frag, "pagerank", pr_delta=0.85, max_round=10, **cfg)
    got = one.by_index(got)
    want = one.g.pagerank(0.85, 10, 1)
    assert np.max(np.abs(got - want) / want) < 1e-6
    assert abs(got.sum() - 1.0) < (1e-6 if cfg.get("reserved") else 1e-9)


def test_one_fragment_lcc_and_cores(one):
    """LCC orients every edge towards the smaller degree, ties towards the smaller gid (lcc.h does the
    same); on R-MAT's repeated edges that orientation decides the count, so the oracle runs in gid order."""
    L = one.L
    got, _ = _run(one.frag, "lcc")
    want = pyoracle.Graph(one.n, L.rank[one.src], L.rank[one.dst], None).lcc()[0]    # per gid rank = lid
    assert np.array_equal(got, want)
    assert not np.array_equal(one.by_index(got), one.g.lcc()[0])                     # the order matters here
    got, _ = _run(one.frag, "core_decomposition")
    assert np.array_equal(one.by_index(got), CO.core_decomposition(one.n, one.src, one.dst)[0])
    got, _ = _run(one.frag, "kcore", k=3)
    assert np.array_equal(one.by_index(got), CO.kcore(one.n, one.src, one.dst, 3))


@pytest.mark.parametrize("k", [3, 4, 5])
def test_one_fragment_kclique(one, k):
    if one.n > 1 << 12 and k > 3:
        pytest.skip("the host count of 4- and 5-cliques of R-MAT 17 takes minutes; R-MAT 12 runs them")
    got, _ = _run(one.frag, "kclique", k=k)
    assert got == KO.count(one.n, one.src, one.dst, k)


@pytest.mark.parametrize("with_vm", [True, False])
@pytest.mark.parametrize("kind,cfg", [("wcc", {}), ("wcc_opt", {}), ("wcc", dict(reserved={0: 1})),
                                      ("cdlp", dict(max_round=1)), ("cdlp", dict(max_round=5))],
                         ids=["wcc", "wcc_opt", "wcc_dense", "cdlp1", "cdlp5"])
def test_one_fragment_labels(one, kind, cfg, with_vm):
    """Ties break on the smallest gid, here the smallest lid; labels come back as oids through the
    vertex map or, without one, through inner_oids."""
    vm = pkg().VertexMap([one.L.frags[0]["inner_oids"]]) if with_vm else None
    got, _ = _run(one.frag, kind, vm=vm, **cfg)
    if vm is not None:
        vm.close()
    L = one.L
    gr = pyoracle.Graph(one.n, L.rank[one.src], L.rank[one.dst], None)
    lab = gr.cdlp(cfg["max_round"]) if kind == "cdlp" else gr.wcc()[0].astype(np.int64)
    want = one.oids[L.by_rank[lab]]                          # per gid rank (= lid here)
    assert np.array_equal(got, want)
    if kind == "wcc":
        assert not np.array_equal(one.by_index(got), one.oids[one.g.wcc()[0].astype(np.int64)])


def test_one_fragment_save_load(one, tmp_path):
    """gl_frag_load goes through gl_frag_create: the reloaded fragment finds a source whose oid is out of
    sorted position and returns the same depths."""
    io = one.L.frags[0]["inner_oids"]
    lid = int(np.flatnonzero(np.diff(io) < 0)[0]) + 1           # io[lid] < io[lid - 1]
    path = str(tmp_path / "frag.bin")
    one.frag.save(path)
    g = pkg().Fragment.load(path)
    assert g.oid2lid(int(io[lid])) == lid
    a, oa = _run(one.frag, "bfs", source_oid=int(io[lid]))
    b, ob = _run(g, "bfs", source_oid=int(io[lid]))
    g.close()
    assert np.array_equal(a, b) and np.array_equal(oa, ob) and a[lid] == 0
    assert np.array_equal(one.by_index(a), one.g.bfs(int(one.inner[lid]))[0])


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("fnum", [1, 2, 3])
def test_model_equals_library_blocks(fnum, directed):
    """On the block partition the model's descriptors are what gl_frag_build_from_edges builds."""
    n = 1 << 11
    src, dst, w = pkg().rmat_edges_host(11, 16, 9, 1)
    oids = 7 * np.arange(n, dtype=np.int64) + 3
    owner, key = P.blocks(n, fnum)
    L = P.describe(n, src, dst, w, oids, directed, owner, key, fnum)
    for fid in range(fnum):
        f = pkg().Fragment.from_edges(n, oids[src], oids[dst], w, directed=directed, oids=oids, fid=fid, fnum=fnum)
        d = L.frags[fid]
        assert (f.ivnum, f.ovnum, f.total_vnum) == (d["ivnum"], d["ovnum"], n)
        for which, k in ((0, "oe"), (1, "ie" if directed else "oe")):
            rp, col, ww = f.csr(which)
            mrp, mcol, mw = d[k]
            assert np.array_equal(rp, mrp) and np.array_equal(col, mcol)
            assert P.same_weights(rp, col, ww, mw)
        vrp, vcol, _ = f.csr(2)
        assert np.array_equal(vrp, d["ovie"][0]) and np.array_equal(vcol, d["ovie"][1])
        assert np.array_equal(f.ovgid(), d["ovgid"])
        assert all(f.oid2lid(o) == lid for lid, o in enumerate(d["inner_oids"][:200]))
        f.close()


@pytest.mark.parametrize("nproc", [2, 3])
def test_partitions_one_device(nproc):
    env = dict(os.environ, GL_ONE_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29620 + nproc),
           os.path.join(ROOT, "tests", "mgpu_partition_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    bad = [l for l in p.stdout.splitlines() if "MISMATCH" in l or "Error" in l]
    sys.stdout.write("\n".join(bad[:60]) + "\n" + p.stdout[-3000:])
    assert p.returncode == 0, "\n".join(bad[:60]) + p.stdout[-3000:]
    assert p.stdout.count(" OK") == W.expected_ok(nproc), p.stdout[-3000:]
