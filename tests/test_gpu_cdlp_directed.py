"""Directed CDLP on the GPU (csrc/app_cdlp_directed.cu): every case of tests/cdlp_directed_cases.py after
0, 1, 2, 5 and 10 rounds bit for bit against the oracle, and R-MAT 16 and 18; equal to GL_APP_CDLP on
the undirected fragment of the same edges; equal to the reference's own directed CDLP run live
(run_cuda_app --application cdlp --directed 1 through oracle/_ref/compat/run_compat_app and
oracle/_ref/ref_gpu_driver, skipped when a binary is absent); repeated queries; the refusals; exact
statistics; GL_APP_CDLP unchanged on a directed fragment; a fragment whose lids are out of oid order;
and fragment groups (mgpu_cdlp_directed_worker.py)."""
import gzip
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import stats_model as M
from tests import golden_io as G
from tests import partition_cases as P
from tests import shapes as S
from tests.cdlp_directed_cases import (REF_EXES, ROUNDS, as_indices, cdlp_directed_cases, oracle, run_ref_cdlp,
                                       write_efile_vfile)
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = cdlp_directed_cases()
# the cases the live reference comparison writes out as text files (all but the larger R-MAT graphs)
SMALL = sorted(k for k, c in CASES.items() if len(c[1]) <= 20000 and k != "p2p31")


def vids(n, oids):
    return np.arange(n, dtype=np.int64) if oids is None else np.sort(np.asarray(oids, dtype=np.int64))


def run(frag, rounds, kind="cdlp_directed"):
    app = pkg().App(kind, frag, max_round=rounds)
    st = app.query()
    out = app.result()
    app.query()
    again = app.result()
    app.close()
    return out, again, st


def check_stats(st, want):
    assert st.supersteps == want.supersteps
    assert st.entries_scanned == want.entries_scanned
    assert st.frontier_vertices == want.frontier_vertices
    assert st.touched_vertices == want.touched_vertices
    n = st.n_steps
    assert list(st.step_entries[:n]) == want.step_entries[:n]
    assert list(st.step_frontier[:n]) == want.step_frontier[:n]
    assert list(st.step_mode[:n]) == want.step_mode[:n]


def combined_rp(frag):
    return frag.csr(0)[0].astype(np.int64) + frag.csr(1)[0].astype(np.int64)


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    vid = vids(n, oids)
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True, oids=oids)
    und = pkg().Fragment.from_edges(n, src, dst, oids=oids)
    rp = combined_rp(frag)
    for r in ROUNDS:
        got, again, st = run(frag, r)
        want = vid[oracle(n, s, d, r)]
        assert np.array_equal(got, want), (name, r, np.flatnonzero(got != want)[:10])
        assert np.array_equal(again, got)
        check_stats(st, M.cdlp(rp, r))
        # the same labels as GL_APP_CDLP on the undirected fragment of the same edges
        u, _, _ = run(und, r, "cdlp")
        assert np.array_equal(u, got)
    und.close()
    frag.close()


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(scale):
    n, s, d, _ = rmat_graph(scale, seed=1)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    got, again, st = run(frag, 10)
    assert np.array_equal(got, oracle(n, s, d, 10))
    assert np.array_equal(again, got)
    check_stats(st, M.cdlp(combined_rp(frag), 10))
    frag.close()


def test_long_rows_reach_the_cta_vote():
    """The rmat18 hubs and the threshold case's centres have more in + out entries than the warp vote
    takes (kCdlpdWarpRow = 1024); the threshold case has rows on both sides of the cut."""
    n, src, dst, _ = CASES["threshold"]
    deg = np.bincount(src, minlength=n) + np.bincount(dst, minlength=n)
    assert {1023, 1024, 1025} <= set(deg[200:].tolist())
    n, s, d, _ = rmat_graph(18, seed=1)
    assert (np.bincount(s, minlength=n) + np.bincount(d, minlength=n)).max() > 1024


def test_out_of_oid_order():
    """A fragment from gl_frag_create whose lids follow first appearance, not oid order: ties break on the
    smallest gid (here the smallest lid), with and without a vertex map."""
    n, src, dst, _ = CASES["multigraph1"]
    oids = np.arange(n, dtype=np.int64) * 7 + 3
    owner, key = P.partition("hash", n, src, dst, oids, 1)
    L = P.describe(n, src, dst, None, oids, True, owner, key, 1)
    assert np.any(np.diff(L.frags[0]["inner_oids"]) < 0)
    frag = P.from_layout(pkg(), L, 0, True)
    want_lid = oracle(n, src, dst, 5, rank=L.rank)
    want = oids[want_lid][L.frags[0]["inner"]]
    got, again, _ = run(frag, 5)
    assert np.array_equal(got, want) and np.array_equal(again, got)
    vm = pkg().VertexMap([L.frags[0]["inner_oids"]])
    app = pkg().App("cdlp_directed", frag, max_round=5)
    app.set_vertex_map(vm)
    app.query()
    assert np.array_equal(app.result(), want)
    app.close()
    vm.close()
    frag.close()


def test_refusals():
    n, s, d, _ = S.clique(5)
    frag = pkg().Fragment.from_edges(n, s, d)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("cdlp_directed", frag)
    assert "GL_APP_CDLP" in str(e.value)
    frag.close()
    # a directed fragment created without its in-edges
    rp = np.array([0, 4, 7, 9, 10, 10], dtype=np.uint64)
    col = np.array([1, 2, 3, 4, 2, 3, 4, 3, 4, 4], dtype=np.uint32)
    frag = pkg().Fragment.from_csr(5, rp, col, directed=True)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("cdlp_directed", frag)
    assert "incoming" in str(e.value)
    frag.close()


def test_cdlp_on_a_directed_fragment_is_unchanged():
    """GL_APP_CDLP keeps its out-edge-only meaning on a directed fragment: it returns what it returns on an
    undirected fragment created with the same out-rows, and an in-only vertex keeps its label."""
    n, src, dst, _ = CASES["only_in"]
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True)
    got, again, _ = run(frag, 5, "cdlp")
    rp, col, _ = frag.csr(0)
    same_rows = pkg().Fragment.from_csr(n, rp, col)
    want, _, _ = run(same_rows, 5, "cdlp")
    assert np.array_equal(got, want) and np.array_equal(again, got)
    assert got[0] == 0
    # one round: directed CDLP moves the in-only vertex to its smallest in-label
    one, _, _ = run(frag, 1, "cdlp")
    directed, _, _ = run(frag, 1)
    assert one[0] == 0 and directed[0] == 1
    same_rows.close()
    frag.close()


# ---- the reference's own directed CDLP, run live ----------------------------------------------------------
def _exe(impl):
    exe = REF_EXES[impl]
    if not os.path.exists(exe):
        pytest.skip("%s not built (needs the reference sources at build time)" % os.path.relpath(exe, ROOT))
    return exe


@pytest.fixture(scope="module")
def p2p_files():
    d = tempfile.mkdtemp()
    for f in ("p2p-31.e", "p2p-31.v"):
        with gzip.open(os.path.join(G.GOLDEN, f + ".gz"), "rb") as i, open(os.path.join(d, f), "wb") as o:
            shutil.copyfileobj(i, o)
    yield os.path.join(d, "p2p-31.e"), os.path.join(d, "p2p-31.v")
    shutil.rmtree(d, ignore_errors=True)


def _ours(name, rounds):
    n, src, dst, oids = CASES[name]
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True, oids=oids)
    got, _, _ = run(frag, rounds)
    frag.close()
    return got


@pytest.mark.parametrize("impl,lb", [("compat", "cm"), ("compat", "wm"), ("compat", "cta"), ("reference-gpu", "cm")])
@pytest.mark.parametrize("np_", [1, 2, 3])
def test_reference_live_p2p31(p2p_files, impl, lb, np_):
    exe = _exe(impl)
    if impl == "reference-gpu" and _ngpus() < np_:
        # the reference's own grape/cuda puts rank r on device r (cudaSetDevice(local rank))
        pytest.skip("the reference's own GPU code needs one GPU per rank")
    want = _ours("p2p31", 10)
    got = run_ref_cdlp(exe, p2p_files[0], p2p_files[1], 10, lb=lb, np_=np_)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]


@pytest.mark.parametrize("impl", ["compat", "reference-gpu"])
def test_reference_live_small_cases(impl):
    exe = _exe(impl)
    tmp = tempfile.mkdtemp()
    try:
        files = {}
        for name in SMALL:
            n, src, dst, oids = CASES[name]
            os.makedirs(os.path.join(tmp, name))
            files[name] = write_efile_vfile(os.path.join(tmp, name), n, src, dst, oids)
        with ThreadPoolExecutor(8) as pool:
            refs = dict(zip(SMALL, pool.map(lambda k: run_ref_cdlp(exe, files[k][0], files[k][1], 10), SMALL)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    bad = [k for k in SMALL if not np.array_equal(refs[k], _ours(k, 10))]
    assert not bad


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nproc", [2, 3])
def test_multi_fragment(nproc):
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29680 + nproc),
           os.path.join(ROOT, "tests", "mgpu_cdlp_directed_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-cdlpd] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
