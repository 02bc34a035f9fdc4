"""Un-normalised PageRank on the GPU (csrc/app_pagerank_local.cu): every case of
tests/pagerank_local_cases.py on undirected and directed fragments at every d and R of DELTAS x ROUNDS,
and R-MAT 16 and 18, against the oracle and the reference's one-rank fixtures (rtol 1e-9); bit-identical
output from two queries and two handles; N x GL_APP_PAGERANK's f64 pull on undirected graphs without
zero-degree vertices; the R <= 0 refusal; exact statistics; a fragment whose lids are out of oid order;
and fragment groups (mgpu_pagerank_local_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import pagerank_local_cases as P
from tests import partition_cases as PC
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = P.pagerank_local_cases()


def run(frag, delta, R):
    """-> (result, stats) of the first query; asserts that a second query and a second handle give the
    same bits."""
    app = pkg().App("pagerank_local", frag, pr_delta=delta, max_round=R)
    st = app.query()
    out = app.result()
    app.query()
    again = app.result()
    app.close()
    app = pkg().App("pagerank_local", frag, pr_delta=delta, max_round=R)
    app.query()
    other = app.result()
    app.close()
    assert out.tobytes() == again.tobytes() == other.tobytes(), (delta, R)
    return out, st


def check_stats(st, R, ivnum, oe_entries):
    assert st.supersteps == R + 1 and st.n_steps == R + 1
    assert st.entries_scanned == R * oe_entries
    assert st.frontier_vertices == R * ivnum
    assert st.touched_vertices == R * ivnum
    assert st.msg_bytes_sent == 0
    assert list(st.step_entries[:R + 1]) == [0] + [oe_entries] * R
    assert list(st.step_frontier[:R + 1]) == [0] + [ivnum] * R
    assert list(st.step_mode[:R + 1]) == [0] + [2] * R


def make_frag(n, s, d, dr):
    return pkg().Fragment.from_edges(n, s, d, directed=dr == "directed")


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("dr", P.DIRS)
def test_cases(name, dr):
    n, s, d = CASES[name]
    _, refs = P.ref_pagerank_local_outputs()
    frag = make_frag(n, s, d, dr)
    oe = len(P.rows(n, s, d, dr == "directed")[0])
    assert frag.oe_num == oe
    runs = [P.P2P] if name == "p2p31" else [(dl, R) for dl in P.DELTAS for R in P.ROUNDS]
    for delta, R in runs:
        got, st = run(frag, delta, R)
        want = P.pagerank_local(n, s, d, delta, R, dr == "directed")
        assert np.allclose(got, want, rtol=1e-9, atol=0), (delta, R, np.abs(got - want).max())
        check_stats(st, R, n, oe)
        key = P.ref_key(name, dr, delta, R, 1)
        if key in refs and P.avg_degree(n, s, d, dr == "directed") <= 10:
            assert np.allclose(got, refs[key], rtol=1e-9, atol=0), key
    frag.close()


@pytest.mark.parametrize("scale", [16, 18])
@pytest.mark.parametrize("dr", P.DIRS)
def test_rmat(scale, dr):
    n, s, d, _ = rmat_graph(scale, seed=1)
    frag = make_frag(n, s, d, dr)
    got, st = run(frag, 0.85, 10)
    want = P.pagerank_local(n, s, d, 0.85, 10, dr == "directed")
    assert np.allclose(got, want, rtol=1e-9, atol=0), np.abs(got - want).max()
    check_stats(st, 10, n, len(P.rows(n, s, d, dr == "directed")[0]))
    frag.close()


def _without_isolated(n, s, d):
    deg = np.bincount(np.concatenate([s, d]), minlength=n)
    keep = deg > 0
    remap = np.cumsum(keep) - 1
    return int(keep.sum()), remap[s], remap[d]


@pytest.mark.parametrize("name", ["random", "tier_rows", "long_rows", "rmat12"])
def test_undirected_equals_n_times_pagerank_pull(name):
    """No zero-degree vertex: N x GL_APP_PAGERANK's f64 pull on the same undirected fragment."""
    if name == "rmat12":
        n, s, d, _ = rmat_graph(12, seed=7)
    else:
        n, s, d = CASES[name]
    n, s, d = _without_isolated(n, s, d)
    frag = pkg().Fragment.from_edges(n, s, d)
    for delta, R in ((0.85, 10), (0.5, 2), (0.85, 1)):
        app = pkg().App("pagerank", frag, pr_pull=1, pr_delta=delta, max_round=R)
        app.query()
        want = n * app.result()
        app.close()
        got, _ = run(frag, delta, R)
        assert np.allclose(got, want, rtol=1e-11, atol=0), (delta, R, np.abs(got / want - 1).max())
    frag.close()


def test_out_of_oid_order():
    """Fragments from gl_frag_create whose lids follow first appearance, not oid order."""
    n, s, d = CASES["random"]
    oids = np.arange(n, dtype=np.int64) * 7 + 3
    owner, key = PC.partition("hash", n, s, d, oids, 1)
    for directed in (False, True):
        L = PC.describe(n, s, d, None, oids, directed, owner, key, 1)
        assert np.any(np.diff(L.frags[0]["inner_oids"]) < 0)
        frag = PC.from_layout(pkg(), L, 0, directed)
        got, _ = run(frag, 0.85, 10)
        want = P.pagerank_local(n, s, d, 0.85, 10, directed)[L.frags[0]["inner"]]
        assert np.allclose(got, want, rtol=1e-9, atol=0)
        frag.close()


def test_directed_without_in_edges():
    """A directed fragment created without ie: the app reads the out-rows only."""
    rp = np.array([0, 4, 7, 9, 10, 10], dtype=np.uint64)
    col = np.array([1, 2, 3, 4, 2, 3, 4, 3, 4, 4], dtype=np.uint32)
    s = np.repeat(np.arange(5), np.diff(rp).astype(np.int64))
    frag = pkg().Fragment.from_csr(5, rp, col, directed=True)
    got, _ = run(frag, 0.85, 10)
    assert np.allclose(got, P.pagerank_local(5, s, col.astype(np.int64), 0.85, 10, True), rtol=1e-9, atol=0)
    frag.close()


def test_refuses_no_rounds():
    n, s, d = CASES["mixed"]
    frag = pkg().Fragment.from_edges(n, s, d)
    for R in (0, -1):
        with pytest.raises(pkg().GrapeError) as e:
            pkg().App("pagerank_local", frag, max_round=R)
        assert "max_round" in str(e.value)
    frag.close()


def test_pr_pull_is_ignored():
    n, s, d = CASES["tier_rows"]
    frag = pkg().Fragment.from_edges(n, s, d)
    a, _ = run(frag, 0.85, 10)
    app = pkg().App("pagerank_local", frag, pr_delta=0.85, max_round=10, pr_pull=1)
    app.query()
    assert app.result().tobytes() == a.tobytes()
    app.close()
    frag.close()


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
           "--master-addr", "127.0.0.1", "--master-port", str(29730 + nproc),
           os.path.join(ROOT, "tests", "mgpu_pagerank_local_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-prl] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
