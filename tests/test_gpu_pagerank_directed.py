"""Directed PageRank on the GPU (csrc/app_pagerank_directed.cu): every case of
tests/pagerank_directed_cases.py at every d and R of DELTAS x ROUNDS, and R-MAT 16 and 18, against the
oracle and the reference's fixtures (rtol 1e-9); bit-identical output from two queries and two handles;
results that sum to 1; equal to GL_APP_PAGERANK's f64 pull on the undirected fragment when every edge is
given in both directions; the refusals; exact statistics; a fragment whose lids are out of oid order;
and fragment groups (mgpu_pagerank_directed_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import pagerank_directed_cases as P
from tests import partition_cases as PC
from tests import shapes as S
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = P.pagerank_directed_cases()


def run(frag, delta, R):
    """-> (result, stats) of the first query; asserts that a second query and a second handle give the
    same bits."""
    app = pkg().App("pagerank_directed", frag, pr_delta=delta, max_round=R)
    st = app.query()
    out = app.result()
    app.query()
    again = app.result()
    app.close()
    app = pkg().App("pagerank_directed", frag, pr_delta=delta, max_round=R)
    app.query()
    other = app.result()
    app.close()
    assert out.tobytes() == again.tobytes() == other.tobytes(), (delta, R)
    return out, st


def check_stats(st, R, ivnum, ie_entries):
    if R <= 0:
        assert st.supersteps == 1
        assert (st.entries_scanned, st.frontier_vertices, st.touched_vertices, st.msg_bytes_sent) == (0, 0, 0, 0)
        return
    assert st.supersteps == R + 1 and st.n_steps == R + 1
    assert st.entries_scanned == R * ie_entries
    assert st.frontier_vertices == R * ivnum
    assert st.touched_vertices == R * ivnum
    assert st.msg_bytes_sent == 0
    assert list(st.step_entries[:R + 1]) == [0] + [ie_entries] * R
    assert list(st.step_frontier[:R + 1]) == [0] + [ivnum] * R
    assert list(st.step_mode[:R + 1]) == [0] + [2] * R


def check(got, n, s, d, delta, R):
    want = P.pagerank_directed(n, s, d, delta, R)
    if R <= 0:
        assert got.tobytes() == np.zeros(n).tobytes()
        return
    assert np.allclose(got, want, rtol=1e-9, atol=0), (delta, R, np.abs(got - want).max())
    assert abs(got.sum() - 1.0) <= 1e-12, (delta, R, got.sum())


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases(name):
    n, s, d = CASES[name]
    _, refs = P.ref_pagerank_directed_outputs()
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    for delta in P.DELTAS:
        for R in P.ROUNDS:
            got, st = run(frag, delta, R)
            check(got, n, s, d, delta, R)
            check_stats(st, R, n, len(s))
            key = P.ref_key(name, delta, R)
            if key in refs:
                ref = refs[key]
                assert (not ref.any()) if R <= 0 else np.allclose(got, ref, rtol=1e-9, atol=0), key
    frag.close()


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(scale):
    n, s, d, _ = rmat_graph(scale, seed=1)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    got, st = run(frag, 0.85, 10)
    check(got, n, s, d, 0.85, 10)
    check_stats(st, 10, n, len(s))
    frag.close()


@pytest.mark.parametrize("name", ["mixed", "long_rows", "rmat12"])
def test_both_directions_equal_pagerank_pull(name):
    """Every edge given in both directions: the same ranks as GL_APP_PAGERANK's f64 pull on the undirected
    fragment of the edges (a self loop counts twice in both degrees)."""
    if name == "rmat12":
        n, s, d, _ = rmat_graph(12, seed=7)
    else:
        n, s, d = CASES[name]
    und = pkg().Fragment.from_edges(n, s, d)
    both = pkg().Fragment.from_edges(n, np.concatenate([s, d]), np.concatenate([d, s]), directed=True)
    for delta, R in ((0.85, 10), (0.5, 2), (0.85, 1)):
        app = pkg().App("pagerank", und, pr_pull=1, pr_delta=delta, max_round=R)
        app.query()
        want = app.result()
        app.close()
        got, _ = run(both, delta, R)
        assert np.allclose(got, want, rtol=1e-11, atol=0), (delta, R, np.abs(got - want).max())
    both.close()
    und.close()


def test_out_of_oid_order():
    """A fragment from gl_frag_create whose lids follow first appearance, not oid order."""
    n, s, d = CASES["random"]
    oids = np.arange(n, dtype=np.int64) * 7 + 3
    owner, key = PC.partition("hash", n, s, d, oids, 1)
    L = PC.describe(n, s, d, None, oids, True, owner, key, 1)
    assert np.any(np.diff(L.frags[0]["inner_oids"]) < 0)
    frag = PC.from_layout(pkg(), L, 0, True)
    got, _ = run(frag, 0.85, 10)
    want = P.pagerank_directed(n, s, d, 0.85, 10)[L.frags[0]["inner"]]
    assert np.allclose(got, want, rtol=1e-9, atol=0)
    frag.close()


def test_refusals():
    n, s, d, _ = S.clique(5)
    frag = pkg().Fragment.from_edges(n, s, d)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("pagerank_directed", frag)
    assert "GL_APP_PAGERANK" in str(e.value)
    frag.close()
    # a directed fragment created without its in-edges
    rp = np.array([0, 4, 7, 9, 10, 10], dtype=np.uint64)
    col = np.array([1, 2, 3, 4, 2, 3, 4, 3, 4, 4], dtype=np.uint32)
    frag = pkg().Fragment.from_csr(5, rp, col, directed=True)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("pagerank_directed", frag)
    assert "incoming" in str(e.value)
    frag.close()


def test_pr_pull_is_ignored():
    n, s, d = CASES["tier_rows"]
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    a, _ = run(frag, 0.85, 10)
    app = pkg().App("pagerank_directed", frag, pr_delta=0.85, max_round=10, pr_pull=1)
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
           "--master-addr", "127.0.0.1", "--master-port", str(29710 + nproc),
           os.path.join(ROOT, "tests", "mgpu_pagerank_directed_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-prd] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
