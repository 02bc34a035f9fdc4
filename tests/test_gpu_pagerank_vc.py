"""PageRank on vertex-cut fragments on the GPU (csrc/vcfrag.cu, csrc/app_pagerank_vc.cu): every case of
tests/pagerank_vc_cases.py and R-MAT 12 / 16 / 20 against the scipy oracle (oracle/pagerank_vc_oracle.py),
agreement with GL_APP_PAGERANK pull on the edge-cut fragment of the same R-MAT 16 edges, bit-identical
repeated queries, the refusals, exact statistics, every case of the reference's stored outputs
(tests/golden/ref_pagerank_vc_outputs.*, p2p-31 included) on one fragment, and 2 x 2 / 3 x 3 fragment
grids against the oracle and the reference's 4- and 9-fragment outputs (mgpu_pagerank_vc_worker.py)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pagerank_vc_oracle as V
from tests import pagerank_vc_cases as RC
from tests.pagerank_vc_cases import pagerank_vc_cases
from tests.util import pkg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = pagerank_vc_cases()


def run(frag, delta, R):
    app = pkg().App("pagerank_vc", frag, pr_delta=delta, max_round=R)
    st = app.query()
    out = app.result()
    oids = app.result_oids()
    app.close()
    return out, oids, st


def close(got, want):
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("R", [0, 1, 10])
@pytest.mark.parametrize("delta", [0.85, 0.5])
def test_cases_one_fragment(name, R, delta):
    n, s, d = CASES[name]
    frag = pkg().VcFragment.from_edges(n, s, d)
    got, oids, st = run(frag, delta, R)
    assert np.array_equal(oids, np.arange(n))
    close(got, V.pagerank_vc(n, s, d, delta, R))
    want = V.stats(n, s, d, 1, R)[0]
    assert st.supersteps == want["supersteps"]
    assert st.entries_scanned == want["entries_scanned"]
    assert st.frontier_vertices == want["frontier_vertices"]
    assert st.touched_vertices == want["touched_vertices"]
    assert st.msg_bytes_sent == 0
    assert list(st.step_entries[1:st.n_steps]) == want["step_entries"]
    assert list(st.step_frontier[1:st.n_steps]) == want["step_frontier"]
    assert all(m == 2 for m in st.step_mode[1:st.n_steps])
    info = frag.info
    assert info["block_edges"] == len(s) and info["entries"] == 2 * len(s) and info["local_vnum"] == n
    frag.close()


REF_META, REF = RC.ref_pagerank_vc_outputs()


@pytest.mark.parametrize("name", sorted(RC.ref_cases()))
def test_one_fragment_against_reference_fixtures(name):
    """Every fixture case, p2p-31 (isolated oid 0) and R-MAT 12 included, at every R and d, against the
    reference's one-fragment output."""
    n, s, d = RC.ref_cases()[name]
    frag = pkg().VcFragment.from_edges(n, s, d)
    idx = RC.sample_index(n) if name in RC.LARGE else np.arange(n)
    for R in RC.REF_ROUNDS:
        for delta in RC.REF_DELTAS:
            got, _, _ = run(frag, delta, R)
            key = RC.ref_key(name, R, delta, 1)
            close(got[idx], REF[key])
            np.testing.assert_allclose(got.sum(), REF_META["sums"][key], rtol=1e-9)
    frag.close()


@pytest.mark.parametrize("scale", [12, 16, 20])
def test_rmat_against_oracle(scale):
    P = pkg()
    s, d, _ = P.rmat_edges_host(scale, 16, seed=3)
    n = 1 << scale
    frag = P.VcFragment.rmat(scale, 16, seed=3)
    assert frag.info["block_edges"] == len(s)
    got, _, _ = run(frag, 0.85, 10)
    close(got, V.pagerank_vc(n, s, d, 0.85, 10))
    frag.close()


def test_rmat16_equals_edge_cut_pagerank_pull():
    P = pkg()
    frag = P.VcFragment.rmat(16, 16, seed=5)
    vc, _, _ = run(frag, 0.85, 10)
    ec = P.Fragment.rmat(16, 16, seed=5)
    app = P.App("pagerank", ec, pr_pull=1, pr_delta=0.85, max_round=10)
    app.query()
    close(vc, app.result())
    app.close()
    ec.close()
    frag.close()


def test_repeated_queries_and_two_apps_are_bit_identical():
    P = pkg()
    frag = P.VcFragment.rmat(14, 16, seed=9)
    a = P.App("pagerank_vc", frag, max_round=10)
    b = P.App("pagerank_vc", frag, max_round=10)
    a.query()
    r1 = a.result().copy()
    a.query()
    r2 = a.result().copy()
    b.query()
    r3 = b.result()
    assert r1.tobytes() == r2.tobytes() == r3.tobytes()
    a.close()
    b.close()
    frag.close()


def test_refusals():
    P = pkg()
    L = P.lib()
    n, s, d = CASES["n_103"]
    for fnum in (2, 3, 5, 8):
        with pytest.raises(P.GrapeError):
            P.VcFragment.from_edges(n, s, d, fid=0, fnum=fnum)
    with pytest.raises(P.GrapeError):
        P.VcFragment.from_edges(n, np.append(s, n), np.append(d, 0))
    with pytest.raises(P.GrapeError):
        P.VcFragment.from_edges(n, np.append(s, 0), np.append(d, -1))
    frag = P.VcFragment.from_edges(n, s, d)
    h = C.c_void_p()
    cfg = P.AppConfig()
    L.gl_app_config_default(C.byref(cfg))
    for kind in (0, 3, 11, 13):
        assert L.gl_vc_app_create(C.byref(h), kind, frag.h, None, C.byref(cfg)) == -2
    ec = P.Fragment.from_edges(n, s, d)
    assert L.gl_app_create(C.byref(h), 12, ec.h, None, C.byref(cfg)) == -2
    app = P.App("pagerank_vc", frag)
    assert L.gl_app_set_vertex_map(app.h, None) == -2
    app.close()
    ec.close()
    frag.close()


def test_two_by_two_layout_on_one_process():
    """Fragments of a 2 x 2 grid built side by side: ranges and block edges equal the host partition."""
    P = pkg()
    n, s, d = CASES["n_103"]
    blk = V.block_of(n, 4, s, d)
    for p in V.partition(n, 4):
        frag = P.VcFragment.from_edges(n, s, d, fid=p["fid"], fnum=4)
        info = frag.info
        assert (info["master_begin"], info["master_end"]) == p["master"]
        assert (info["src_begin"], info["src_end"]) == p["src"]
        assert (info["dst_begin"], info["dst_end"]) == p["dst"]
        assert info["local_vnum"] == p["local_vnum"]
        assert info["block_edges"] == int((blk == p["fid"]).sum())
        frag.close()


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nproc", [4, 9])
def test_fragment_grid(nproc):
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29690 + nproc),
           os.path.join(ROOT, "tests", "mgpu_pagerank_vc_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-prvc] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
