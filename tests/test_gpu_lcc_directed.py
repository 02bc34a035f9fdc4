"""Directed local clustering coefficient on the GPU (csrc/app_lcc_directed.cu): every case of
tests/lcc_directed_cases.py bit for bit against the exact oracle (oracle/lcc_directed_oracle.py) and,
where no pair reaches 256 entries, against the digests of the reference's LCCDirected; R-MAT 16 and 18
directed; repeated queries; the refusals; exact statistics (oracle/lcc_directed_oracle.py stats); and
fragment groups (mgpu_lcc_directed_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import lcc_directed_oracle as LO
from tests import golden_io as G
from tests import shapes as S
from tests.lcc_directed_cases import WRAP, as_indices, lcc_directed_cases, ref_lcc_directed_outputs
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = lcc_directed_cases()
REF = ref_lcc_directed_outputs()


def run(frag, kind="lcc_directed"):
    app = pkg().App(kind, frag)
    st = app.query()
    out = app.result()
    again = app.query() and app.result()
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


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True, oids=oids)
    got, again, st = run(frag)
    lcc, tri, deg = LO.lcc_directed(n, s, d)
    assert got.tobytes() == lcc.tobytes()
    assert again.tobytes() == got.tobytes()
    check_stats(st, LO.stats(n, s, d))
    _, rtri, rdeg = LO.lcc_directed(n, s, d, reference=True)
    assert G.digest(rtri) == REF[name]["tri"] and G.digest(rdeg) == REF[name]["d"]
    if name in ("pair256", "pair300"):
        # the reference's uint8_t weight wraps: its tri differs on the two vertices opposite the heavy pair
        assert np.flatnonzero(tri != rtri).tolist() == [2, 3] and np.all((tri - rtri) % WRAP == 0)
        assert not np.array_equal(got, rtri / np.maximum(deg * (deg - 1.0), 1.0))
    else:
        # bit for bit the reference's result: tri / (d (d - 1)) from its digests
        assert np.array_equal(tri, rtri)
    frag.close()


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(scale):
    n, s, d, _ = rmat_graph(scale, seed=1)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    got, again, st = run(frag)
    lcc, _, _ = LO.lcc_directed_fast(n, s, d)
    assert got.tobytes() == lcc.tobytes()
    assert again.tobytes() == got.tobytes()
    check_stats(st, LO.stats(n, s, d))
    frag.close()


def test_refusals():
    n, s, d, _ = S.clique(5)
    frag = pkg().Fragment.from_edges(n, s, d)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("lcc_directed", frag)
    assert "GL_APP_LCC" in str(e.value)
    frag.close()
    # a directed fragment created without its in-edges
    rp = np.array([0, 4, 7, 9, 10, 10], dtype=np.uint64)
    col = np.array([1, 2, 3, 4, 2, 3, 4, 3, 4, 4], dtype=np.uint32)
    frag = pkg().Fragment.from_csr(5, rp, col, directed=True)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("lcc_directed", frag)
    assert "incoming" in str(e.value)
    frag.close()


def test_lcc_on_a_directed_fragment_is_unchanged():
    """GL_APP_LCC keeps its out-edge-only meaning on a directed fragment: it reads the out-rows alone, so
    it returns what it returns on an undirected fragment created with the same rows."""
    n, src, dst, _ = CASES["multigraph1"]
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True)
    got, again, _ = run(frag, "lcc")
    rp, col, _ = frag.csr(0)
    same_rows = pkg().Fragment.from_csr(n, rp, col)
    want, _, _ = run(same_rows, "lcc")
    assert got.tobytes() == want.tobytes()
    assert again.tobytes() == got.tobytes()
    ld, _, _ = run(frag)
    assert ld.tobytes() != got.tobytes()
    same_rows.close()
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
           "--master-addr", "127.0.0.1", "--master-port", str(29670 + nproc),
           os.path.join(ROOT, "tests", "mgpu_lcc_directed_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-lccd] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
