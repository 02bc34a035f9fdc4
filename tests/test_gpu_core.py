"""Core decomposition and k-core on the GPU (csrc/app_core.cu): bit for bit
against the reference CPU apps' digests (tests/golden/ref_core_outputs.json) on
every case of tests/core_cases.py (p2p-31, R-MAT 12 and 20, random multigraphs,
the threshold graphs of tests/shapes.py), and against the CPU oracle
(oracle/core_oracle.py) on R-MAT and more k values, on one fragment (one
cooperative launch per query) and on fragment groups (mgpu_core_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import core_oracle as CO
from tests import golden_io as G
from tests import shapes as S
from tests.core_cases import SHAPES, as_indices, core_cases, ref_core_outputs
from tests.golden_io import load_p2p31
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def run(kind, frag, **cfg):
    app = pkg().App(kind, frag, **cfg)
    st = app.query()
    out = app.result()
    stats = (st.supersteps, st.kernel_launches, st.entries_scanned, st.frontier_vertices)
    app.close()
    return out, stats


_RMAT = {}


def rmat_case(scale):
    if scale not in _RMAT:
        n, s, d, _ = rmat_graph(scale, seed=1)
        core, rounds = CO.core_decomposition(n, s, d)
        _RMAT[scale] = (n, s, d, core, rounds)
    return _RMAT[scale]


CASES = core_cases()
REF = ref_core_outputs()


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_digests(name):
    n, src, dst, oids, _ = CASES[name]
    want = REF[name]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    got, _ = run("core_decomposition", frag)
    assert G.digest(got) == want["core"]
    for k, dg in want["kcore"].items():
        got, _ = run("kcore", frag, k=int(k))
        assert G.digest(got) == dg, k
    frag.close()


def test_p2p31_core_and_kcore():
    oids, s, d, _ = load_p2p31()
    si, di = np.searchsorted(oids, s), np.searchsorted(oids, d)
    n = len(oids)
    frag = pkg().Fragment.from_edges(n, s, d, None, oids=oids)
    want, _ = CO.core_decomposition(n, si, di)
    got, _ = run("core_decomposition", frag)
    assert np.array_equal(got, want)
    assert want.max() == 6
    for k in (0, 3, 6, 7):
        got, _ = run("kcore", frag, k=k)
        assert np.array_equal(got, CO.kcore(n, si, di, k)), k
    frag.close()


@pytest.mark.parametrize("scale", [10, 16, 20])
def test_rmat_core(scale):
    n, s, d, want, rounds = rmat_case(scale)
    frag = pkg().Fragment.rmat(scale, 16, seed=1)
    got, (steps, launches, scanned, peeled) = run("core_decomposition", frag)
    assert np.array_equal(got, want)
    # one cooperative launch per query, whatever the number of levels; the fused peel runs exactly the
    # level-synchronous sub-rounds
    assert launches == 1
    assert steps == rounds
    assert peeled == int(np.count_nonzero(np.diff(frag.csr()[0]).astype(np.int64)))
    assert scanned > 0
    # a second query on the same app object returns the same array
    app = pkg().App("core_decomposition", frag)
    app.query()
    a = app.result()
    app.query()
    assert np.array_equal(app.result(), a)
    app.close()
    frag.close()


@pytest.mark.parametrize("scale", [10, 16])
def test_rmat_kcore(scale):
    n, s, d, core, _ = rmat_case(scale)
    frag = pkg().Fragment.rmat(scale, 16, seed=1)
    mx = int(core.max())
    for k in (0, 1, 2, 16, mx, mx + 1):
        got, (_, launches, _, _) = run("kcore", frag, k=k)
        want = CO.kcore(n, s, d, k)
        assert np.array_equal(got, want), k
        assert np.array_equal(got >= k, core >= k) if k > 0 else True
        assert launches == 1
    frag.close()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shapes(name):
    n, s, d, _ = SHAPES[name]
    frag = pkg().Fragment.from_edges(n, s, d)
    core, rounds = CO.core_decomposition(n, s, d)
    got, (steps, _, _, _) = run("core_decomposition", frag)
    assert np.array_equal(got, core)
    assert steps == rounds
    mx = int(core.max())
    for k in (0, 1, 2, mx, mx + 1):
        got, _ = run("kcore", frag, k=k)
        assert np.array_equal(got, CO.kcore(n, s, d, k)), k
    frag.close()


def test_shapes_reach_the_hub_phase():
    # the hub shapes put rows longer than kHubDeg in the peel frontier, more than kMaxTileHubs of them in one tile
    n, s, d, _ = SHAPES["hub64"]
    rp, _ = CO.undirected_csr(n, s, d)
    assert S.long_rows_per_block(rp) > S.K_MAX_TILE_HUBS
    assert np.diff(rp).max() > S.K_HUB_DEG


def test_directed_fragment_is_refused():
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    for kind, cfg in (("core_decomposition", {}), ("kcore", {"k": 2})):
        with pytest.raises(pkg().GrapeError) as e:
            pkg().App(kind, frag, **cfg)
        assert "status 1" in str(e.value) or "undirected" in str(e.value)
    frag.close()


def test_kcore_needs_k():
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d)
    with pytest.raises(pkg().GrapeError):
        pkg().App("kcore", frag)
    frag.close()


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nproc,one_device", [(2, True), (3, True), (2, False)])
def test_multi_fragment(nproc, one_device):
    if _ngpus() < (1 if one_device else nproc):
        pytest.skip("needs %d GPUs" % nproc)
    env = dict(os.environ, GL_ONE_DEVICE="1" if one_device else "0")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29560 + nproc + (0 if one_device else 5)),
           os.path.join(ROOT, "tests", "mgpu_core_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    assert p.stdout.count(" OK") == 8 * 3, p.stdout[-4000:]   # 8 graphs x (core + kcore at two k)
