"""Betweenness centrality on the GPU (csrc/app_bc.cu): depth and sigma bit for
bit against the digests of the reference CPU app (tests/golden/ref_bc_outputs.json)
on every case of tests/bc_cases.py, and depth, sigma and c bit for bit against
the order-exact oracle (oracle/bc_oracle.py bc_rows) on the fragment's own CSR;
R-MAT 16 and 20 the same way; repeated queries and push-only discovery
bit-identical; and fragment groups (mgpu_bc_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bc_oracle as BO
from tests import golden_io as G
from tests import shapes as S
from tests.bc_cases import bc_cases, max_degree_index, ref_bc_outputs
from tests.test_gpu_bc_shapes import check_exact
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = bc_cases()
REF = ref_bc_outputs()


def run(frag, source, **cfg):
    app = pkg().App("bc", frag, source_oid=int(source), **cfg)
    st = app.query()
    out = app.result()
    steps = [(st.step_frontier[i], st.step_mode[i]) for i in range(st.n_steps)]
    stats = dict(supersteps=st.supersteps, launches=st.kernel_launches, scanned=st.entries_scanned,
                 reached=st.frontier_vertices, steps=steps)
    app.close()
    return out, stats


def oracle_of(frag, source):
    """bc_rows on the fragment's own CSR (lids are vertex indices in ascending-oid order)."""
    rp, col, _ = frag.csr(0)
    return BO.bc_rows(frag.ivnum, rp, col, frag.oid2lid(source))


def check_stats(st, depth, launches=1):
    reached = int(np.count_nonzero(depth != BO.INF))
    levels = int(depth[depth != BO.INF].max()) + 1 if reached else 0
    assert st["launches"] == launches
    assert st["supersteps"] == 2 * levels
    assert st["reached"] == reached
    # steps 0..L: forward levels, then the backward levels L..0, as far as the step arrays reach
    sizes = np.bincount(depth[depth != BO.INF], minlength=levels).tolist() if reached else []
    want = (sizes + sizes[::-1])[:pkg().GL_MAX_STEP_STATS]
    assert [f for f, _ in st["steps"]] == want
    assert all((m == 2) == (i >= levels) for i, (_, m) in enumerate(st["steps"]))
    if 2 * levels <= pkg().GL_MAX_STEP_STATS:
        assert sum(f for f, m in st["steps"] if m != 2) == reached


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_digests(name):
    n, src, dst, oids, source = CASES[name]
    want = REF[name]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    got, st = run(frag, source)
    exact = oracle_of(frag, source)
    depth = exact[2]
    assert G.digest(got["depth"]) == want["depth"]
    if name.startswith("diamond_chain"):
        # past 2^53 a sum of path counts rounds, and sigma is the kernel's order (check_exact below)
        assert exact[1].max() > 2.0 ** 53
    else:
        assert G.digest(got["path_num"]) == want["sigma"]
    check_exact(got, exact)
    check_stats(st, depth)
    # a second query on another app object is bit-identical
    again, _ = run(frag, source)
    assert again.tobytes() == got.tobytes()
    frag.close()


@pytest.mark.parametrize("scale", [16, 20])
def test_rmat(scale):
    n, s, d, _ = rmat_graph(scale, seed=1)
    source = max_degree_index(n, s, d)
    frag = pkg().Fragment.rmat(scale, 16, seed=1)
    app = pkg().App("bc", frag, source_oid=source)
    app.query()
    got = app.result()
    check_exact(got, oracle_of(frag, source))
    # two queries on one app are bit-identical
    app.query()
    assert app.result().tobytes() == got.tobytes()
    modes = [app.stats.step_mode[i] for i in range(app.stats.n_steps)]
    app.close()
    assert 1 in modes, "the maximum-degree source should reach a pull level"
    # push-only discovery finds the same level sets, so every gather and the whole result are identical
    push, st = run(frag, source, direction_opt=0)
    assert push.tobytes() == got.tobytes()
    assert all(m != 1 for _, m in st["steps"])
    frag.close()


def test_directed_fragment_is_refused_weighted_accepted():
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    with pytest.raises(pkg().GrapeError) as e:
        pkg().App("bc", frag, source_oid=0)
    assert "status 1" in str(e.value) or "undirected" in str(e.value)
    frag.close()
    w = np.linspace(1.0, 2.0, len(s))
    frag = pkg().Fragment.from_edges(n, s, d, w)
    got, _ = run(frag, 0)
    assert got["depth"].tolist() == list(range(n))
    assert got["centrality"].tolist() == [float(n - 1 - v) for v in range(n)]
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
           "--master-addr", "127.0.0.1", "--master-port", str(29590 + nproc),
           os.path.join(ROOT, "tests", "mgpu_bc_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-bc] runs=")]
    assert runs, p.stdout[-4000:]
    assert p.stdout.count(" OK") == int(runs[-1].split("=")[1]) > 0
    # the graphs whose sums round, a fan and long backward rows, each from at least its root and an absent oid
    for name in ("order_chain", "back_chain", "fans", "kab33_2048"):
        assert sum(l.startswith("[mgpu-bc] %s " % name) and l.endswith(" OK") for l in p.stdout.splitlines()) >= 2, name
