"""Betweenness centrality over a list of sources on the GPU (csrc/app_bc_sources.cu): bit for bit
against the order-exact oracle (oracle/bc_sources_oracle.py) on every case of tests/bc_cases.py, on the
BC threshold shapes and on R-MAT; bit-identical across batch widths, queries, handles and a list set
again; each source's delta against GL_APP_BC's f32 c; the refusals; the exact statistics; and fragment
groups (mgpu_bc_sources_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bc_sources_oracle as BSO
from tests import bc_shapes as BS
from tests import shapes as S
from tests.bc_cases import bc_cases, max_degree_index
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = bc_cases()
ALL_VERTICES_MAX_N = 2100
SAME_GRAPH = ("p2p31_src0", "rmat12_deg1", "rmat12_absent")   # graphs another case already lists


def seeded_sources(n, s, d, k, seed, oids=None):
    """k sources: the maximum-degree vertex first, then a seeded sample (repeats allowed), as oids."""
    rng = np.random.default_rng(seed)
    idx = [max_degree_index(n, s, d)] + rng.integers(0, n, size=k - 1).tolist()
    return [int(oids[i]) if oids is not None else int(i) for i in idx]


def run(frag, sources, **cfg):
    app = pkg().App("bc_sources", frag, sources=sources, **cfg)
    st = app.query()
    got = app.result()
    stats = dict(supersteps=st.supersteps, frontier=st.frontier_vertices, touched=st.touched_vertices,
                 scanned=st.entries_scanned, steps=[(st.step_frontier[i], st.step_mode[i]) for i in range(st.n_steps)])
    app.close()
    return got, stats


def oracle_of(frag, sources):
    """bc_sources on the fragment's own CSR; sources: a list of oids, or None for every vertex in lid order."""
    rp, col, _ = frag.csr(0)
    n = frag.ivnum
    if sources is None:
        lids = list(range(n))
    else:
        lids = [frag.oid2lid(o) for o in sources]
    return BSO.bc_sources(n, rp, col, lids) + (lids,)


def check_stats(st, want, lids, B):
    per = want["per_source"]
    batches = [sum(per[i:i + B]) for i in range(0, len(per), B)]
    assert st["supersteps"] == len(batches)
    assert [f for f, _ in st["steps"]] == batches[:pkg().GL_MAX_STEP_STATS]
    assert all(m == 2 for _, m in st["steps"])
    assert st["frontier"] == want["frontier_vertices"]
    assert st["touched"] == want["touched_vertices"]
    if want["touched_vertices"] > 0:
        assert st["scanned"] > 0


def check(frag, sources, **cfg):
    got, st = run(frag, sources, **cfg)
    want, stats, lids = oracle_of(frag, sources)
    assert got.tobytes() == want.tobytes(), "max abs diff %g" % float(np.max(np.abs(got - want))) if len(got) else ""
    check_stats(st, stats, lids, cfg.get("reserved", {}).get(0, 32) or 32)
    return got


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases(name):
    n, src, dst, oids, source = CASES[name]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    if name in SAME_GRAPH:
        pass
    elif n <= ALL_VERTICES_MAX_N:
        check(frag, None)
    else:
        from tests.core_cases import as_indices
        s, d = as_indices(n, src, dst, oids)
        check(frag, seeded_sources(n, s, d, 256, seed=5, oids=oids))
    check(frag, [source])
    frag.close()


def test_rmat12_seeded_and_special_lists():
    n, src, dst, oids, _ = CASES["rmat12"]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    lst = seeded_sources(n, src, dst, 256, seed=7)
    check(frag, lst)
    check(frag, lst[:5] + lst[:5] + [lst[0]])            # duplicates count once per occurrence
    check(frag, [lst[0], 1 << 40, lst[1], -3])          # oids that are not vertices contribute nothing
    check(frag, [lst[3]])
    got = check(frag, [])                                # the empty list
    assert not got.any()
    frag.close()


# R-MAT 20 runs 16 sources: the numpy oracle needs about 4 s per source there
@pytest.mark.parametrize("scale,k", [(16, 256), (20, 16)])
def test_rmat(scale, k):
    n, s, d, _ = rmat_graph(scale, seed=1)
    frag = pkg().Fragment.rmat(scale, 16, seed=1)
    check(frag, seeded_sources(n, s, d, k, seed=scale))
    frag.close()


def test_batch_widths_queries_handles_and_lists():
    n, src, dst, oids, _ = CASES["p2p31_src6"]
    from tests.core_cases import as_indices
    s, d = as_indices(n, src, dst, oids)
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    lst = seeded_sources(n, s, d, 70, seed=3, oids=oids)
    ref = check(frag, lst)
    for B in (1, 7, 32):
        got = check(frag, lst, reserved={0: B})
        assert got.tobytes() == ref.tobytes(), B
    app = pkg().App("bc_sources", frag, sources=lst, reserved={0: 7})
    app2 = pkg().App("bc_sources", frag, sources=lst)
    app.query()
    a = app.result()
    app.query()
    assert app.result().tobytes() == a.tobytes()
    app2.query()
    assert app2.result().tobytes() == a.tobytes()
    app.set_sources(list(lst))
    app.query()
    assert app.result().tobytes() == a.tobytes()
    app.set_sources(lst[1:])
    app.query()
    assert app.result().tobytes() != a.tobytes()
    app.close()
    app2.close()
    frag.close()


def test_delta_matches_bc_f32():
    n, src, dst, oids, _ = CASES["rmat12"]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    for source in seeded_sources(n, src, dst, 3, seed=11):
        got, _ = run(frag, [source])
        app = pkg().App("bc", frag, source_oid=source)
        app.query()
        c = app.result()["centrality"]
        app.close()
        keep = np.arange(n) != frag.oid2lid(source)
        assert np.allclose(got.astype(np.float32)[keep], c[keep], rtol=1e-5, atol=0)
    frag.close()


@pytest.mark.parametrize("name", sorted(BS.BC_SHAPES))
def test_shapes(name):
    build, root = BS.BC_SHAPES[name]
    n, s, d, _ = build()
    frag = pkg().Fragment.from_edges(n, s, d)
    rp, col, _ = frag.csr(0)
    check(frag, BS.sources(n, rp, col, root))
    if n <= 2100:
        check(frag, None, reserved={0: 7})
    frag.close()


def test_refusals():
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    with pytest.raises(pkg().GrapeError):
        pkg().App("bc_sources", frag)
    frag.close()
    frag = pkg().Fragment.from_edges(n, s, d)
    for bad in (-1, 33):
        with pytest.raises(pkg().GrapeError):
            pkg().App("bc_sources", frag, reserved={0: bad})
    app = pkg().App("bc", frag, source_oid=0)
    with pytest.raises(pkg().GrapeError):
        app.set_sources([0])
    app.close()
    app = pkg().App("bc_sources", frag)
    with pytest.raises(pkg().GrapeError):
        app.query()
    app.close()
    frag.close()


def test_hbm_batch_width_hook():
    """reserved[1] stands in for the width free HBM allows: batches of 3, the same bits as any other width."""
    n, src, dst, oids, _ = CASES["rmat12"]
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    lst = seeded_sources(n, src, dst, 20, seed=4)
    want = check(frag, lst, reserved={0: 3})
    got, st = run(frag, lst, reserved={1: 3})
    assert st["supersteps"] == 7
    assert got.tobytes() == want.tobytes()
    with pytest.raises(pkg().GrapeError):
        pkg().App("bc_sources", frag, reserved={1: -1})
    frag.close()


def test_path_values():
    """From one end of a path of n vertices, delta(v) = n - 1 - v."""
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d, np.linspace(1.0, 2.0, len(s)))
    got, st = run(frag, [0])
    assert got.tolist() == [0.0] + [float(n - 1 - v) for v in range(1, n)]
    assert st["frontier"] == n and st["touched"] == n - 1 and st["supersteps"] == 1
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
           "--master-addr", "127.0.0.1", "--master-port", str(29620 + nproc),
           os.path.join(ROOT, "tests", "mgpu_bc_sources_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    runs = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-bcs] runs=")]
    assert runs, p.stdout[-4000:]
    ok = [l for l in p.stdout.splitlines() if l.startswith("[mgpu-bcs] ") and l.endswith(" OK") and "refused" not in l]
    assert len(ok) == int(runs[-1].split("=")[1]) > 0
    assert "[mgpu-bcs] refused mirror_bytes OK" in p.stdout
