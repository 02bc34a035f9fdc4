"""Every buffer an app allocates is released when the app is destroyed, and when its creation is
refused: after one warm-up cycle (which pays for the process-wide lazy state: device info, launch
geometry, host pools), further create -> query -> result -> destroy cycles leave the free device
memory exactly where the warm-up left it.

R-MAT scale 17 puts BFS and PageRank on their hub-first paths (shadow graph, permuted columns);
the 2-fragment group on one device covers the message manager, the mirror plan, LCC's peer
replicas and the delegated hubs of the several-fragment BFS (mgpu_worker.py GL_RESOURCES=1)."""
import os
import subprocess
import sys

import pytest

from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

APPS = [
    ("bfs", dict(fuse_supersteps=1)),
    ("bfs", dict(fuse_supersteps=0)),
    ("sssp", dict(sssp_f64=0)),
    ("sssp", dict(sssp_f64=1)),
    ("wcc", {}),
    ("wcc_opt", {}),
    ("pagerank", dict(pr_pull=0)),
    ("pagerank", dict(pr_pull=1)),
    ("cdlp", dict(max_round=5)),
    ("lcc", {}),
]


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def assert_cycles_release(cycle, reps=3):
    cycle()
    base = free_bytes()
    for _ in range(reps):
        cycle()
    assert free_bytes() == base


@pytest.fixture(scope="module")
def rmat17():
    frag = pkg().Fragment.rmat(17, 16, seed=7, weight_mode=1)
    yield frag
    frag.close()


@pytest.mark.parametrize("kind,cfg", APPS, ids=["%s-%s" % (k, "-".join("%s%s" % kv for kv in c.items())) for k, c in APPS])
def test_app_destroy_releases_buffers(rmat17, kind, cfg):
    cfg = dict(cfg)
    if kind in ("bfs", "sssp"):
        cfg["source_oid"] = rmat17.max_degree_vertex()[0]

    def cycle():
        app = pkg().App(kind, rmat17, **cfg)
        app.query()
        app.result()
        app.close()

    assert_cycles_release(cycle)


def test_refused_creation_releases_buffers():
    n, src, dst, w = rmat_graph(12, seed=2, weight_mode=1)
    w = w.copy()
    w[3] = -1.0
    weighted = pkg().Fragment.from_edges(n, src, dst, w)
    built = pkg().Fragment.from_edges(n, src, dst, directed=True)
    rp, col, _ = built.csr(0)
    built.close()
    out_only = pkg().Fragment.from_csr(n, rp, col, directed=True)    # directed, no ie CSR

    def cycle():
        for f64 in (0, 1):
            with pytest.raises(pkg().GrapeError):
                pkg().App("sssp", weighted, source_oid=0, sssp_f64=f64)
        for kind in ("wcc", "wcc_opt"):
            with pytest.raises(pkg().GrapeError):
                pkg().App(kind, out_only)

    assert_cycles_release(cycle)
    weighted.close()
    out_only.close()


def test_multi_fragment_destroy_releases_buffers():
    import torch
    if torch.cuda.device_count() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1", GL_RESOURCES="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29561",
           os.path.join(ROOT, "tests", "mgpu_worker.py"), "17"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert p.stdout.count(" RELEASED") == 10, p.stdout[-4000:]
