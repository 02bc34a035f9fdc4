"""k-clique counting on the GPU (csrc/app_kclique.cu): equal to the reference
app's counts (tests/golden/ref_kclique_outputs.json) and to the CPU oracle
(oracle/kclique_oracle.py) on every case of tests/kclique_cases.py; the tier
item counts equal the host's reading of the kernel's rule; refusals; fragment
groups through mgpu_kclique_worker.py."""
import os
import subprocess
import sys
from math import comb

import numpy as np
import pytest

from oracle import kclique_oracle as KO
from tests import shapes as S
from tests.kclique_cases import (MAX_K, THRESHOLDS, as_indices, candidate_sizes, kclique_cases,
                                 ref_kclique_outputs, tier_items)
from tests.util import pkg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = kclique_cases()
REF = ref_kclique_outputs()


def run(frag, k):
    app = pkg().App("kclique", frag, k=k)
    st = app.query()
    got = app.result()
    tiers = (st.step_frontier[0], st.step_frontier[1], st.step_frontier[2], st.step_frontier[3])
    app.close()
    return got, tiers, st


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_counts(name):
    n, src, dst, oids = CASES[name]
    si, di = as_indices(n, src, dst, oids)
    frag = pkg().Fragment.from_edges(n, src, dst, None, oids=oids)
    for k, want in REF[name].items():
        got, _, _ = run(frag, k)
        assert got == want, k
        if n <= 5000:
            assert got == KO.count(n, si, di, k), k
    frag.close()


@pytest.mark.parametrize("seed", range(8))
def test_multigraph_counts_its_simplification(seed):
    from tests.core_cases import random_multigraph
    n, s, d = random_multigraph(seed)
    a, b = KO.simple_edges(n, s, d)
    f1 = pkg().Fragment.from_edges(n, s, d)
    f2 = pkg().Fragment.from_edges(n, a, b)
    for k in (3, 4, 5):
        assert run(f1, k)[0] == run(f2, k)[0] == KO.count(n, s, d, k), k
    f1.close()
    f2.close()


@pytest.mark.parametrize("name", sorted(THRESHOLDS))
def test_tiers(name):
    n, s, d, _ = THRESHOLDS[name]
    sizes = candidate_sizes(n, s, d)
    frag = pkg().Fragment.from_edges(n, s, d)
    for k in (4, 5):
        got, tiers, _ = run(frag, k)
        assert tuple(int(x) for x in tiers) == tier_items(sizes, k), k
        assert got == KO.count(n, s, d, k), k
    frag.close()


def test_every_tier_runs():
    seen = [0, 0, 0]
    for name in ("block32", "block33", "block1025"):
        n, s, d, _ = THRESHOLDS[name]
        frag = pkg().Fragment.from_edges(n, s, d)
        _, tiers, _ = run(frag, 4)
        for i in range(3):
            seen[i] += int(tiers[1 + i])
        frag.close()
    assert all(seen), seen
    # the host reading of the rule puts the block edges at and above each limit
    assert tier_items(candidate_sizes(*THRESHOLDS["block1025"][:3]), 4)[0] == 1025
    assert tier_items(candidate_sizes(*THRESHOLDS["block1024"][:3]), 4)[0] == 1024


def test_apps_with_different_k_side_by_side():
    # the shared-memory opt-in is a property of the kernels: an app made later with a smaller k must not
    # take it away from one with a larger k (the k = 6 and k = 30 apps need more than the k = 4 one)
    n, s, d, _ = THRESHOLDS["clique35"]
    frag = pkg().Fragment.from_edges(n, s, d)
    apps = {k: pkg().App("kclique", frag, k=k) for k in (6, 30, 4)}
    for _ in range(2):
        for k, app in apps.items():
            st = app.query()
            assert app.result() == comb(n, k), k
            assert st.step_frontier[2] == 1, k   # the edge (0, 1) with s = 33 ran in the CTA bitmap tier
    with pytest.raises(pkg().GrapeError):
        apps[4].result(out=np.zeros(1, dtype=np.int64))
    for app in apps.values():
        app.close()
    frag.close()


def test_second_query_same_count():
    n, s, d, _ = CASES["rmat12"]
    frag = pkg().Fragment.from_edges(n, s, d)
    app = pkg().App("kclique", frag, k=4)
    app.query()
    a = app.result()
    st = app.query()
    assert app.result() == a == REF["rmat12"][4]
    assert st.supersteps == 1 and st.entries_scanned > 0 and st.frontier_vertices > 0
    app.close()
    frag.close()


def test_refusals():
    n, s, d, _ = S.path(10)
    frag = pkg().Fragment.from_edges(n, s, d, directed=True)
    with pytest.raises(pkg().GrapeError):
        pkg().App("kclique", frag, k=3)
    frag.close()
    frag = pkg().Fragment.from_edges(n, s, d)
    for k in (-1, 0, 1, 2, MAX_K + 1):
        with pytest.raises(pkg().GrapeError):
            pkg().App("kclique", frag, k=k)
    with pytest.raises(pkg().GrapeError):
        pkg().App("kclique", frag)
    got, _, _ = run(frag, MAX_K)
    assert got == 0
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
           "--master-addr", "127.0.0.1", "--master-port", str(29600 + nproc + (0 if one_device else 5)),
           os.path.join(ROOT, "tests", "mgpu_kclique_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert " MISMATCH" not in p.stdout
    assert p.stdout.count(" OK") == 8 * 3, p.stdout[-4000:]   # 8 graphs x k = 3, 4, 5
