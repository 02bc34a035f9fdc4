"""Directed graphs split into 2 and 3 fragments on one device (one torchrun rank
per fragment, tests/mgpu_directed_worker.py): BFS, SSSP, WCC and PageRank in
every configuration of tests/directed_cases.py against the whole-graph oracle,
p2p-31 against the reference's directed golden files, and the path-taken checks
(fragment geometry, pull levels) gathered to rank 0."""
import os
import re
import subprocess
import sys

import pytest

from tests import directed_cases as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nproc", [2, 3])
def test_directed_fragment_group_one_device(nproc):
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29640 + nproc),
           os.path.join(ROOT, "tests", "mgpu_directed_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    lines = p.stdout.splitlines()
    bad = [l for l in lines if l.startswith("[mgpu-dir]") and not l.endswith(" OK")]    # mismatches, timings
    sys.stdout.write("\n".join(bad + lines[-40:]) + "\n")
    assert p.returncode == 0, "\n".join(bad + lines[-60:])
    ok = sum(1 for l in lines if re.match(r"\[mgpu-dir\] .* OK$", l))
    assert ok == D.ok_lines_expected(), (ok, D.ok_lines_expected())
