"""Edge-cut multi-fragment parity through the peer-memory message manager
(csrc/comm.cu): one process per fragment, launched with torchrun.

* test_multi_fragment_one_device: every rank's fragment lives on cuda:0 (the
  rank processes' contexts time-slice the GPU, CUDA IPC maps the landing areas
  across them).  Runs on a 1-GPU box and exercises the whole data plane --
  msg_send / pack_outer_phase / k_unpack, the device-side round barrier and
  vote, the dense mirror sync, the fused multi-fragment BFS kernel with its
  in-kernel collectives -- for all six apps at 2 and 3 fragments.
* test_multi_fragment_parity: one fragment per GPU over NVLink (>= 2 devices)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nproc", [2, 4])
def test_multi_fragment_parity(nproc):
    if _ngpus() < nproc:
        pytest.skip("needs %d GPUs" % nproc)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + nproc),
           os.path.join(ROOT, "tests", "mgpu_worker.py"), "13"]
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]


@pytest.mark.parametrize("nproc,scale,apps,min_ok", [(2, 12, None, 22), (3, 11, None, 22),
                                                    # 2^17 vertices: the default configuration takes the hub-first
                                                    # order + delegated hubs of the several-fragment fused BFS
                                                    (2, 17, "bfs,bfs_hub_src2,bfs_spill,bfs_nohub,bfs_r1ship,bfs_step", 6)])
def test_multi_fragment_one_device(nproc, scale, apps, min_ok):
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1")
    if apps:
        env["GL_APPS"] = apps
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29520 + nproc + (7 if apps else 0)),
           os.path.join(ROOT, "tests", "mgpu_worker.py"), str(scale)]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert p.stdout.count(" OK") >= min_ok, p.stdout[-4000:]


@pytest.mark.parametrize("nproc", [2, 3])
def test_multi_fragment_shapes_one_device(nproc):
    """The threshold graphs of tests/shapes.py (star, path, empty, hub block, multi-edge) split into
    fragments on one device: fragments without edges or outer vertices, owner boundaries inside a
    bitmap word, a hub with outer copies on every peer -- all six apps (mgpu_worker.py GL_SHAPES=1)."""
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1", GL_SHAPES="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29540 + nproc),
           os.path.join(ROOT, "tests", "mgpu_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-4000:]
    assert p.stdout.count(" OK") == 60, p.stdout[-4000:]     # 6 shapes x 10 app configurations


@pytest.mark.parametrize("nproc", [2, 3])
def test_message_manager_face2_one_device(nproc):
    """The message manager of the C ABI on 2 and 3 fragments of one device, item by item
    (mgpu_worker.py GL_FACE2=1): send_outer + process for every value size, clear_bits and
    consumer kind, the round protocol and its termination vote, round 0 of a second query,
    the dense mirror sync of values and bits, gl_allreduce and a landing-slot overflow -- on
    a star whose centre has copies on every peer, a path with owner boundaries inside a
    bitmap word (alone and padded with isolated vertices), fragments without outer vertices
    and R-MAT 12."""
    if _ngpus() < 1:
        pytest.skip("needs a GPU")
    env = dict(os.environ, GL_ONE_DEVICE="1", GL_FACE2="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(29580 + nproc),
           os.path.join(ROOT, "tests", "mgpu_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    sys.stdout.write(p.stdout[-6000:])
    assert p.returncode == 0, p.stdout[-6000:]
    assert p.stdout.count(" OK") == 5, p.stdout[-6000:]      # 5 graphs
