"""Core decomposition and k-core on a fragment group: launched by torchrun (one
rank per fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  Rank
0 compares the concatenated inner results with the whole-graph oracle
(oracle/core_oracle.py) and prints one OK / MISMATCH line per run."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    one_dev = os.environ.get("GL_ONE_DEVICE", "0") == "1"
    if one_dev:
        local = 0
    torch.cuda.set_device(local)
    if one_dev:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = "cpu" if one_dev else "cuda"
    pkg = importlib.import_module("libgrape-lite_b200")
    gdist = importlib.import_module("libgrape-lite_b200.dist")
    from oracle import core_oracle as CO
    from tests import shapes as S
    failures = []

    def gather(arr):
        out = [None] * world
        dist.all_gather_object(out, arr)
        return np.concatenate(out)

    rm = [pkg.rmat_edges_host(sc, 16, 17, 0) for sc in (12, 14)]
    cases = {"rmat12": (1 << 12, rm[0][0], rm[0][1]), "rmat14": (1 << 14, rm[1][0], rm[1][1])}
    # a star whose centre has outer copies on every peer, fragments without edges, a path followed by
    # isolated vertices, a block of long rows, a long multi-edge with self loops, a shuffled union
    for name, (n, s, d, _) in {"star": S.star(4097), "path_then_isolated": S.pad_to(S.path(300), 1000),
                               "empty": S.empty(33), "hub_block": S.hub_block(33), "multi_loop": S.multi_loop(),
                               "union": S.union([S.star(1500), S.clique(30), S.path(40), S.empty(5)], seed=9)}.items():
        cases[name] = (n, s, d)
    for name, (n, s, d) in cases.items():
        frag = pkg.Fragment.from_edges(n, s, d, None, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        core = CO.core_decomposition(n, s, d)[0] if rank == 0 else None
        mx = torch.tensor([int(core.max()) if rank == 0 else 0], dtype=torch.int64, device=dev)
        dist.broadcast(mx, 0)
        mx = int(mx.item())
        for kind, k in (("core_decomposition", None), ("kcore", 2), ("kcore", mx)):
            app = pkg.App(kind, frag, comm, **({} if k is None else {"k": k}))
            st = app.query()
            got = gather(app.result())
            if rank == 0:
                want = core if k is None else CO.kcore(n, s, d, k)
                ok = np.array_equal(got, want)
                print("[mgpu-core] %-18s %-18s k=%-5s fnum=%d n=%d sub-rounds=%d msg_bytes=%d %s"
                      % (name, kind, k, world, n, st.supersteps, st.msg_bytes_sent, "OK" if ok else "MISMATCH"),
                      flush=True)
                if not ok:
                    failures.append("%s:%s:%s" % (name, kind, k))
            app.close()
            dist.barrier()
        comm.close()
        frag.close()
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
