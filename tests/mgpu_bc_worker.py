"""Betweenness centrality on a fragment group: launched by torchrun (one rank
per fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  For every
graph the source is taken on each fragment in turn (its largest row), plus one
source that is not in the graph.  Rank 0 compares the concatenated inner
results with a one-fragment run of the same graph: depth and sigma exactly, c
within (L + 1) * 2^-22 relative; it prints one OK / MISMATCH line per run and a
closing "runs=" line."""
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
    from tests import shapes as S
    from tests.bc_cases import degrees
    failures, runs = [], 0

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
        iv = [None] * world
        dist.all_gather_object(iv, int(frag.ivnum))
        off = np.concatenate([[0], np.cumsum(iv)])
        deg = degrees(n, s, d)
        sources = [int(off[f] + np.argmax(deg[off[f]:off[f + 1]])) for f in range(world) if iv[f]] + [n + 5]
        whole = pkg.Fragment.from_edges(n, s, d) if rank == 0 else None
        for source in sources:
            app = pkg.App("bc", frag, comm, source_oid=source)
            st = app.query()
            got = gather(app.result())
            if rank == 0:
                one = pkg.App("bc", whole, source_oid=source)
                one.query()
                want = one.result()
                one.close()
                reached = want["depth"] != np.iinfo(np.int64).max
                L = int(want["depth"][reached].max()) if reached.any() else 0
                ok = (np.array_equal(got["depth"], want["depth"]) and np.array_equal(got["path_num"], want["path_num"])
                      and bool(np.all(np.abs(got["centrality"] - want["centrality"])
                                      <= (L + 1) * 2.0 ** -22 * np.abs(want["centrality"]))))
                print("[mgpu-bc] %-18s source=%-6d fnum=%d n=%d levels=%d rounds=%d %s"
                      % (name, source, world, n, L + 1 if reached.any() else 0, st.supersteps,
                         "OK" if ok else "MISMATCH"), flush=True)
                runs += 1
                if not ok:
                    failures.append("%s:%d" % (name, source))
            app.close()
            dist.barrier()
        if whole is not None:
            whole.close()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-bc] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
