"""k-clique counting on a fragment group: launched by torchrun (one rank per
fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  Every rank
checks that the count is the same on all ranks and equals the 1-fragment
count; rank 0 also compares it with the oracle (oracle/kclique_oracle.py) and
prints one OK / MISMATCH line per run."""
import importlib
import os
import sys

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
    from oracle import kclique_oracle as KO
    from tests import shapes as S
    from tests.kclique_cases import THRESHOLDS
    failures = []

    rm = [pkg.rmat_edges_host(sc, 16, 17, 0) for sc in (12, 14)]
    cases = {"rmat12": (1 << 12, rm[0][0], rm[0][1]), "rmat14": (1 << 14, rm[1][0], rm[1][1])}
    # tier limits, fragments owning no clique vertex, a fragment without inner vertices, multi-edges and
    # self loops, a shuffled union
    for name, (n, s, d, _) in {"block33": THRESHOLDS["block33"], "block1025": THRESHOLDS["block1025"],
                               "last_block": THRESHOLDS["last_block"], "empty": S.empty(1),
                               "multi_loop": S.multi_loop(),
                               "union": S.union([S.star(1500), S.clique(30), S.path(40), S.empty(5)], seed=9)}.items():
        cases[name] = (n, s, d)
    for name, (n, s, d) in cases.items():
        frag = pkg.Fragment.from_edges(n, s, d, None, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        one = pkg.Fragment.from_edges(n, s, d) if rank == 0 else None
        for k in (3, 4, 5):
            app = pkg.App("kclique", frag, comm, k=k)
            st = app.query()
            got = app.result()
            allv = [None] * world
            dist.all_gather_object(allv, got)
            if rank == 0:
                a1 = pkg.App("kclique", one, k=k)
                a1.query()
                want1 = a1.result()
                a1.close()
                want = KO.count(n, s, d, k)
                ok = all(x == got for x in allv) and got == want1 == want
                print("[mgpu-kclique] %-12s k=%d fnum=%d n=%d count=%d entries=%d %s"
                      % (name, k, world, n, got, st.entries_scanned, "OK" if ok else "MISMATCH"), flush=True)
                if not ok:
                    failures.append("%s:%d %r %d %d" % (name, k, allv, want1, want))
            app.close()
            dist.barrier()
        if one is not None:
            one.close()
        comm.close()
        frag.close()
    if failures:
        print("failures:", failures, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
