"""Directed local clustering coefficient on a fragment group: launched by torchrun (one rank per
fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).

Every case of tests/lcc_directed_cases.py runs on the library's block partition
(Fragment.from_edges(..., directed=True)); R-MAT 12, the multigraphs, the clique and the 300-entry pair
also run on hash-partitioned fragments from tests/partition_cases.py (`oid % fnum`, lids in order of
first appearance, so out of oid order), created through gl_frag_create with their in-edges.  Rank 0
scatters the results into vertex order through result_oids and compares them bit for bit with the exact
oracle (oracle/lcc_directed_oracle.py), and checks every rank's statistics against its share of
oracle/lcc_directed_oracle.py stats (degree ties broken by gid rank), and that the shares add up to the
one-fragment value.  Rank 0 prints one OK / MISMATCH line per run and a closing "runs=" line."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HASHED = ("rmat12", "multigraph1", "multigraph2", "clique40", "pair300", "in_star4097")


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
    from oracle import lcc_directed_oracle as LO
    from tests import partition_cases as P
    from tests.lcc_directed_cases import as_indices, lcc_directed_cases
    failures, runs = [], 0

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    runs_todo = [(name, "blocks") for name in sorted(lcc_directed_cases())] + [(name, "hash") for name in HASHED]
    cases = lcc_directed_cases()
    for name, part in runs_todo:
        n, src, dst, oids = cases[name]
        s, d = as_indices(n, src, dst, oids)
        vid = np.arange(n, dtype=np.int64) if oids is None else np.sort(np.asarray(oids, dtype=np.int64))
        if part == "blocks":
            frag = pkg.Fragment.from_edges(n, src, dst, directed=True, oids=oids, fid=rank, fnum=world)
            owner, _ = P.blocks(n, world)
            grank = np.arange(n, dtype=np.int64)
        else:
            owner, key = P.partition("hash", n, s, d, vid, world)
            L = P.describe(n, s, d, None, vid, True, owner, key, world)
            frag = P.from_layout(pkg, L, rank, True)
            grank = L.rank
        comm = gdist.make_comm(rank, world, frag.ivnum)
        app = pkg.App("lcc_directed", frag, comm)
        st = app.query()
        got = app.result()
        ids = app.result_oids()
        app.query()
        again = app.result()
        mine = (st.supersteps, st.entries_scanned, st.frontier_vertices, st.touched_vertices,
                list(st.step_entries[:st.n_steps]), list(st.step_frontier[:st.n_steps]),
                list(st.step_mode[:st.n_steps]))
        parts = gather((got, ids, again.tobytes() == got.tobytes(), mine))
        if rank == 0:
            lcc, _, _ = LO.lcc_directed(n, s, d)
            res = np.zeros(n, dtype=np.float64)
            seen = np.zeros(n, dtype=bool)
            ok = all(p[2] for p in parts)
            for f, (vals, oid_list, _, stats) in enumerate(parts):
                idx = np.searchsorted(vid, oid_list)
                res[idx] = vals
                seen[idx] = True
                want = LO.stats(n, s, d, rank=grank, owned=owner == f)
                ok = ok and stats == (want.supersteps, want.entries_scanned, want.frontier_vertices,
                                      want.touched_vertices, want.step_entries[:len(stats[4])],
                                      want.step_frontier[:len(stats[5])], want.step_mode[:len(stats[6])])
            whole = LO.stats(n, s, d, rank=grank)
            ok = ok and sum(p[3][1] for p in parts) == whole.entries_scanned
            ok = ok and bool(seen.all()) and res.tobytes() == lcc.tobytes()
            print("[mgpu-lccd] %-14s %-6s fnum=%d n=%d %s" % (name, part, world, n, "OK" if ok else "MISMATCH"),
                  flush=True)
            runs += 1
            if not ok:
                failures.append("%s:%s" % (name, part))
        app.close()
        dist.barrier()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-lccd] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
