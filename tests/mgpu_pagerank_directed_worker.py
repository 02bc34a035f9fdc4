"""Directed PageRank on a fragment group: launched by torchrun (one rank per fragment; GL_ONE_DEVICE=1 puts
every rank's fragment on cuda:0).

Every case of tests/pagerank_directed_cases.py and R-MAT 12 runs on the library's block partition
(Fragment.from_edges(..., directed=True)) and on hash-partitioned fragments from tests/partition_cases.py
(`oid % fnum`, lids in order of first appearance, so out of oid order), created through gl_frag_create
with their in-edges.  Rank 0 scatters the results into vertex order and compares them with the oracle and,
where a fixture run exists, with the reference's output (rtol 1e-9), checks that they sum to 1 and that a
second query gave the same bits on every rank, and checks every rank's statistics: R + 1 supersteps,
R x (ie entries of its inner rows), and msg_bytes_sent = R x 8 M + (R - 1) x 8 (F - 1), M = the outer
copies of its inner vertices on the other fragments.  Rank 0 prints one OK / MISMATCH line per run and a
closing "runs=" line."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RUNS = ((0.85, 10), (0.5, 2), (0.85, 1), (0.85, 0))
HASHED = ("mixed", "tier_rows", "long_rows", "random", "p2p31", "rmat12")


def outer_counts(n, s, d, owner, fnum):
    """M per fragment: the vertices it owns that another fragment holds as outer copies (an endpoint of an
    edge, either direction, whose other endpoint that fragment owns)."""
    M = np.zeros(fnum, dtype=np.int64)
    for g in range(fnum):
        mine_s, mine_d = owner[s] == g, owner[d] == g
        adj = np.unique(np.concatenate([d[mine_s], s[mine_d]]))
        adj = adj[owner[adj] != g]
        M += np.bincount(owner[adj], minlength=fnum)
    return M


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
    from tests import partition_cases as P
    from tests import pagerank_directed_cases as C
    failures, runs = [], 0
    cases = C.pagerank_directed_cases()
    s12, d12, _ = pkg.rmat_edges_host(12, 16, 7, 0)
    cases["rmat12"] = (1 << 12, s12.astype(np.int64), d12.astype(np.int64))
    _, refs = C.ref_pagerank_directed_outputs()

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    todo = [(name, "blocks") for name in sorted(cases)] + [(name, "hash") for name in HASHED]
    for name, part in todo:
        n, s, d = cases[name]
        if part == "blocks":
            frag = pkg.Fragment.from_edges(n, s, d, directed=True, fid=rank, fnum=world)
            owner, _ = P.blocks(n, world)
            inner_of = [np.flatnonzero(owner == f) for f in range(world)]
        else:
            oids = np.arange(n, dtype=np.int64)
            owner, key = P.partition("hash", n, s, d, oids, world)
            L = P.describe(n, s, d, None, oids, True, owner, key, world)
            frag = P.from_layout(pkg, L, rank, True)
            inner_of = [f["inner"] for f in L.frags]
        comm = gdist.make_comm(rank, world, frag.ivnum)
        M = outer_counts(n, s, d, np.asarray(owner), world)
        ind = np.bincount(d, minlength=n)
        for delta, R in RUNS:
            app = pkg.App("pagerank_directed", frag, comm, pr_delta=delta, max_round=R)
            st = app.query()
            got = app.result()
            app.query()
            again = app.result()
            app.close()
            mine = (st.supersteps, st.entries_scanned, st.touched_vertices, st.msg_bytes_sent,
                    list(st.step_entries[:st.n_steps]))
            parts = gather((got, again.tobytes() == got.tobytes(), mine))
            if rank == 0:
                res = np.full(n, np.nan)
                ok = all(p[1] for p in parts)
                for f, (vals, _, stats) in enumerate(parts):
                    inner = inner_of[f]
                    ok = ok and len(vals) == len(inner)
                    res[inner] = vals
                    ie = int(ind[inner].sum())
                    if R <= 0:
                        want_st = (1, 0, 0, 0)
                    else:
                        want_st = (R + 1, R * ie, R * len(inner), R * 8 * int(M[f]) + (R - 1) * 8 * (world - 1))
                    ok = ok and stats[:4] == want_st
                    if R > 0:
                        ok = ok and stats[4] == [0] + [ie] * R
                want = C.pagerank_directed(n, s, d, delta, R)
                if R <= 0:
                    ok = ok and not res.any()
                else:
                    ok = ok and np.allclose(res, want, rtol=1e-9, atol=0) and abs(res.sum() - 1.0) <= 1e-12
                    key = C.ref_key(name, delta, R)
                    if key in refs:
                        ok = ok and np.allclose(res, refs[key], rtol=1e-9, atol=0)
                print("[mgpu-prd] %-12s %-6s d=%-4g R=%-2d fnum=%d n=%d %s"
                      % (name, part, delta, R, world, n, "OK" if ok else "MISMATCH"), flush=True)
                runs += 1
                if not ok:
                    failures.append("%s:%s:%g:%d" % (name, part, delta, R))
        dist.barrier()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-prd] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
