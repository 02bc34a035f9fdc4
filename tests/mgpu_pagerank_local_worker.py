"""Un-normalised PageRank on a fragment group: launched by torchrun (one rank per fragment;
GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).

Every case of tests/pagerank_local_cases.py and R-MAT 12 runs on undirected and directed fragments, on the
library's block partition (Fragment.from_edges) and on hash-partitioned fragments from
tests/partition_cases.py (`oid % fnum`, lids in order of first appearance, so out of oid order), created
through gl_frag_create.  Rank 0 scatters the results into vertex order and compares them with the oracle
and, where the reference completed the run on this many ranks, with its output (rtol 1e-9), checks that
a second query gave the same bits on every rank, and checks every rank's statistics: R + 1 supersteps,
R x (oe entries of its inner rows), and msg_bytes_sent = R x 8 M, M = the outer copies of its inner
vertices on the other fragments.  Rank 0 prints one OK / MISMATCH line per run and a closing "runs=" line."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RUNS = ((0.85, 10), (0.5, 2), (0.85, 1))
HASHED = ("mixed", "tier_rows", "long_rows", "random", "dense", "p2p31", "rmat12")


def outer_counts(n, s, d, owner, fnum):
    """M per fragment: the vertices it owns that another fragment holds as outer copies (an endpoint of an
    edge, either direction, whose other endpoint that fragment owns; directed fragments are built with
    their in-edges)."""
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
    from tests import pagerank_local_cases as C
    failures, runs = [], 0
    cases = C.pagerank_local_cases()
    s12, d12, _ = pkg.rmat_edges_host(12, 16, 7, 0)
    cases["rmat12"] = (1 << 12, s12.astype(np.int64), d12.astype(np.int64))
    _, refs = C.ref_pagerank_local_outputs()

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    todo = [(name, "blocks", dr) for name in sorted(cases) for dr in C.DIRS]
    todo += [(name, "hash", dr) for name in HASHED for dr in C.DIRS]
    for name, part, dr in todo:
        n, s, d = cases[name]
        directed = dr == "directed"
        if part == "blocks":
            frag = pkg.Fragment.from_edges(n, s, d, directed=directed, fid=rank, fnum=world)
            owner, _ = P.blocks(n, world)
            inner_of = [np.flatnonzero(owner == f) for f in range(world)]
        else:
            oids = np.arange(n, dtype=np.int64)
            owner, key = P.partition("hash", n, s, d, oids, world)
            L = P.describe(n, s, d, None, oids, directed, owner, key, world)
            frag = P.from_layout(pkg, L, rank, directed)
            inner_of = [f["inner"] for f in L.frags]
        comm = gdist.make_comm(rank, world, frag.ivnum)
        M = outer_counts(n, s, d, np.asarray(owner), world)
        r_of, _ = C.rows(n, s, d, directed)
        outd = np.bincount(r_of, minlength=n)
        for delta, R in RUNS:
            app = pkg.App("pagerank_local", frag, comm, pr_delta=delta, max_round=R)
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
                    oe = int(outd[inner].sum())
                    ok = ok and stats[:4] == (R + 1, R * oe, R * len(inner), R * 8 * int(M[f]))
                    ok = ok and stats[4] == [0] + [oe] * R
                want = C.pagerank_local(n, s, d, delta, R, directed)
                ok = ok and np.allclose(res, want, rtol=1e-9, atol=0)
                key = C.ref_key(name, dr, delta, R, world)
                if key in refs:
                    ok = ok and np.allclose(res, refs[key], rtol=1e-9, atol=0)
                print("[mgpu-prl] %-12s %-6s %-10s d=%-4g R=%-2d fnum=%d n=%d%s %s"
                      % (name, part, dr, delta, R, world, n, " ref" if key in refs else "",
                         "OK" if ok else "MISMATCH"), flush=True)
                runs += 1
                if not ok:
                    failures.append("%s:%s:%s:%g:%d" % (name, part, dr, delta, R))
        dist.barrier()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-prl] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
