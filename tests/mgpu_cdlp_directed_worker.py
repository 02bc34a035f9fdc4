"""Directed CDLP on a fragment group: launched by torchrun (one rank per fragment; GL_ONE_DEVICE=1 puts
every rank's fragment on cuda:0).

Every case of tests/cdlp_directed_cases.py runs after 10 rounds on the library's block partition
(Fragment.from_edges(..., directed=True)), without a vertex map (labels come back as global indices,
which are the oids there) and, for p2p-31 (explicit oids: it needs one) and a few others, with one.
The cycle also runs after 1 and 2 rounds: every fragment's only in-edge from outside comes from the
previous fragment, so from round 2 on its label travels to an outer copy seen only through an in-edge.
The multigraphs, the in-only vertex, the threshold rows and R-MAT 12 also run on hash-partitioned
fragments from tests/partition_cases.py (`oid % fnum`, lids in order of first appearance, so out of oid
order), created through gl_frag_create with their in-edges, with a vertex map (labels as oids) and
without one (labels as raw gids).  Rank 0 scatters the results into vertex order through result_oids
and compares them with the oracle (ties on the smallest gid), and checks every rank's statistics
against its share (stats_model.cdlp over the combined row pointer ie_rp + oe_rp of its inner rows) and
that the shares add up to the one-fragment value.  Rank 0 prints one OK / MISMATCH line per run and a
closing "runs=" line."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WITH_VM = ("p2p31", "cycle", "multigraph1", "threshold")
HASHED = ("multigraph1", "multigraph2", "only_in", "threshold", "rmat12")


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
    from oracle import stats_model as M
    from tests import partition_cases as P
    from tests.cdlp_directed_cases import as_indices, cdlp_directed_cases, oracle
    failures, runs = [], 0
    cases = cdlp_directed_cases()

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    todo = []
    for name in sorted(cases):
        if cases[name][3] is None:
            todo.append((name, "blocks", False, 10))
        if name in WITH_VM:
            todo.append((name, "blocks", True, 10))
    todo += [("cycle", "blocks", False, 1), ("cycle", "blocks", False, 2)]
    todo += [(name, "hash", vm, 10) for name in HASHED for vm in (True, False)]
    for name, part, with_vm, rounds in todo:
        n, src, dst, oids = cases[name]
        s, d = as_indices(n, src, dst, oids)
        vid = np.arange(n, dtype=np.int64) if oids is None else np.sort(np.asarray(oids, dtype=np.int64))
        if part == "blocks":
            frag = pkg.Fragment.from_edges(n, src, dst, directed=True, oids=oids, fid=rank, fnum=world)
            owner, _ = P.blocks(n, world)
            grank = np.arange(n, dtype=np.int64)
            gid = None
            chunk = -(-n // world)
            vm_lists = [vid[f * chunk:(f + 1) * chunk] for f in range(world)]
        else:
            owner, key = P.partition("hash", n, s, d, vid, world)
            L = P.describe(n, s, d, None, vid, True, owner, key, world)
            frag = P.from_layout(pkg, L, rank, True)
            grank = L.rank
            gid = L.gid
            vm_lists = [f["inner_oids"] for f in L.frags]
        comm = gdist.make_comm(rank, world, frag.ivnum)
        vm = pkg.VertexMap(vm_lists) if with_vm else None
        app = pkg.App("cdlp_directed", frag, comm, max_round=rounds)
        if vm is not None:
            app.set_vertex_map(vm)
        st = app.query()
        got = app.result()
        app.query()
        again = app.result()
        # result_oids needs the vertex map on hash partitions; the lids give the vertices otherwise
        mine = (st.supersteps, st.entries_scanned, st.frontier_vertices, st.touched_vertices,
                list(st.step_entries[:st.n_steps]), list(st.step_frontier[:st.n_steps]),
                list(st.step_mode[:st.n_steps]))
        parts = gather((got, again.tobytes() == got.tobytes(), mine))
        if rank == 0:
            lab = oracle(n, s, d, rounds, rank=grank)
            want = vid[lab] if (with_vm or part == "blocks") else gid[lab]
            res = np.full(n, -1, dtype=np.int64)
            ok = all(p[1] for p in parts)
            deg = np.bincount(s, minlength=n) + np.bincount(d, minlength=n)
            total = 0
            for f, (vals, _, stats) in enumerate(parts):
                inner = np.flatnonzero(owner == f) if part == "blocks" else L.frags[f]["inner"]
                ok = ok and len(vals) == len(inner)
                res[inner] = vals
                rp = np.concatenate([[0], np.cumsum(deg[inner])])
                w = M.cdlp(rp, rounds)
                if part == "blocks":
                    b = M.cdlp(np.concatenate([[0], np.cumsum(deg)]), rounds, f, world)
                    ok = ok and (b.step_entries, b.touched_vertices) == (w.step_entries, w.touched_vertices)
                ok = ok and stats == (w.supersteps, w.entries_scanned, w.frontier_vertices, w.touched_vertices,
                                      w.step_entries[:len(stats[4])], w.step_frontier[:len(stats[5])],
                                      w.step_mode[:len(stats[6])])
                total += stats[1]
            ok = ok and total == rounds * 2 * len(s)
            ok = ok and np.array_equal(res, want)
            print("[mgpu-cdlpd] %-16s %-6s %-5s R=%-2d fnum=%d n=%d %s"
                  % (name, part, "vm" if with_vm else "no-vm", rounds, world, n, "OK" if ok else "MISMATCH"),
                  flush=True)
            runs += 1
            if not ok:
                failures.append("%s:%s:%s:%d" % (name, part, with_vm, rounds))
        app.close()
        if vm is not None:
            vm.close()
        dist.barrier()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-cdlpd] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
