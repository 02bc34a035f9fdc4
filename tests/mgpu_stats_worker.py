"""Query statistics on a fragment group: launched by torchrun (one rank per fragment;
GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  Every rank evaluates the host
model (oracle/stats_model.py) for its own fragment on the whole graph's CSR and compares
what its app reports: push-only BFS (fused, stepwise, with the round-1 shipment and the
hub-first order switches set), PageRank push and pull, CDLP.  Per rank the per-step
arrays, the totals and supersteps equal the fragment's share; rank 0 adds the shares up
against the one-fragment model, checks the depths and prints one OK / MISMATCH line per
case and a closing "runs=" line."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BFS_CFGS = {"fused": dict(fuse_supersteps=1), "stepwise": dict(fuse_supersteps=0),
            "fused_r1ship": dict(fuse_supersteps=1, reserved={7: 1}), "fused_order3": dict(fuse_supersteps=1, reserved={1: 3})}


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
    from oracle import pyoracle
    from oracle import stats_model as M
    from tests import shapes as S
    failures, runs = [], 0

    def everyone(x):
        out = [None] * world
        dist.all_gather_object(out, x)
        return out

    def compare(st, want, touched, spare=0):
        """this rank's statistics against its share; returns a list of what differs.  spare = 1: one more
        superstep than the model's, with nothing in it, is allowed (a BFS on several fragments runs an
        empty closing round when the last level re-reported outer copies that were already visited,
        and the stepwise query when the source is in no fragment)."""
        n = st.n_steps
        extra = st.supersteps - want.supersteps
        bad = []
        if extra not in range(spare + 1) or n != min(st.supersteps, M.GL_MAX_STEP_STATS):
            bad.append("supersteps %d/%d n_steps %d/%d" % (st.supersteps, want.supersteps, n, want.n_steps))
        pad = [0] * max(n - want.n_steps, 0)
        for name, got, exp in (("step_frontier", list(st.step_frontier[:n]), want.step_frontier[:n] + pad),
                               ("step_entries", list(st.step_entries[:n]), want.step_entries[:n] + pad),
                               ("step_mode", list(st.step_mode[:n]), want.step_mode[:n] + pad)):
            if got != exp:
                i = next((k for k in range(min(len(got), len(exp))) if got[k] != exp[k]), -1)
                bad.append("%s[%d] %s/%s" % (name, i, got[i] if i >= 0 else len(got), exp[i] if i >= 0 else len(exp)))
        if st.entries_scanned != want.entries_scanned:
            bad.append("entries %d/%d" % (st.entries_scanned, want.entries_scanned))
        if st.frontier_vertices != want.frontier_vertices:
            bad.append("frontier %d/%d" % (st.frontier_vertices, want.frontier_vertices))
        if touched and st.touched_vertices != want.touched_vertices:
            bad.append("touched %d/%d" % (st.touched_vertices, want.touched_vertices))
        return bad

    def report(label, bad, extra_ok=True):
        nonlocal runs
        allbad = everyone(bad)
        if rank == 0:
            ok = extra_ok and not any(allbad)
            print("[mgpu-stats] %-44s fnum=%d %s %s" % (label, world, "OK" if ok else "MISMATCH",
                                                        "" if ok else "(device/model per rank: %s)" % allbad), flush=True)
            runs += 1
            if not ok:
                failures.append(label)

    rm = pkg.rmat_edges_host(12, 16, 7, 0)
    cases = {"rmat12": (1 << 12, rm[0], rm[1]), "star": S.star(4097)[:3], "path300": S.path(300)[:3],
             "path1000": S.path(1000)[:3]}
    for name, (n, s, d) in cases.items():
        frag = pkg.Fragment.from_edges(n, s, d, None, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        rp, col, _ = pyoracle.Graph(n, s, d, None).csr()
        deg = np.diff(rp.astype(np.int64))
        lo, hi = M.fragment_range(n, rank, world)
        assert frag.ivnum == hi - lo
        for source in dict.fromkeys([int(np.argmax(deg)), 0, n - 1, n + 5]):
            src = source if source < n else None
            one = M.bfs_push(rp, col, src)
            want = M.bfs_push(rp, col, src, rank, world)
            depths = np.full(n, np.iinfo(np.int64).max, dtype=np.int64)
            for k, l in enumerate(M.bfs_levels(rp, col, src)):
                depths[l] = k
            items = M.bfs_push_cut_items(rp, col, src, rank, world)
            for cname, cfg in BFS_CFGS.items():
                app = pkg.App("bfs", frag, comm, source_oid=source, direction_opt=0, **cfg)
                st = app.query()
                bad = compare(st, want, False, spare=1)
                if cname == "stepwise" and st.msg_bytes_sent != 4 * items:
                    bad.append("msg_bytes %d/%d" % (st.msg_bytes_sent, 4 * items))
                if cname != "stepwise" and st.msg_bytes_sent < 4 * items:
                    bad.append("msg_bytes %d < %d" % (st.msg_bytes_sent, 4 * items))
                got = np.concatenate(everyone(app.result()))
                fr = everyone(list(st.step_frontier[:st.n_steps]))
                en = everyone((int(st.entries_scanned), int(st.frontier_vertices), int(st.supersteps)))
                ok = True
                if rank == 0:
                    ok = (np.array_equal(got, depths) and len({e[2] for e in en}) == 1
                          and [sum(x) for x in zip(*fr)][:one.n_steps] == one.step_frontier[:one.n_steps]
                          and sum(e[0] for e in en) == one.entries_scanned
                          and sum(e[1] for e in en) == one.frontier_vertices)
                report("%s bfs %s source=%d" % (name, cname, source), bad, ok)
                app.close()
                dist.barrier()
        if name != "path1000":
            for rounds in (0, 1, 3):
                for label, kind, cfg, model in (("pagerank push", "pagerank", dict(pr_pull=0), M.pagerank),
                                                ("pagerank pull", "pagerank", dict(pr_pull=1), M.pagerank),
                                                ("cdlp", "cdlp", {}, M.cdlp)):
                    app = pkg.App(kind, frag, comm, max_round=rounds, **cfg)
                    st = app.query()
                    bad = compare(st, model(rp, rounds, rank, world), True)
                    en = everyone((int(st.entries_scanned), int(st.frontier_vertices), int(st.touched_vertices)))
                    one = model(rp, rounds)
                    ok = [sum(e[k] for e in en) for k in range(3)] == [one.entries_scanned, one.frontier_vertices,
                                                                       one.touched_vertices]
                    report("%s %s rounds=%d" % (name, label, rounds), bad, ok)
                    app.close()
                    dist.barrier()
        comm.close()
        frag.close()
    if rank == 0:
        print("[mgpu-stats] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
