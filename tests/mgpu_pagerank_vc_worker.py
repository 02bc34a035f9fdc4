"""PageRank on a grid of vertex-cut fragments: launched by torchrun with 4 or 9 ranks (one fragment
each; GL_ONE_DEVICE=1 puts every rank on cuda:0).

Every rank passes the whole edge list; rank 0 checks each rank's block layout against the host
partition (oracle/pagerank_vc_oracle.py), the values scattered into oid order against the oracle and
against the reference's output at the same fragment count (tests/golden/ref_pagerank_vc_outputs.*), that a
second query gave bit-identical values, and each rank's statistics, msg_bytes_sent included, against
the host model.  Every rank also checks that a communicator whose mirror slots are shorter than
8 * mvc bytes is refused.  Rank 0 prints one OK / MISMATCH line per run and a closing "runs=" line."""
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
    from oracle import pagerank_vc_oracle as V
    from tests import pagerank_vc_cases as P
    failures, runs = [], 0
    ref_meta, ref = P.ref_pagerank_vc_outputs()

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    cases = P.ref_cases()
    todo = [(name, R, 0.85) for name in sorted(cases) if name != "p2p31" for R in (0, 1, 10)]
    todo += [("rmat12", 10, 0.5), ("p2p31", 10, 0.85)]
    for name, R, delta in todo:
        n, s, d = cases[name]
        frag = pkg.VcFragment.from_edges(n, s, d, fid=rank, fnum=world)
        mvc = -(-n // world)
        comm = gdist.make_comm(rank, world, mvc)
        app = pkg.App("pagerank_vc", frag, comm, pr_delta=delta, max_round=R)
        st = app.query()
        got = app.result().copy()
        ids = app.result_oids()
        app.query()
        again = app.result()
        mine = (st.supersteps, st.entries_scanned, st.frontier_vertices, st.touched_vertices, st.msg_bytes_sent,
                list(st.step_entries[1:st.n_steps]), list(st.step_frontier[1:st.n_steps]))
        parts = gather((got, ids, again.tobytes() == got.tobytes(), mine, frag.info))
        if rank == 0:
            want = V.pagerank_vc(n, s, d, delta, R)
            model = V.stats(n, s, d, world, R)
            layout = V.partition(n, world)
            res = np.zeros(n)
            seen = np.zeros(n, dtype=bool)
            ok = all(p[2] for p in parts)
            for f, (vals, oid_list, _, stats, info) in enumerate(parts):
                res[oid_list] = vals
                seen[oid_list] = True
                m, L = model[f], layout[f]
                ok = ok and stats == (m["supersteps"], m["entries_scanned"], m["frontier_vertices"],
                                      m["touched_vertices"], m["msg_bytes_sent"], m["step_entries"],
                                      m["step_frontier"])
                ok = ok and (info["master_begin"], info["master_end"]) == L["master"]
                ok = ok and (info["src_begin"], info["src_end"]) == L["src"]
                ok = ok and (info["dst_begin"], info["dst_end"]) == L["dst"]
                ok = ok and info["local_vnum"] == L["local_vnum"] and info["block_edges"] == m["block_edges"]
            ok = ok and bool(seen.all()) and np.allclose(res, want, rtol=1e-9, atol=0)
            key = P.ref_key(name, R, delta, world)
            if key in ref:   # absent: the reference's loader aborted on this run
                idx = P.sample_index(n) if name in P.LARGE else np.arange(n)
                ok = ok and np.allclose(res[idx], ref[key], rtol=1e-9, atol=0)
                ok = ok and np.isclose(res.sum(), ref_meta["sums"][key], rtol=1e-9)
            else:
                ok = ok and key in ref_meta["aborted"]
            print("[mgpu-prvc] %-12s R=%-2d d=%.2f fnum=%d n=%d %s" % (name, R, delta, world, n,
                                                                      "OK" if ok else "MISMATCH"), flush=True)
            runs += 1
            if not ok:
                failures.append(name)
        app.close()
        dist.barrier()
        comm.close()
        frag.close()

    # a mirror slot shorter than 8 * mvc bytes is refused (gl_comm_create rounds the size up to a
    # multiple of 256 bytes, so ask for the largest such multiple below 8 * mvc)
    n, s, d = cases["star_9000"]
    mvc = -(-n // world)
    frag = pkg.VcFragment.from_edges(n, s, d, fid=rank, fnum=world)
    small = pkg.Comm(rank, world, lambda a, op: None, landing_bytes=1 << 12,
                     mirror_bytes=((8 * mvc - 1) // 256) * 256)
    handles = [None] * world
    dist.all_gather_object(handles, small.export())
    small.open(handles)
    try:
        pkg.App("pagerank_vc", frag, small)
        refused = False
    except pkg.GrapeError:
        refused = True
    flags = gather(refused)
    if rank == 0:
        print("[mgpu-prvc] small-mirror refused fnum=%d %s" % (world, "OK" if all(flags) else "MISMATCH"), flush=True)
        runs += 1
        if not all(flags):
            failures.append("small-mirror")
    dist.barrier()
    small.close()
    frag.close()

    if rank == 0:
        print("[mgpu-prvc] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
