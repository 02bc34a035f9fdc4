"""Betweenness centrality on a fragment group: launched by torchrun (one rank
per fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  For every
graph the source is taken on each fragment in turn (its largest row), plus a
smallest-positive-degree vertex, the vertex a constructed graph is built
around, and one source that is not in the graph.  Every rank sends its own CSR,
mapped to global vertex indices, to rank 0, which compares the concatenated
inner results bit for bit -- depth, sigma and c -- with the order-exact oracle
(oracle/bc_oracle.py bc_rows, short=None: k_bc_pull_multi and k_bc_back_multi
sum every row sequentially in the fragment's row order).  Rank 0 prints one
OK / MISMATCH line per run and a closing "runs=" line."""
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
    from oracle import bc_oracle as BO
    from tests import bc_shapes as B
    from tests import shapes as S
    from tests.bc_cases import degrees
    failures, runs = [], 0

    def gather(arr):
        out = [None] * world
        dist.all_gather_object(out, arr)
        return np.concatenate(out)

    rm = [pkg.rmat_edges_host(sc, 16, 17, 0) for sc in (12, 14)]
    cases = {"rmat12": (1 << 12, rm[0][0], rm[0][1]), "rmat14": (1 << 14, rm[1][0], rm[1][1])}
    roots = {}
    # a star whose centre has outer copies on every peer, fragments without edges, a path followed by
    # isolated vertices, a block of long rows, a long multi-edge with self loops, a shuffled union
    for name, (n, s, d, _) in {"star": S.star(4097), "path_then_isolated": S.pad_to(S.path(300), 1000),
                               "empty": S.empty(33), "hub_block": S.hub_block(33), "multi_loop": S.multi_loop(),
                               "union": S.union([S.star(1500), S.clique(30), S.path(40), S.empty(5)], seed=9)}.items():
        cases[name] = (n, s, d)
    # sums that round (sigma past 2^53 in long rows; a backward row of t values far apart), a fan of rows on
    # the chunk cuts, and backward rows of 2049 entries
    for name in ("order_chain", "back_chain", "fans", "kab33_2048"):
        build, roots[name] = B.BC_SHAPES[name]
        n, s, d, _ = build()
        cases[name] = (n, s, d)
    for name, (n, s, d) in cases.items():
        frag = pkg.Fragment.from_edges(n, s, d, None, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        iv = [None] * world
        dist.all_gather_object(iv, int(frag.ivnum))
        off = np.concatenate([[0], np.cumsum(iv)])
        deg = degrees(n, s, d)
        sources = [int(off[f] + np.argmax(deg[off[f]:off[f + 1]])) for f in range(world) if iv[f]]
        if np.any(deg > 0):
            pos = np.flatnonzero(deg > 0)
            sources.append(int(pos[np.argmin(deg[pos])]))
        if name in roots:
            sources.append(roots[name])
        sources = list(dict.fromkeys(sources + [n + 5]))
        # this fragment's rows in global indices: inner lid + the ivnum prefix, outer lid through its gid
        rp, col, _ = frag.csr(0)
        col = col.astype(np.int64)
        ovg = frag.ovgid().astype(np.int64)
        outer = col >= frag.ivnum
        g = ovg[col[outer] - frag.ivnum]
        col[outer] = off[g >> frag.fid_offset] + (g & ((1 << frag.fid_offset) - 1))
        col[~outer] += off[rank]
        parts = [None] * world
        dist.all_gather_object(parts, (np.diff(rp.astype(np.int64)), col))
        if rank == 0:
            grp = np.concatenate([[0], np.cumsum(np.concatenate([p[0] for p in parts]))]).astype(np.int64)
            gcol = np.concatenate([p[1] for p in parts])
            assert len(grp) == n + 1 and len(gcol) == grp[-1]
        for source in sources:
            app = pkg.App("bc", frag, comm, source_oid=source)
            st = app.query()
            got = gather(app.result())
            if rank == 0:
                c, sigma, depth = BO.bc_rows(n, grp, gcol, source if source < n else None, short=None)
                reached = depth != BO.INF
                L = int(depth[reached].max()) if reached.any() else 0
                ok = (np.array_equal(got["depth"], depth)
                      and got["path_num"].tobytes() == sigma.tobytes()
                      and got["centrality"].tobytes() == c.astype(np.float64).tobytes())
                print("[mgpu-bc] %-18s source=%-6d fnum=%d n=%d levels=%d rounds=%d %s"
                      % (name, source, world, n, L + 1 if reached.any() else 0, st.supersteps,
                         "OK" if ok else "MISMATCH"), flush=True)
                runs += 1
                if not ok:
                    failures.append("%s:%d" % (name, source))
            app.close()
            dist.barrier()
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
