"""Betweenness centrality over a list of sources on a fragment group: launched by torchrun (one rank per
fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  Block- and hash-partitioned graphs
(hash: lids out of oid order); every rank sends its CSR, mapped to global vertex indices, to rank 0,
which compares the concatenated inner results with the oracle (oracle/bc_sources_oracle.py) on that
CSR within 1e-12 relative (the fragments' rows are summed in their own order), checks that batch widths
1, 7 and 32 give bit-identical output and that the shares of frontier_vertices / touched_vertices add
up to the oracle's counts.  When the ranks' free HBM allows different batch widths (reserved[1], set on
rank 0 only), the group runs at the smallest: every rank makes the same worker rounds as with that width
requested, with the same bits.  An empty list gives zeros and zero counts on every rank.  A communicator whose mirror area cannot hold one 8-byte row per outer copy
is refused.  Rank 0 prints one OK / MISMATCH line per run and a closing "runs=" line."""
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
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    pkg = importlib.import_module("libgrape-lite_b200")
    gdist = importlib.import_module("libgrape-lite_b200.dist")
    from oracle import bc_sources_oracle as BSO
    from tests import bc_shapes as B
    from tests import partition_cases as P
    from tests import shapes as S
    failures, runs = [], 0

    def gather(arr):
        out = [None] * world
        dist.all_gather_object(out, arr)
        return out

    rm = pkg.rmat_edges_host(12, 16, 17, 0)
    cases = {"rmat12": (1 << 12, rm[0], rm[1]), "star": S.star(4097)[:3],
             "union": S.union([S.star(1500), S.clique(30), S.path(40), S.empty(5)], seed=9)[:3],
             "multi_loop": S.multi_loop()[:3], "kab33_2048": B.BC_SHAPES["kab33_2048"][0]()[:3]}
    for name, (n, s, d) in cases.items():
        for part in ("block", "hash"):
            if part == "block":
                frag = pkg.Fragment.from_edges(n, s, d, None, fid=rank, fnum=world)
            else:
                oids = np.arange(n, dtype=np.int64)
                owner, key = P.partition("hash", n, s, d, oids, world)
                frag = P.from_layout(pkg, P.describe(n, s, d, None, oids, False, owner, key, world), rank, False)
            # a mirror area of 8 * 33 bytes per inner vertex of the largest fragment: 32-lane rows fit, so the
            # batch widths below are the ones run, not clamped by the area
            comm = gdist.make_comm(rank, world, 33 * max(frag.ivnum, 1))
            # global vertex index = oid; this fragment's rows with every column mapped to its oid
            app0 = pkg.App("bc_sources", frag, comm, sources=[])
            my_oids = app0.result_oids()
            app0.close()
            rp, col, _ = frag.csr(0)
            col = col.astype(np.int64)
            ovg = frag.ovgid().astype(np.int64)
            all_oids = gather(my_oids)
            outer = col >= frag.ivnum
            g = ovg[col[outer] - frag.ivnum]
            fo = g >> frag.fid_offset
            lo = g & ((1 << frag.fid_offset) - 1)
            gcol = np.empty_like(col)
            gcol[~outer] = my_oids[col[~outer]]
            gcol[outer] = np.array([all_oids[f][l] for f, l in zip(fo, lo)], dtype=np.int64)
            parts = gather((my_oids, np.diff(rp.astype(np.int64)), gcol))
            rng = np.random.default_rng(n)
            lst = [int(np.argmax(np.bincount(np.concatenate([s, d]), minlength=n)))] + \
                rng.integers(0, n, size=40).tolist() + [n + 5]
            outs = {}
            for Bw in (1, 7, 32):
                app = pkg.App("bc_sources", frag, comm, sources=lst, reserved={0: Bw})
                st = app.query()
                res = gather((my_oids, app.result(), st.frontier_vertices, st.touched_vertices, st.supersteps))
                app.close()
                outs[Bw] = res
            # rank 0's free HBM taken to hold 3 lanes, the others' 32: the group must agree on 3
            app = pkg.App("bc_sources", frag, comm, sources=lst, reserved={1: 3} if rank == 0 else {})
            st = app.query()
            hook = gather((app.result().tobytes(), st.supersteps))
            app.close()
            app = pkg.App("bc_sources", frag, comm, sources=lst, reserved={0: 3})
            st = app.query()
            three = gather((app.result().tobytes(), st.supersteps))
            app.close()
            app = pkg.App("bc_sources", frag, comm, sources=[])
            st = app.query()
            empty = gather((bool(app.result().any()), st.frontier_vertices, st.touched_vertices))
            app.close()
            if rank == 0:
                # the group's CSR in oid order
                rows = {}
                for oids_f, deg_f, col_f in parts:
                    off = np.concatenate([[0], np.cumsum(deg_f)])
                    for i, o in enumerate(oids_f):
                        rows[int(o)] = col_f[off[i]:off[i + 1]]
                grp = np.zeros(n + 1, dtype=np.int64)
                grp[1:] = np.cumsum([len(rows.get(v, ())) for v in range(n)])
                gc = np.concatenate([rows.get(v, np.zeros(0, np.int64)) for v in range(n)]) if n else np.zeros(0)
                want, stats = BSO.bc_sources(n, grp, gc.astype(np.int64), [v if v < n else None for v in lst])
                ok = True
                ref_bytes = None
                for Bw, res in outs.items():
                    got = np.zeros(n)
                    for oids_f, vals, _, _, _ in res:
                        got[oids_f] = vals
                    ok &= bool(np.allclose(got, want, rtol=1e-12, atol=1e-12))
                    ok &= sum(r[2] for r in res) == stats["frontier_vertices"]
                    ok &= sum(r[3] for r in res) == stats["touched_vertices"]
                    b = got.tobytes()
                    ok &= ref_bytes is None or b == ref_bytes
                    ref_bytes = b
                ok &= hook == three and len({r[1] for r in hook}) == 1
                ok &= hook[0][1] != outs[32][0][4]   # 14 batches of 3, not 2 of 32
                ok &= all(e == (False, 0, 0) for e in empty)
                print("[mgpu-bcs] %-12s %-5s fnum=%d n=%d sources=%d %s"
                      % (name, part, world, n, len(lst), "OK" if ok else "MISMATCH"), flush=True)
                runs += 1
                if not ok:
                    failures.append("%s:%s" % (name, part))
            dist.barrier()
            comm.close()
            frag.close()
    # a mirror area too small for one 8-byte row per outer copy
    frag = pkg.Fragment.rmat(14, 16, seed=1, fid=rank, fnum=world)
    small = gdist.make_comm(rank, world, 1)
    refused = False
    try:
        pkg.App("bc_sources", frag, small)
    except pkg.GrapeError as e:
        refused = "mirror" in str(e) or "status -2" in str(e)
    flags = gather(refused)
    if rank == 0:
        print("[mgpu-bcs] refused mirror_bytes %s" % ("OK" if all(flags) else "MISMATCH"), flush=True)
        if not all(flags):
            failures.append("refusal")
    small.close()
    frag.close()
    if rank == 0:
        print("[mgpu-bcs] runs=%d" % runs, flush=True)
    flag = torch.tensor([len(failures)])
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
