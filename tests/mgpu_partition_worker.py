"""Every app on fragments that a host cut itself and handed to gl_frag_create: launched by torchrun
(one rank per fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).

Each rank builds its own gl_frag_desc from tests/partition_cases.py -- hash (the reference's edge-file
loader: `oid % fnum`, lids in order of first appearance), map (MapPartitioner over a shuffled vertex
list), skew (the 16 largest rows alone on the last fid), hollow (one fid without vertices) or the
library's own blocks -- and creates it with Fragment.from_csr(ovgid=, inner_oids=, total_vnum=, fid=,
fnum=, ie=).  It first checks that the library holds the fragment as described (csr 0/1/2, ovgid,
oid2lid), then runs the apps; rank 0 scatters every rank's result into oid order through result_oids
and compares it with the oracles.  Labels of WCC / CDLP follow gid order: the oracle runs on the graph
relabelled to gid rank and its labels are mapped back to oids (vertex map attached) or to raw gids
(several fragments, no vertex map).  LCC breaks degree ties on the gid too, which on a multigraph decides
what repeated edges count, so its oracle also runs in gid-rank order.  Rank 0 prints one OK / MISMATCH line per check; `expected_ok`
counts the OK lines a clean run prints."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

INT64_MAX = np.iinfo(np.int64).max
F64_MAX = np.finfo(np.float64).max
UNDIRECTED = ("rmat12", "star", "path", "multi_loop", "hub_block", "clique")


def cases(world):
    """(graph, partition) pairs run on `world` fragments."""
    out = [(g, p) for g in UNDIRECTED + ("rmat11_directed",) for p in ("hash", "map", "skew")]
    out.append(("rmat12", "blocks"))
    if world == 3:
        out += [("rmat12", "hollow"), ("p2p31", "hash")]
    if world == 2:
        out.append(("rmat17", "hash"))     # the default several-fragment BFS: hub-first order, delegated hubs
    return out


def app_runs(graph):
    """(label, kind, cfg, source role) of every run on one graph; role picks the source of BFS / SSSP / BC."""
    if graph == "rmat17":
        return [("bfs", "bfs", {}, "root")]
    bfs = [("bfs dopt=%d fuse=%d" % (o, f), "bfs", dict(direction_opt=o, fuse_supersteps=f), "root")
           for o in (0, 1) for f in (0, 1)]
    if graph == "rmat11_directed":
        return bfs + [("sssp f32", "sssp", {}, "root"),
                      ("pagerank push", "pagerank", dict(pr_delta=0.85, max_round=10), None),
                      ("wcc +vm", "wcc", {}, None)]
    runs = bfs + [("bfs hub-first", "bfs", dict(reserved={1: 2}), "root"),
                  ("bfs hub-first no-delegates", "bfs", dict(reserved={1: 3}), "root"),
                  ("bfs round-1 shipment", "bfs", dict(reserved={7: 1}), "root"),
                  ("bfs", "bfs", {}, "last"), ("bfs", "bfs", {}, "unknown")]
    if graph == "path":
        runs.append(("bfs ring=5", "bfs", dict(reserved={3: 5}), "root"))
    runs += [("sssp f32", "sssp", {}, "root"), ("sssp f32", "sssp", {}, "last")]
    if graph == "rmat12":
        runs.append(("sssp f64 real weights", "sssp", dict(sssp_f64=1), "root"))
    pr = dict(pr_delta=0.85, max_round=10)
    runs += [("pagerank push", "pagerank", pr, None), ("pagerank pull", "pagerank", dict(pr, pr_pull=1), None),
             ("pagerank pull f32", "pagerank", dict(pr, pr_pull=1, reserved={5: 1}), None),
             ("pagerank pull f32 no-hub", "pagerank", dict(pr, pr_pull=1, reserved={4: 1, 5: 1}), None),
             ("lcc", "lcc", {}, None), ("core_decomposition", "core_decomposition", {}, None),
             ("kcore k=3", "kcore", dict(k=3), None)]
    runs += [("kclique k=%d" % k, "kclique", dict(k=k), None) for k in (3, 4, 5)]
    runs += [("bc", "bc", {}, role) for role in ("root", "last", "unknown")]
    for vm in ("+vm", "-vm"):
        runs += [("wcc " + vm, "wcc", {}, None), ("wcc_opt " + vm, "wcc_opt", {}, None),
                 ("wcc dense " + vm, "wcc", dict(reserved={0: 1}), None),
                 ("cdlp r=1 " + vm, "cdlp", dict(max_round=1), None), ("cdlp r=5 " + vm, "cdlp", dict(max_round=5), None)]
    return runs


def expected_ok(world):
    """OK lines of a clean run: one layout check per case plus one per app run."""
    return sum(1 + len(app_runs(g)) for g, _ in cases(world))


def graph_of(pkg, name):
    """(n, src, dst, w, w_real, oids, directed): src / dst are vertex indices, oids ascending."""
    from tests import golden_io as G
    from tests import shapes as S
    w_real = None
    if name == "p2p31":
        oids, s, d, w = G.load_p2p31()
        return len(oids), np.searchsorted(oids, s), np.searchsorted(oids, d), w, None, oids, False
    if name.startswith("rmat"):
        scale = int(name[4:6])
        s, d, w = pkg.rmat_edges_host(scale, 16, 17, 1)
        if name == "rmat12":
            w_real = pkg.rmat_edges_host(scale, 16, 17, 2)[2]
        n = 1 << scale
    else:
        n, s, d, w = {"star": S.star(4097), "path": S.path(300), "multi_loop": S.multi_loop(),
                      "hub_block": S.hub_block(33), "clique": S.clique(40)}[name]
    return n, s, d, w, w_real, 7 * np.arange(n, dtype=np.int64) + 3, name.endswith("directed")


def main():
    import torch
    import torch.distributed as dist
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
    from oracle import core_oracle as CO
    from oracle import kclique_oracle as KO
    from oracle import pyoracle
    from tests import golden_io as G
    from tests import partition_cases as P
    failures = []

    def all_obj(x):
        out = [None] * world
        dist.all_gather_object(out, x)
        return out

    def report(what, ok):
        if rank == 0:
            print("[part] %-16s %-7s fnum=%d %-28s %s" % (case[0], case[1], world, what, "OK" if ok else "MISMATCH"),
                  flush=True)
            if not ok:
                failures.append("%s/%s/%s" % (case[0], case[1], what))

    def check(kind, cfg, label, got, s_idx, role):
        """p2p-31 is also held to the golden files where they exist (BFS and SSSP from oid 6)."""
        n, src, dst, w, w_real, oids, directed = graphs[case[0]]
        L_rank, by_rank = L.rank, L.by_rank
        golden = case[0] == "p2p31"
        if kind == "bfs":
            want = np.full(n, INT64_MAX) if s_idx is None else g.bfs(s_idx)[0]
            if golden and role == "root" and G.render(oids, [str(int(d)) for d in got]) != G.golden_lines("p2p-31-BFS"):
                return False
            return np.array_equal(got, want)
        if kind == "sssp":
            if s_idx is None:
                return np.all(got == F64_MAX)
            if cfg.get("sssp_f64"):
                want = pyoracle.Graph(n, src, dst, w_real.astype(np.float64)).sssp(s_idx)[0]
            else:
                want = g.sssp(s_idx)[0]
            if golden and role == "root" and (G.render(oids, ["infinity" if d == F64_MAX else G.fmt_sci(d) for d in got])
                                              != G.golden_lines("p2p-31-SSSP")):
                return False
            return np.array_equal(got, want)
        if kind == "pagerank":
            want = g.pagerank(0.85, 10, 2 if directed else 1)
            if golden:
                gold = np.array([float(v) for _, v in G.golden_pairs("p2p-31-PR")])
                if np.max(np.abs(got - gold) / gold) >= 1e-6:
                    return False
            if np.max(np.abs(got - want) / want) >= 1e-6:
                return False
            # a directed vertex without out-edges keeps rank = base and drops what arrives: no unit sum there
            f32 = cfg.get("reserved", {}).get(5) == 1
            return directed or abs(got.sum() - 1.0) < (1e-6 if f32 else 1e-9)
        if kind == "lcc":
            if golden and G.render(oids, [G.fmt_sci(x) for x in got]) != G.golden_lines("p2p-31-LCC"):
                return False
            # degree ties orient the triangles by gid, which decides what a multigraph's repeated edges count
            return np.array_equal(got, gr.lcc()[0][L_rank])
        if kind == "core_decomposition":
            return np.array_equal(got, CO.core_decomposition(n, src, dst)[0])
        if kind == "kcore":
            return np.array_equal(got, CO.kcore(n, src, dst, cfg["k"]))
        if kind == "bc":
            rp, col = L.global_csr()
            c, sigma, depth = BO.bc_rows(n, rp, col, None if s_idx is None else int(L_rank[s_idx]),
                                         short=None if world > 1 else 32)
            return (np.array_equal(got["depth"], depth[L_rank]) and got["path_num"].tobytes() == sigma[L_rank].tobytes()
                    and got["centrality"].tobytes() == c.astype(np.float64)[L_rank].tobytes())
        # WCC / CDLP: labels are gids inside the library; the oracle runs in gid-rank indices
        lab = gr.cdlp(cfg["max_round"]) if kind == "cdlp" else gr.wcc()[0].astype(np.int64)
        lab = lab[L_rank]                                  # per vertex index: the label's gid rank
        if label.endswith("+vm") or directed or world == 1:
            want = oids[by_rank[lab]]
        else:
            want = L.gid[by_rank[lab]]
        return np.array_equal(got, want)

    graphs, want_cache = {}, {}
    for case in cases(world):
        gname, part = case
        if gname not in graphs:
            graphs[gname] = graph_of(pkg, gname)
        n, src, dst, w, w_real, oids, directed = graphs[gname]
        w32 = None if w is None else np.asarray(w, np.float32)
        owner, key = P.partition(part, n, src, dst, oids, world)
        L = P.describe(n, src, dst, w32, oids, directed, owner, key, world)
        me = L.frags[rank]
        frag = P.from_layout(pkg, L, rank, directed)

        # ---- the library holds the fragment as described
        ok = True
        for which, k in ((0, "oe"), (1, "ie" if directed else "oe")):
            rp, col, ww = frag.csr(which)
            mrp, mcol, mw = me[k]
            ok = ok and np.array_equal(rp, mrp) and np.array_equal(col, mcol)
            ok = ok and (mw is None or P.same_weights(rp, col, ww, mw))
        vrp, vcol, _ = frag.csr(2)
        ok = ok and np.array_equal(vrp, me["ovie"][0]) and np.array_equal(vcol, me["ovie"][1])
        ok = ok and np.array_equal(frag.ovgid(), me["ovgid"]) and frag.ivnum == me["ivnum"] and frag.ovnum == me["ovnum"]
        ok = ok and all(frag.oid2lid(o) == l for l, o in enumerate(me["inner_oids"]))
        others = oids[owner != rank][:50]
        ok = ok and all(frag.oid2lid(o) is None for o in list(others) + [-1, int(oids[-1]) + 1])
        report("layout", all(all_obj(bool(ok))))

        comm = gdist.make_comm(rank, world, frag.ivnum)
        frag_real = None
        if w_real is not None:
            Lr = P.describe(n, src, dst, w_real, oids, directed, owner, key, world)
            frag_real = P.from_layout(pkg, Lr, rank, directed)
        vm = pkg.VertexMap([f["inner_oids"] for f in L.frags])
        deg = P.degrees(n, src, dst)
        iv = np.array([f["ivnum"] for f in L.frags])
        small = int(np.argmin(np.where(iv > 0, iv, n + 1)))
        sources = {"root": 0 if gname == "path" else int(np.argmax(deg)),    # the end of the path, else the largest row
                   "last": int(L.frags[small]["inner"][-1]), "unknown": None}
        if gname == "p2p31":
            sources["root"] = int(np.searchsorted(oids, 6))
        unknown_oid = int(oids[-1]) + 1000
        g = gr = None
        if rank == 0:
            g = pyoracle.Graph(n, src, dst, None if w is None else np.asarray(w32, np.float64), directed=directed)
            gr = pyoracle.Graph(n, L.rank[src], L.rank[dst], None, directed=directed)
        for label, kind, cfg, role in app_runs(gname):
            s_idx = sources.get(role) if role else None
            cfg = dict(cfg)
            if role:
                cfg["source_oid"] = unknown_oid if s_idx is None else int(oids[s_idx])
            use_vm = label.endswith("+vm") or (kind in ("wcc", "wcc_opt") and directed)
            f = frag_real if cfg.get("sssp_f64") else frag
            app = pkg.App(kind, f, comm, **cfg)
            if use_vm:
                app.set_vertex_map(vm)
            app.query()
            res = app.result()
            parts = all_obj((res, None if kind == "kclique" else app.result_oids()))
            app.close()
            if rank == 0:
                if kind == "kclique":
                    ck = (gname, cfg["k"])
                    if ck not in want_cache:
                        want_cache[ck] = KO.count(n, src, dst, ck[1])
                    ok = all(int(p[0]) == want_cache[ck] for p in parts)
                else:
                    ro = np.concatenate([p[1] for p in parts])
                    ok = np.array_equal(np.sort(ro), oids)
                    got = np.empty(n, dtype=res.dtype)
                    got[np.searchsorted(oids, ro)] = np.concatenate([p[0] for p in parts])
                    try:
                        ok = ok and check(kind, cfg, label, got, s_idx, role)
                    except Exception as e:     # a broken check is a failed case, not a hung group
                        print("[part] check raised %r" % e, flush=True)
                        ok = False
                report(label, ok)
            dist.barrier()

        comm.close()
        vm.close()
        frag.close()
        if frag_real is not None:
            frag_real.close()

    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
