"""Multi-fragment parity worker: launched by torchrun (one rank per GPU).
Every app runs on an edge-cut R-MAT graph split into WORLD_SIZE fragments and
rank 0 compares the concatenated inner results with the whole-graph oracle."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    scale = int(sys.argv[1]) if len(sys.argv) > 1 else 14
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    # GL_ONE_DEVICE=1: every rank's fragment lives on cuda:0 (the contexts of the
    # rank processes time-slice one GPU; CUDA IPC maps the landing areas across
    # them) -- the multi-fragment data plane on a 1-GPU box.  Rendezvous: gloo.
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
    failures = []

    def gather(arr):
        out = [None] * world
        dist.all_gather_object(out, arr)
        return np.concatenate(out)

    def face2_sssp(frag, comm, source):
        """SSSP written against Face 2 only (gl_mm_* + gl_edge_scan_queue +
        gl_compact_bitmap): what a C host would do per IncEval (cuda/sssp/sssp.h:173-305)."""
        capi = pkg.capi
        tv = frag.ivnum + frag.ovnum
        words = (tv + 31) // 32 + 1
        dist_h = np.full(tv, np.finfo(np.float32).max, dtype=np.float32)
        active_h = np.zeros(words, dtype=np.uint32)
        lid = frag.oid2lid(source)
        if lid is not None:
            dist_h[lid] = 0.0
            active_h[lid >> 5] |= np.uint32(1 << (lid & 31))
        dist = capi.DeviceArray(dist_h)
        active = capi.DeviceArray(active_h)
        nxt = capi.DeviceArray(np.zeros(words, dtype=np.uint32))
        queue = capi.DeviceArray(nbytes=4 * (frag.ivnum + 1))
        mm = capi.MessageManager(comm)
        mm.init_buffer(8 * frag.ovnum, 8 * frag.ivnum)
        mm.start()
        mm.start_round()
        mm.force_continue()          # PEval
        mm.finish_round()
        rounds = 1
        while not mm.to_terminate():
            mm.start_round()
            mm.process("min_f32", state=dist, out_bitmap=active)
            n = capi.compact_bitmap(active, frag.ivnum, queue)
            active.fill(0)
            if n:
                capi.edge_scan_queue(frag, queue, n, "min_relax_f32", "cm", state=dist, out_bitmap=nxt, use_weight=1)
            mm.send_outer(frag, nxt, state=dist, value_bytes=4, clear_bits=True)
            if capi.bitmap_count(nxt, frag.ivnum) > 0:
                mm.force_continue()
            active, nxt = nxt, active
            mm.finish_round()
            rounds += 1
        out = dist.download(np.float32, tv)[: frag.ivnum].astype(np.float64)
        out[out == np.finfo(np.float32).max] = np.finfo(np.float64).max
        total = mm.allreduce(mm.bytes_sent())
        mm.close()
        return out, rounds, total

    if os.environ.get("GL_SHAPES", "0") == "1" or os.environ.get("GL_RESOURCES", "0") == "1":
        if os.environ.get("GL_SHAPES", "0") == "1":
            run_shapes(pkg, gdist, pyoracle, rank, world, gather, failures)
        else:
            run_resources(pkg, gdist, rank, world, scale, dist.barrier, failures)
        flag = torch.tensor([len(failures)], device=dev)
        dist.broadcast(flag, 0)
        dist.destroy_process_group()
        sys.exit(1 if int(flag.item()) else 0)

    for wmode, apps in ((0, ["bfs", "bfs_hub", "bfs_hub_src2", "bfs_hub_nodlg", "bfs_spill", "bfs_spill_src2", "bfs_nohub", "bfs_r1ship", "bfs_push", "bfs_step", "bfs_push_step", "wcc", "wcc_opt", "pagerank", "pagerank_pull", "cdlp", "lcc"]), (1, ["sssp", "face2_sssp"])):
        n = 1 << scale
        frag = pkg.Fragment.rmat(scale, 16, seed=17, weight_mode=wmode, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        g = None
        if rank == 0:
            src, dst, w = pkg.rmat_edges_host(scale, 16, 17, wmode)
            g = pyoracle.Graph(n, src, dst, None if w is None else w.astype(np.float64))
            source = g.max_degree_vertex()
            # a second source that is NOT one of the highest-degree vertices (the delegated hubs)
            deg = np.bincount(np.concatenate([src, dst]), minlength=n)
            source2 = int(np.flatnonzero(deg == np.sort(deg[deg > 0])[len(deg[deg > 0]) // 2])[0])
        else:
            source = source2 = 0
        src_t = torch.tensor([source, source2], dtype=torch.int64, device=dev)
        dist.broadcast(src_t, 0)
        source, source2 = int(src_t[0].item()), int(src_t[1].item())
        only = os.environ.get("GL_APPS")
        if only:
            apps = [a for a in apps if a in only.split(",")]
        for name in apps:
            cfg = {}
            kind = name
            if name.startswith("bfs"):
                kind = "bfs"
                # default = whole query fused into one cooperative kernel per GPU;
                # *_step = one superstep per round through the host loop
                cfg = dict(source_oid=source, direction_opt=0 if "push" in name else 1,
                           fuse_supersteps=0 if name.endswith("_step") else 1)
                if name == "bfs_r1ship":     # round-1 frontier shipment (per-holder bit-compressed slices)
                    cfg["reserved"] = {7: 1}
                if name == "bfs_hub":        # hub-first relabelling inside every fragment, also on a small graph
                    cfg["reserved"] = {1: 2}
                if name == "bfs_hub_src2":   # hub-first order, source of median degree (not a delegated hub)
                    cfg["reserved"] = {1: 2}
                    cfg["source_oid"] = source2
                if name == "bfs_hub_nodlg":  # hub-first order without the delegated-hub lists
                    cfg["reserved"] = {1: 3}
                if name == "bfs_spill":      # a ring of 4 level bitmaps: the fused kernel parks, the host spills, relaunch
                    cfg["reserved"] = {1: 2, 3: 4}
                if name == "bfs_spill_src2":
                    cfg["reserved"] = {1: 1, 3: 4}
                    cfg["source_oid"] = source2
                if name == "bfs_nohub":      # the fragment's own vertex order
                    cfg["reserved"] = {1: 1}
            elif name == "sssp":
                cfg = dict(source_oid=source)
            elif name.startswith("pagerank"):
                kind = "pagerank"
                cfg = dict(pr_delta=0.85, max_round=10, pr_pull=1 if name.endswith("pull") else 0)
            elif name == "cdlp":
                cfg = dict(max_round=5)
            if name == "face2_sssp":
                res, rounds, total = face2_sssp(frag, comm, source)
                got = gather(res)
                if rank == 0:
                    ok = np.array_equal(got, g.sssp(source)[0])
                    print("[mgpu] %-13s fnum=%d scale=%d supersteps=%d msg_bytes=%d %s"
                          % (name, world, scale, rounds, total, "OK" if ok else "MISMATCH"), flush=True)
                    if not ok:
                        failures.append(name)
                dist.barrier()
                continue
            app = pkg.App(kind, frag, comm, **cfg)
            st = app.query()
            got = gather(app.result())
            if rank == 0:
                if kind == "bfs":
                    ok = np.array_equal(got, g.bfs(cfg["source_oid"])[0])
                elif kind == "sssp":
                    ok = np.array_equal(got, g.sssp(source)[0])
                elif kind in ("wcc", "wcc_opt"):
                    ok = np.array_equal(got, g.wcc()[0].astype(np.int64))
                elif kind == "cdlp":
                    ok = np.array_equal(got, g.cdlp(5))
                elif kind == "lcc":
                    ok = np.array_equal(got, g.lcc()[0])
                else:
                    want = g.pagerank(0.85, 10, 1)
                    ok = bool(np.max(np.abs(got - want) / want) < 1e-6)
                print("[mgpu] %-13s fnum=%d scale=%d supersteps=%d msg_bytes=%d %s"
                      % (name, world, scale, st.supersteps, st.msg_bytes_sent, "OK" if ok else "MISMATCH"), flush=True)
                if not ok:
                    failures.append(name)
            app.close()
            dist.barrier()
        comm.close()
        frag.close()
    # WCC / CDLP on a fragment group with EXPLICIT oids: labels are gids internally; with the device
    # vertex map attached (gl_vm_*, gl_app_set_vertex_map) the results come back as oids
    scale2 = min(scale, 11)
    n2 = 1 << scale2
    oids = (np.arange(n2, dtype=np.int64) * 7 + 3)
    src, dst, _ = pkg.rmat_edges_host(scale2, 16, 23, 0)
    frag = pkg.Fragment.from_edges(n2, oids[src], oids[dst], None, oids=oids, fid=rank, fnum=world)
    comm = gdist.make_comm(rank, world, frag.ivnum)
    chunk = (n2 + world - 1) // world
    vm = pkg.VertexMap([oids[f * chunk:(f + 1) * chunk] for f in range(world)])
    g2 = pyoracle.Graph(n2, oids[src], oids[dst], None, oids=oids) if rank == 0 else None
    for kind in ("wcc", "wcc_opt", "cdlp"):
        app = pkg.App(kind, frag, comm, **({"max_round": 5} if kind == "cdlp" else {}))
        app.set_vertex_map(vm)
        app.query()
        got = gather(app.result())
        if rank == 0:
            want = g2.cdlp(5) if kind == "cdlp" else oids[g2.wcc()[0].astype(np.int64)]
            ok = np.array_equal(got, want)
            print("[mgpu] %-13s fnum=%d scale=%d explicit oids + vertex map %s" % (kind + "_oids", world, scale2, "OK" if ok else "MISMATCH"), flush=True)
            if not ok:
                failures.append(kind + "_oids")
        app.close()
        dist.barrier()
    vm.close()
    comm.close()
    frag.close()
    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


def run_resources(pkg, gdist, rank, world, scale, barrier, failures):
    """GL_RESOURCES=1: every app configuration runs create -> query -> result -> destroy on its
    fragment group once as warm-up and three more times; the free device memory (all ranks share
    cuda:0) must end where the warm-up left it."""
    frag = pkg.Fragment.rmat(scale, 16, seed=17, weight_mode=1, fid=rank, fnum=world)
    comm = gdist.make_comm(rank, world, frag.ivnum)

    def free_bytes():
        torch.cuda.synchronize()
        barrier()
        f = torch.cuda.mem_get_info()[0]
        barrier()
        return f

    configs = [("bfs", dict(source_oid=0, fuse_supersteps=1)), ("bfs", dict(source_oid=0, fuse_supersteps=0)),
               ("sssp", dict(source_oid=0, sssp_f64=0)), ("sssp", dict(source_oid=0, sssp_f64=1)),
               ("wcc", {}), ("wcc_opt", {}), ("pagerank", dict(pr_pull=0)), ("pagerank", dict(pr_pull=1)),
               ("cdlp", dict(max_round=5)), ("lcc", {})]
    for kind, cfg in configs:
        frees = []
        for it in range(4):
            app = pkg.App(kind, frag, comm, **cfg)
            app.query()
            app.result()
            app.close()
            frees.append(free_bytes())
        ok = frees[-1] == frees[0]
        if rank == 0:
            print("[mgpu] %-9s %-32s fnum=%d scale=%d free after cycles %s %s"
                  % (kind, cfg, world, scale, frees, "RELEASED" if ok else "LEAKED"), flush=True)
        if not ok:
            failures.append(kind)
    comm.close()
    frag.close()


def run_shapes(pkg, gdist, pyoracle, rank, world, gather, failures):
    """GL_SHAPES=1: the constructed threshold graphs of tests/shapes.py split into
    WORLD_SIZE fragments -- a star whose centre (fragment 0) has outer copies on
    every peer, fragments without edges or outer vertices, owner boundaries inside
    a bitmap word, a block of long rows and a long multi-edge -- through all six apps."""
    from tests import shapes as S
    cases = {"star": S.star(4097), "path": S.path(300), "path_then_isolated": S.pad_to(S.path(300), 1000),
             "empty": S.empty(33), "hub_block": S.hub_block(33), "multi_loop": S.multi_loop()}
    apps = [("bfs", dict(direction_opt=1)), ("bfs_push", dict(direction_opt=0)), ("bfs_step", dict(fuse_supersteps=0)),
            ("sssp", {}), ("wcc", {}), ("wcc_opt", {}), ("pagerank", dict(pr_delta=0.85, max_round=10)),
            ("pagerank_pull", dict(pr_delta=0.85, max_round=10, pr_pull=1)), ("cdlp", dict(max_round=5)), ("lcc", {})]
    for shape, (n, src, dst, w) in cases.items():
        frag = pkg.Fragment.from_edges(n, src, dst, w, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        g = pyoracle.Graph(n, src, dst, w) if rank == 0 else None
        source = 0                                   # the star centre, an end of the path, an isolated vertex
        for name, cfg in apps:
            kind = name.split("_")[0] if name != "wcc_opt" else name
            if kind in ("bfs", "sssp"):
                cfg = dict(cfg, source_oid=source)
            app = pkg.App(kind, frag, comm, **cfg)
            app.query()
            got = gather(app.result())
            if rank == 0:
                if kind == "bfs":
                    ok = np.array_equal(got, g.bfs(source)[0])
                elif kind == "sssp":
                    ok = np.array_equal(got, g.sssp(source)[0])
                elif kind in ("wcc", "wcc_opt"):
                    ok = np.array_equal(got, g.wcc()[0].astype(np.int64))
                elif kind == "cdlp":
                    ok = np.array_equal(got, g.cdlp(5))
                elif kind == "lcc":
                    ok = np.array_equal(got, g.lcc()[0])
                else:
                    want = g.pagerank(0.85, 10, 1)
                    ok = bool(np.max(np.abs(got - want) / want) < 1e-6)
                print("[mgpu] shape %-18s %-13s fnum=%d n=%d %s" % (shape, name, world, n, "OK" if ok else "MISMATCH"),
                      flush=True)
                if not ok:
                    failures.append(shape + ":" + name)
            app.close()
            dist.barrier()
        comm.close()
        frag.close()


if __name__ == "__main__":
    main()
