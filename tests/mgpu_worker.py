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

    if any(os.environ.get(k, "0") == "1" for k in ("GL_SHAPES", "GL_RESOURCES", "GL_FACE2")):
        if os.environ.get("GL_SHAPES", "0") == "1":
            run_shapes(pkg, gdist, pyoracle, rank, world, gather, failures)
        elif os.environ.get("GL_FACE2", "0") == "1":
            run_face2(pkg, gdist, rank, world, failures)
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


def run_face2(pkg, gdist, rank, world, failures):
    """GL_FACE2=1: the message manager of the C ABI checked item by item.  Every rank builds the
    same seeded inputs for every fragment, so it can compute what each call must do on its own
    fragment: send_outer + process for every (value_bytes, clear_bits, consumer kind), the round
    protocol (visibility, termination vote, force_continue, bytes_sent, round 0 of a second
    query), the dense mirror sync of values and bits, gl_allreduce, and a symmetric landing-slot
    overflow.  A failed check is recorded and the run carries on, so every rank issues the same
    sequence of collective calls."""
    import math
    import struct
    import zlib
    import ctypes as C
    import torch.distributed as dist
    from tests import shapes as S
    capi = pkg.capi
    L = capi.lib()
    mine = []

    def check(what, ok):
        if not ok:
            mine.append(what)
            print("[face2] rank %d FAIL %s" % (rank, what), flush=True)

    def all_obj(x):
        out = [None] * world
        dist.all_gather_object(out, x)
        return out

    def rng_of(*tag):
        return np.random.default_rng([zlib.crc32(repr(tag).encode())])

    def bits_of(words, n):
        return np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)

    def words_of(bits, nwords):
        w = np.zeros(nwords, dtype=np.uint32)
        idx = np.flatnonzero(bits)
        np.bitwise_or.at(w, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
        return w

    src12, dst12, _ = pkg.rmat_edges_host(12, 16, 5, 0)
    cases = {"star": S.star(4097), "path": S.path(300), "path_then_isolated": S.pad_to(S.path(300), 1000),
             "empty": S.empty(33),
             "rmat12": (1 << 12, src12, dst12, None)}
    for shape, (n, src, dst, w) in cases.items():
        nfail0 = len(mine)
        frag = pkg.Fragment.from_edges(n, src, dst, w, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        info = all_obj((frag.ivnum, frag.ovnum, frag.ovgid().astype(np.int64)))
        iv = [i[0] for i in info]
        ov = [i[1] for i in info]
        tvs = [iv[r] + ov[r] for r in range(world)]
        tv = tvs[rank]
        nw = [(t + 31) // 32 + 1 for t in tvs]
        mm = capi.MessageManager(comm)
        vw = mm.view()
        off, mask = vw.fid_offset, vw.id_mask
        owner = [info[r][2] >> off for r in range(world)]
        olid = [info[r][2] & mask for r in range(world)]

        # ---- dense mirror sync: values (4 and 8 bytes, three syncs each) and bits
        mm.mirror_plan(frag)
        special = {4: np.array([0x7FC00001, 0xFFC12345, 0x80000000, 0x00000001, 0x007FFFFF, 0x7F800000], np.uint32),
                   8: np.array([0x7FF0000000000001, 0xFFF8DEADBEEF0000, 0x8000000000000000, 1,
                                0x000FFFFFFFFFFFFF, 0xFFF0000000000000], np.uint64)}
        for eb, dt in ((4, np.uint32), (8, np.uint64)):
            for it in range(3):
                vals = []
                for r in range(world):
                    g = rng_of(shape, "vals", eb, it, r)
                    v = g.integers(0, np.iinfo(dt).max, tvs[r], dtype=dt, endpoint=True)
                    k = min(iv[r], len(special[eb]))
                    v[:k] = np.roll(special[eb], it + r)[:k]       # the star centre is lid 0 of fragment 0
                    vals.append(v)
                d_v = capi.DeviceArray(vals[rank])
                mm.sync_values(d_v, eb)
                got = d_v.download(dt, tv)
                want = vals[rank].copy()
                for f in range(world):
                    sel = np.flatnonzero(owner[rank] == f)
                    want[iv[rank] + sel] = vals[f][olid[rank][sel]]
                check("%s sync_values %dB #%d" % (shape, eb, it), np.array_equal(got, want))
        for it in range(2):
            bms = [rng_of(shape, "bits", it, r).random(tvs[r]) < 0.3 for r in range(world)]
            d_b = capi.DeviceArray(words_of(bms[rank], nw[rank]))
            mm.sync_bits(d_b)
            want = bms[rank].copy()
            for f in range(world):
                sel = np.flatnonzero(owner[rank] == f)
                want[iv[rank] + sel] |= bms[f][olid[rank][sel]]
            check("%s sync_bits #%d" % (shape, it), np.array_equal(bits_of(d_b.download(np.uint32, nw[rank]), tv), want))

        # ---- send_outer + process, every value_bytes x clear_bits x consumer kind
        mm.start()
        sent_bytes = 0
        item_size = {0: 4, 4: 8, 8: 16}
        combos = [(0, "set_bit"), (4, "min_u32"), (4, "min_f32"), (4, "add_f32"), (4, "add_f32_real"),
                  (8, "min_f64"), (8, "add_f64")]
        for vb, kind in combos:
            for clear in (0, 1):
                tag = (shape, vb, kind, clear)
                remote = [rng_of(tag, "remote", r).random(nw[r] * 32) < 0.5 for r in range(world)]
                dt = {0: np.uint32, 4: np.uint32, 8: np.uint64}[vb]
                fdt = np.float64 if vb == 8 else np.float32
                sstate = []
                for r in range(world):
                    g = rng_of(tag, "send", r)
                    if kind == "min_u32":
                        sstate.append(g.integers(0, 1 << 20, tvs[r]).astype(np.uint32))
                    elif kind.startswith("min"):
                        sstate.append((g.random(tvs[r]) * 1000).astype(fdt).view(dt))
                    elif kind == "add_f32_real":
                        sstate.append((g.standard_normal(tvs[r]) * 10.0 ** g.uniform(-2, 2, tvs[r])).astype(fdt).view(dt))
                    else:
                        sstate.append(g.integers(-100, 100, tvs[r]).astype(fdt).view(dt))
                # items each owner receives: (lid, value bits)
                inbox_l, inbox_v, total = [], [], 0
                for r in range(world):
                    sel = np.flatnonzero(remote[r][iv[r]:tvs[r]])
                    total += len(sel)
                    if r == rank:
                        sent_bytes += len(sel) * item_size[vb]
                    to_me = sel[owner[r][sel] == rank]
                    inbox_l.append(olid[r][to_me])
                    inbox_v.append(sstate[r][iv[r] + to_me])
                lids = np.concatenate(inbox_l).astype(np.int64)
                vals = np.concatenate(inbox_v).astype(dt)
                d_remote = capi.DeviceArray(words_of(remote[rank], nw[rank]))
                d_sstate = capi.DeviceArray(sstate[rank]) if vb else None
                mm.start_round()
                check("%s: nothing visible in the round after a process round" % (tag,), mm.process("set_bit") == 0)
                mm.send_outer(frag, d_remote, state=d_sstate, value_bytes=vb, clear_bits=clear)
                mm.finish_round()
                check("%s: vote after the send round" % (tag,), mm.to_terminate() == (total == 0))
                want_remote = remote[rank].copy()
                if clear:
                    want_remote[iv[rank]:tv] = False
                check("%s: remote bitmap after send_outer" % (tag,),
                      np.array_equal(bits_of(d_remote.download(np.uint32, nw[rank]), nw[rank] * 32), want_remote))
                # the receiving round
                g = rng_of(tag, "recv", rank)
                ob0 = g.random(tv) < (0.0 if kind.startswith("min") else 0.3)
                d_ob = capi.DeviceArray(words_of(ob0, nw[rank]))
                if kind == "set_bit":
                    init = None
                elif kind == "min_u32":
                    init = np.where(g.random(tv) < 0.2, 0xFFFFFFFF, g.integers(0, 1 << 20, tv)).astype(np.uint32)
                elif kind.startswith("min"):
                    init = (g.random(tv) * 1000).astype(fdt)
                elif kind == "add_f32_real":
                    init = np.zeros(tv, fdt)
                else:
                    init = g.integers(-100, 100, tv).astype(fdt)
                d_st = capi.DeviceArray(init) if init is not None else None
                mm.start_round()
                items = mm.process(kind.replace("_real", ""), state=d_st, out_bitmap=d_ob)
                mm.finish_round()
                check("%s: items received" % (tag,), items == len(lids))
                check("%s: vote after the receiving round" % (tag,), mm.to_terminate())
                ob = bits_of(d_ob.download(np.uint32, nw[rank]), tv)
                if kind == "set_bit":
                    want_ob = ob0.copy()
                    want_ob[lids] = True
                    check("%s: bits ORed" % (tag,), np.array_equal(ob, want_ob))
                    continue
                got = d_st.download(init.dtype, tv)
                if kind.startswith("min"):
                    want = init.copy()
                    np.minimum.at(want, lids, vals.view(init.dtype))
                    check("%s: min state" % (tag,), np.array_equal(got, want))
                    check("%s: out_bitmap = dropped lids" % (tag,), np.array_equal(ob, want < init))
                    continue
                check("%s: out_bitmap untouched" % (tag,), np.array_equal(ob, ob0))
                x = vals.view(init.dtype).astype(np.float64)
                if kind == "add_f32_real":
                    bad = 0
                    for v in np.unique(lids):
                        xs = x[lids == v]        # k addends from 0: k - 1 f32 roundings (u = 2^-24)
                        err = math.fsum(np.concatenate([[float(got[v])], -xs]))
                        j, u = len(xs) - 1, 2.0 ** -24
                        if abs(err) > j * u / (1.0 - j * u) * math.fsum(np.abs(xs)):
                            bad += 1
                    bad += int(np.sum(got[np.setdiff1d(np.arange(tv), lids)] != 0))
                    check("%s: sums within the f32 recursive-summation bound" % (tag,), bad == 0)
                else:
                    want = init.astype(np.float64)
                    np.add.at(want, lids, x)
                    check("%s: integer sums" % (tag,), np.array_equal(got, want.astype(init.dtype)))
        check("%s: bytes_sent" % shape, mm.bytes_sent() == sent_bytes)

        # ---- round protocol
        senders = [r for r in range(world) if ov[r] > 0]
        if senders:
            sr = senders[-1]
            one = np.zeros(nw[sr] * 32, bool)
            one[iv[sr]] = True
            d_one = capi.DeviceArray(words_of(one if rank == sr else np.zeros(nw[rank] * 32, bool), nw[rank]))
            mm.start_round()
            mm.send_outer(frag, d_one, value_bytes=0)
            mm.finish_round()
            check("%s: one item from fid %d keeps every rank running" % (shape, sr), not mm.to_terminate())
            mm.start_round()
            got = mm.process("set_bit")
            mm.finish_round()
            check("%s: the one item arrives at its owner only" % shape, got == int(rank == owner[sr][0]))
            check("%s: then every rank terminates" % shape, mm.to_terminate())
        mm.start_round()
        if rank == world - 1:
            mm.force_continue()
        mm.finish_round()
        check("%s: force_continue on one rank keeps every rank running" % shape, not mm.to_terminate())
        mm.start_round()
        mm.finish_round()
        check("%s: no sends, no force_continue: every rank terminates" % shape, mm.to_terminate())
        # a second query receives nothing in its round 0, whichever parity the first one ended on
        full = [rng_of(shape, "full", r).random(nw[r] * 32) < 0.7 for r in range(world)]
        d_full = capi.DeviceArray(nbytes=4 * nw[rank])
        for rounds in (2, 3):
            mm.start()
            for r in range(rounds):
                mm.start_round()
                if r > 0:
                    d_full.upload(words_of(full[rank], nw[rank]))
                    mm.send_outer(frag, d_full, value_bytes=0)
                mm.finish_round()
            mm.start()
            mm.start_round()
            got = mm.process("set_bit")
            mm.finish_round()
            check("%s: round 0 after a %d-round query receives nothing (got %d)" % (shape, rounds, got), got == 0)

        # ---- gl_allreduce
        I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
        ivals = [[-(1 << 40) + 3, 7, -5, 11][r % 4] for r in range(world)]
        check("%s: allreduce int64 sum" % shape, mm.allreduce(ivals[rank], op=0) == sum(ivals))
        mins = [[I64_MIN, -5, 9][r % 3] for r in range(world)]
        check("%s: allreduce int64 min" % shape, mm.allreduce(mins[rank], op=1) == I64_MIN)
        maxs = [-5] * (world - 1) + [I64_MAX]
        check("%s: allreduce int64 max" % shape, mm.allreduce(maxs[rank], op=2) == I64_MAX)
        negs = [-3 - r for r in range(world)]
        check("%s: allreduce int64 max of negatives" % shape, mm.allreduce(negs[rank], op=2) == -3)

        def fold(vs, op):
            c = vs[0]
            for x in vs[1:]:
                c = c + x if op == 0 else (c if c < x else x) if op == 1 else (c if c > x else x)
            return c

        bits = lambda d: struct.pack("<d", d)
        dcases = [([1e16, 1.0, 1.0], 0), ([0.1, 0.2, 0.3], 0), ([-0.0, -0.0, -0.0], 0),
                  ([math.inf, -math.inf, 3.5], 1), ([3.5, math.inf, -math.inf], 2),
                  ([0.0, -0.0, 0.0], 1), ([-0.0, 0.0, -0.0], 1), ([0.0, -0.0, 0.0], 2), ([-0.0, 0.0, -0.0], 2)]
        for vs, op in dcases:
            vs = vs[:world]
            got = mm.allreduce(vs[rank], is_double=True, op=op)
            check("%s: allreduce double op %d of %r = left fold in fid order" % (shape, op, vs),
                  bits(got) == bits(fold(vs, op)))
            check("%s: allreduce double op %d of %r bitwise equal on every rank" % (shape, op, vs),
                  len(set(all_obj(bits(got)))) == 1)

        # ---- landing-slot overflow on every rank at once (last: the manager is torn down after it)
        cap = vw.capacity_bytes
        claim = np.full(world, cap + 16, dtype=np.uint32)
        claim[rank] = 0
        mm.start()
        mm.start_round()
        capi.check(L.gl_dev_h2d(C.c_void_p(mm.view().send_bytes), claim.ctypes.data_as(C.c_void_p), C.c_size_t(4 * world)))
        st = L.gl_mm_finish_round(mm.h, None)
        check("%s: overflow returns GL_ERR_COMM (got %d)" % (shape, st), st == -5)
        check("%s: overflow message" % shape, b"landing slot overflow" in L.gl_last_error())
        mm.close()
        dist.barrier()
        comm.close()
        frag.close()
        nbad = sum(all_obj(len(mine) - nfail0))
        if rank == 0:
            print("[face2] shape %-18s fnum=%d %s" % (shape, world, "OK" if nbad == 0 else "FAILED"), flush=True)
    for f in all_obj(mine):
        failures.extend(f)


if __name__ == "__main__":
    main()
