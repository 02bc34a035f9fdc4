"""Directed graphs on a fragment group: launched by torchrun (one rank per
fragment; GL_ONE_DEVICE=1 puts every rank's fragment on cuda:0).  Every case of
tests/directed_cases.py runs BFS, SSSP, WCC and PageRank in the configurations
listed there, each followed by a second query on the same app; rank 0 compares
the concatenated inner results with the whole-graph oracle on the same directed
edge list and prints one OK / MISMATCH line per (case, configuration).  Also:
p2p-31 against the reference's directed golden files, the geometry of the
fragments actually built, pull levels on the fused and the stepwise BFS path,
the f64 SSSP and f32-contribution PageRank paths on an undirected split, and the
refusal of the undirected-only apps on a directed group."""
import importlib
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

INT64_MAX = np.iinfo(np.int64).max
F64_MAX = np.finfo(np.float64).max


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
    from tests import directed_cases as D
    failures = []

    def all_obj(x):
        out = [None] * world
        dist.all_gather_object(out, x)
        return out

    def gather(arr):
        return np.concatenate(all_obj(arr))

    def report(case, what, ok):
        if rank == 0:
            print("[mgpu-dir] %-18s %-34s fnum=%d %s" % (case, what, world, "OK" if ok else "MISMATCH"), flush=True)
            if not ok:
                failures.append("%s:%s" % (case, what))

    def first_diff(got, want):
        bad = np.flatnonzero(~np.isclose(got, want, rtol=1e-6, atol=0) if got.dtype.kind == "f" else got != want)
        if rank == 0 and len(bad):
            print("[mgpu-dir]   %d differ, first %s: got %s want %s" % (len(bad), bad[:5], got[bad[:5]], want[bad[:5]]),
                  flush=True)

    def run_twice(kind, frag, comm, vm=None, **cfg):
        """(result of query 1, result of query 2, any pull level in query 1) gathered over the group."""
        app = pkg.App(kind, frag, comm, **cfg)
        if vm is not None:
            app.set_vertex_map(vm)
        st = app.query()
        pulled = any(st.step_mode[i] == 1 for i in range(min(st.n_steps, pkg.GL_MAX_STEP_STATS)))
        r1 = app.result()
        app.query()
        r2 = app.result()
        app.close()
        return gather(r1), gather(r2), any(all_obj(pulled))

    def rel_close(got, want, tol=1e-6):
        return got.shape == want.shape and bool(np.all(np.abs(got - want) <= tol * np.abs(want)))

    pulled = {"fused": False, "step": False}
    for name, (_, real) in D.CASES.items():
        t0 = time.time()
        n, src, dst, w = D.build(name)
        oids = D.p2p31_oids() if name == "p2p31" else None
        chunk = D.chunk_of(n, world)

        def to_oid(v):
            if oids is None:
                return int(v)
            return int(oids[v]) if v < n else int(oids[-1]) + 7
        s_e, d_e = (src, dst) if oids is None else (oids[src], oids[dst])
        frag = pkg.Fragment.from_edges(n, s_e, d_e, w, directed=True, oids=oids, fid=rank, fnum=world)
        comm = gdist.make_comm(rank, world, frag.ivnum)
        g = pyoracle.Graph(n, s_e, d_e, w, directed=True, oids=oids) if rank == 0 else None

        # the geometry the case is listed for, on the fragments the library built
        geo = D.geometry(n, src, dst, world)[rank]
        ovgid = frag.ovgid()
        off = frag.fid_offset
        glob_outer = (ovgid >> off).astype(np.int64) * chunk + (ovgid & ((1 << off) - 1)).astype(np.int64)
        _, col0, _ = frag.csr(0)
        _, col1, _ = frag.csr(1)
        oe_cols = np.unique(col0[col0 >= frag.ivnum]).astype(np.int64) - frag.ivnum
        ie_cols = np.unique(col1[col1 >= frag.ivnum]).astype(np.int64) - frag.ivnum
        mine = (frag.ovnum == len(geo["outer"]) and np.array_equal(glob_outer, geo["outer"])
                and np.array_equal(glob_outer[np.setdiff1d(ie_cols, oe_cols)], geo["ie_only"]))
        report(name, "geometry of the built fragments", all(all_obj(bool(mine))))

        srcs = D.sources(n, src, dst, world)
        for cname, cfg in D.BFS_CONFIGS:
            for sname in D.BFS_SOURCES + (D.BFS_SOURCES_FUSED if cname == "fused" else ()):
                v = srcs[sname]
                got, got2, pl = run_twice("bfs", frag, comm, source_oid=to_oid(v), **cfg)
                if cname in pulled:
                    pulled[cname] |= pl
                if rank == 0:
                    want = g.bfs(v)[0] if v < n else np.full(n, INT64_MAX, dtype=np.int64)
                    ok = np.array_equal(got, want) and np.array_equal(got2, got)
                    if not ok:
                        first_diff(got, want)
                report(name, "bfs %s from %s" % (cname, sname), rank != 0 or ok)

        # SSSP: f32 edge data on `frag`, f64 edge data on a second build of the same split
        frag64 = comm64 = None
        for f64, prio, eb in (D.SSSP_REAL if real else D.SSSP_INT):
            if eb == 8 and frag64 is None:
                frag64 = pkg.Fragment.from_edges(n, s_e, d_e, w, directed=True, oids=oids, fid=rank, fnum=world,
                                                 w_dtype=np.float64)
                comm64 = gdist.make_comm(rank, world, frag64.ivnum)
            for sname in D.SSSP_SOURCES:
                v = srcs[sname]
                fr, cm = (frag64, comm64) if eb == 8 else (frag, comm)
                got, got2, _ = run_twice("sssp", fr, cm, source_oid=to_oid(v), sssp_f64=f64, sssp_prio=prio)
                if rank == 0:
                    want = g.sssp(v)[0]
                    if real and not f64:
                        fin = want < F64_MAX
                        ok = (np.array_equal(got >= F64_MAX, ~fin) and rel_close(got[fin], want[fin]))
                    else:
                        ok = np.array_equal(got, want)
                    ok = ok and np.array_equal(got2, got)
                    if not ok:
                        first_diff(got, want)
                report(name, "sssp f64=%d prio=%g edata=%dB from %s" % (f64, prio, eb, sname), rank != 0 or ok)
        if frag64 is not None:
            comm64.close()
            frag64.close()

        # WCC: minimum-id labels (oids through the device vertex map when the case has its own oids)
        vm = None if oids is None else pkg.VertexMap([oids[f * chunk:(f + 1) * chunk] for f in range(world)])
        for kind in D.WCC_KINDS:
            got, got2, _ = run_twice(kind, frag, comm, vm=vm)
            if rank == 0:
                want = g.wcc()[0].astype(np.int64)
                if oids is not None:
                    want = oids[want]
                ok = np.array_equal(got, want) and np.array_equal(got2, got)
                if not ok:
                    first_diff(got, want)
            report(name, kind, rank != 0 or ok)
        if vm is not None:
            vm.close()

        # PageRank: push along oe, the dangling rule of the directed app (pr_pull falls back to push).
        # The push adds with f64 atomics, so two queries agree within the tolerance, not bit for bit.
        for pull, delta, rounds in D.PR_CONFIGS:
            got, got2, _ = run_twice("pagerank", frag, comm, pr_pull=pull, pr_delta=delta, max_round=rounds)
            if rank == 0:
                want = g.pagerank(delta, rounds, 2) if rounds else np.full(n, 1.0 / n)
                ok = rel_close(got, want) and rel_close(got2, want)
                if not ok:
                    first_diff(got, want)
            report(name, "pagerank pull=%d delta=%g rounds=%d" % (pull, delta, rounds), rank != 0 or ok)

        if name == "p2p31":
            run_p2p_golden(pkg, frag, comm, rank, all_obj, report)
        comm.close()
        frag.close()
        if rank == 0:
            print("[mgpu-dir] %s done in %.1f s" % (name, time.time() - t0), flush=True)

    report("all cases", "pull level on the fused path", pulled["fused"])
    report("all cases", "pull level on the stepwise path", pulled["step"])
    run_undirected_extras(pkg, gdist, pyoracle, rank, world, run_twice, report, rel_close)
    run_refusals(pkg, gdist, rank, world, all_obj, report, D)

    flag = torch.tensor([len(failures)], device=dev)
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


def run_p2p_golden(pkg, frag, comm, rank, all_obj, report):
    """p2p-31 loaded directed with its own oids, results through result_oids, against the
    reference's golden files (misc/app_tests.sh rules: text for BFS and SSSP, eps_check for
    PageRank, wcc_check's partition rule for WCC)."""
    from tests import directed_cases as D
    from tests import golden_io as G

    def run(kind, **cfg):
        app = pkg.App(kind, frag, comm, **cfg)
        app.query()
        r = (app.result_oids(), app.result())
        app.close()
        parts = all_obj(r)
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    o, depth = run("bfs", source_oid=D.P2P_SOURCE_OID)
    if rank == 0:
        ok = G.render(o, [str(int(d)) for d in depth]) == G.golden_lines("p2p-31-BFS-directed")
    report("p2p31", "golden p2p-31-BFS-directed", rank != 0 or ok)
    for f64 in (0, 1):
        o, dd = run("sssp", source_oid=D.P2P_SOURCE_OID, sssp_f64=f64)
        if rank == 0:
            text = G.render(o, ["infinity" if d == F64_MAX else G.fmt_sci(d) for d in dd])
            ok = text == G.golden_lines("p2p-31-SSSP-directed")
        report("p2p31", "golden p2p-31-SSSP-directed f64=%d" % f64, rank != 0 or ok)
    o, pr = run("pagerank", pr_delta=0.85, max_round=10)
    if rank == 0:
        gp = G.golden_pairs("p2p-31-PR-directed")
        want = np.array([float(v) for _, v in gp])
        ok = (np.array_equal(o, [k for k, _ in gp]) and G.eps_check(pr, want, 1e-4)
              and bool(np.max(np.abs(pr - want) / want) < 1e-6))
    report("p2p31", "golden p2p-31-PR-directed", rank != 0 or ok)
    o, lab = run("wcc")
    if rank == 0:
        gp = G.golden_pairs("p2p-31-WCC")
        ok = np.array_equal(o, [k for k, _ in gp]) and G.same_partition(lab, [int(v) for _, v in gp])
    report("p2p31", "golden p2p-31-WCC (partition)", rank != 0 or ok)


def run_undirected_extras(pkg, gdist, pyoracle, rank, world, run_twice, report, rel_close):
    """Undirected R-MAT 12 with integer weights as f64 edge data: SSSP in f64 with the priority
    threshold, and PageRank gathering f32 contributions (the 4-byte dense mirror sync of the
    contributions), with and without the shared-memory hub table."""
    src, dst, w = pkg.rmat_edges_host(12, 16, 29, 1)
    n = 1 << 12
    w = w.astype(np.float64)
    frag = pkg.Fragment.from_edges(n, src, dst, w, fid=rank, fnum=world, w_dtype=np.float64)
    comm = gdist.make_comm(rank, world, frag.ivnum)
    g = pyoracle.Graph(n, src, dst, w) if rank == 0 else None
    source = int(np.argmax(np.bincount(np.concatenate([src, dst]), minlength=n)))
    got, got2, _ = run_twice("sssp", frag, comm, source_oid=source, sssp_f64=1, sssp_prio=0.5)
    ok = rank != 0 or (np.array_equal(got, g.sssp(source)[0]) and np.array_equal(got2, got))
    report("undirected_rmat12", "sssp f64=1 prio=0.5 edata=8B", ok)
    for what, res in (("pr_pull32", {5: 1}), ("pr_pull32_nohub", {4: 1, 5: 1})):
        got, got2, _ = run_twice("pagerank", frag, comm, pr_pull=1, pr_delta=0.85, max_round=10, reserved=res)
        if rank == 0:
            want = g.pagerank(0.85, 10, 1)
            ok = rel_close(got, want) and rel_close(got2, want)
            if not ok:
                print("[mgpu-dir]   max relative error %.3g / %.3g" % (np.max(np.abs(got - want) / want),
                                                                   np.max(np.abs(got2 - want) / want)), flush=True)
        report("undirected_rmat12", what, rank != 0 or ok)
    comm.close()
    frag.close()


def run_refusals(pkg, gdist, rank, world, all_obj, report, D):
    """The undirected-only apps refuse a directed fragment group on every rank, without a hang."""
    n, src, dst, w = D.build("union")
    frag = pkg.Fragment.from_edges(n, src, dst, w, directed=True, fid=rank, fnum=world)
    comm = gdist.make_comm(rank, world, frag.ivnum)
    for kind, cfg in (("core_decomposition", {}), ("kcore", {"k": 2}), ("kclique", {"k": 3})):
        try:
            pkg.App(kind, frag, comm, **cfg).close()
            refused = False
        except pkg.GrapeError:
            refused = True
        report("directed union", "%s refused" % kind, all(all_obj(refused)))
    comm.close()
    frag.close()


if __name__ == "__main__":
    main()
