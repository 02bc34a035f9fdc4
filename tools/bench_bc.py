#!/usr/bin/env python
"""Times single-source betweenness centrality (csrc/app_bc.cu) on one GPU and
prints one JSON line.  MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

On R-MAT scale --scale (edge factor 16, seed 1, one fragment) the app runs from
the maximum-degree vertex (CSR entries, ties to the smallest id, as bench.py's
BFS source): warmed up, then timed over --steps queries with the L2 flushed
(256 MB memset) in front of each, as bench.py does.  Reported: the median device
query_ms, CSR entries read per second, levels, kernel launches per query.
Before timing, the GPU result at --check-scale is compared with the CPU oracle
(oracle/bc_oracle.py, f64 arithmetic): depth and sigma exactly, c within
(L + 1) * 2^-22 relative: "parity".  The card's name and power limit are read
(query only) in the same run.  GL_KTIME=1 in the environment also prints, per
GPU query, the device time of the forward and the backward pass (stderr).

--impl reference adds, in the same line, the reference's own CPU app
(oracle/_ref/ref_bc_driver, built by __graft_entry__.build()) timed with
oracle/refbc.run_rmat on the same R-MAT input and source, generated inside the
driver: Query() of fresh workers per query, all host threads, --ref-repeat
queries.

usage: bench_bc.py [--scale 24] [--check-scale 20] [--steps 3] [--warmup 1]
                   [--impl gpu|reference] [--ref-repeat 1]"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_core import card  # noqa: E402


def max_degree_source(frag):
    return int(frag.max_degree_vertex()[0])   # lid == oid on the R-MAT builder


def parity(pkg, scale):
    from oracle import bc_oracle as BO
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    n = 1 << scale
    frag = pkg.Fragment.rmat(scale, 16, seed=1)
    source = max_degree_source(frag)
    app = pkg.App("bc", frag, source_oid=source)
    app.query()
    got = app.result()
    app.close()
    frag.close()
    c, sigma, depth = BO.bc(n, src, dst, source)
    L = int(depth[depth != BO.INF].max())
    return {"depth": bool(np.array_equal(got["depth"], depth)),
            "path_num": bool(np.array_equal(got["path_num"], sigma)),
            "centrality": bool(np.all(np.abs(got["centrality"] - c) <= (L + 1) * 2.0 ** -22 * np.abs(c.astype(np.float64))))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--check-scale", type=int, default=20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-repeat", type=int, default=1)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    checks = parity(pkg, args.check_scale)
    frag = pkg.Fragment.rmat(args.scale, 16, seed=1)
    source = max_degree_source(frag)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    app = pkg.App("bc", frag, source_oid=source)
    rows = []
    for it in range(args.warmup + args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        st = app.query()
        if it >= args.warmup:
            modes = [st.step_mode[i] for i in range(st.n_steps)]
            rows.append((st.query_ms, st.entries_scanned, st.supersteps, st.kernel_launches, st.frontier_vertices,
                         modes))
    app.close()
    ms = [r[0] for r in rows]
    med = float(np.median(ms))
    gpu = {"query_ms": med, "query_ms_all": [round(x, 3) for x in ms], "entries_scanned": int(rows[-1][1]),
           "entries_per_s": rows[-1][1] / (med * 1e-3), "levels": int(rows[-1][2]) // 2,
           "pull_levels": rows[-1][5].count(1), "kernel_launches": int(rows[-1][3]), "reached": int(rows[-1][4])}
    line = {"bench": "bc", "graph": "R-MAT scale %d, edge factor 16, seed 1, one fragment" % args.scale,
            "source": source, "vertices": 1 << args.scale, "csr_entries": int(frag.oe_num), "steps": args.steps,
            "warmup": args.warmup, "l2": "flushed (256 MB memset) before every query", "gpu": gpu, "card": card(),
            "check_scale": args.check_scale, "parity_detail": checks, "parity": all(checks.values())}
    frag.close()
    if args.impl == "reference":
        from oracle import refbc
        if not refbc.available():
            raise SystemExit("oracle/_ref/ref_bc_driver is not built (needs the reference sources at build time)")
        info = refbc.run_rmat(args.scale, 16, 1, source="maxdeg", repeat=args.ref_repeat)
        assert int(info["source"]) == source, "the driver picked another maximum-degree vertex"
        rms = [float(x) for x in info["query_ms"]]
        line["reference"] = {"query_ms": float(np.median(rms)), "query_ms_all": [round(x, 1) for x in rms],
                             "load_s": info["load_s"], "threads": info["threads"],
                             "hardware_concurrency": info["hardware_concurrency"]}
        line["reference_note"] = ("the reference's unmodified CPU app bc (StagedBCBFS + StagedBC, ParallelWorkerOpt), "
                                  "Query() of fresh workers per query on the same R-MAT input, generated inside the "
                                  "driver")
        line["speedup_vs_reference"] = line["reference"]["query_ms"] / med
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
