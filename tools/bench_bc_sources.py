#!/usr/bin/env python
"""Times betweenness centrality over a list of sources (csrc/app_bc_sources.cu) on one GPU against the
single-source app (csrc/app_bc.cu) run once per source, and prints one JSON line.  MEASUREMENT
INFRASTRUCTURE (needs a GPU; writes nothing).

For each R-MAT scale of --scales (undirected, edge factor 16, seed 1, one fragment) and each list length
of --sources, the list is the maximum-degree vertex followed by a seeded sample (numpy default_rng(scale),
repeats allowed).  GL_APP_BC_SOURCES runs the whole list per query: warmed up, then --steps queries with
the L2 flushed (256 MB memset) in front of each; reported: the median device query_ms and ms per source.
GL_APP_BC runs on the first 32 sources of the same list in the same process, one query per source with
the L2 flushed in front of each; reported: the median ms per source.  Before timing, the result at
--check-scale (64 sources) is compared bit for bit with the order-exact CPU oracle
(oracle/bc_sources_oracle.py): "parity".  The card's name and power limit are read (query only) in the
same run.

--impl reference adds the reference's own CPU app (oracle/_ref/ref_bc_driver) timed per source with
oracle/refbc.run_rmat at --ref-scale on the first --ref-sources sources of that scale's list.

usage: bench_bc_sources.py [--scales 22,24] [--sources 64,256] [--check-scale 16] [--steps 3]
                           [--warmup 1] [--impl gpu|reference] [--ref-scale 20] [--ref-sources 3]"""
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


def source_list(frag, scale, k):
    n = 1 << scale
    hub = int(frag.max_degree_vertex()[0])   # lid == oid on the R-MAT builder
    return [hub] + np.random.default_rng(scale).integers(0, n, size=k - 1).tolist()


def parity(pkg, scale):
    from oracle import bc_sources_oracle as BSO
    frag = pkg.Fragment.rmat(scale, 16, seed=1)
    sources = source_list(frag, scale, 64)
    app = pkg.App("bc_sources", frag, sources=sources)
    app.query()
    got = app.result()
    app.close()
    rp, col, _ = frag.csr(0)
    want, _ = BSO.bc_sources(frag.ivnum, rp, col, sources)
    frag.close()
    return got.tobytes() == want.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24")
    ap.add_argument("--sources", default="64,256")
    ap.add_argument("--check-scale", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-scale", type=int, default=20)
    ap.add_argument("--ref-sources", type=int, default=3)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    ok = parity(pkg, args.check_scale)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    runs = []
    for scale in [int(x) for x in args.scales.split(",")]:
        frag = pkg.Fragment.rmat(scale, 16, seed=1)
        kmax = max(int(x) for x in args.sources.split(","))
        full = source_list(frag, scale, kmax)
        # the single-source app on the first 32 sources
        app = pkg.App("bc", frag, source_oid=full[0])
        app.query()
        app.close()
        one = []
        for s in full[:32]:
            app = pkg.App("bc", frag, source_oid=int(s))
            flush.zero_()
            torch.cuda.synchronize()
            one.append(app.query().query_ms)
            app.close()
        bc_ms = float(np.median(one))
        for k in [int(x) for x in args.sources.split(",")]:
            app = pkg.App("bc_sources", frag, sources=full[:k])
            ms = []
            for it in range(args.warmup + args.steps):
                flush.zero_()
                torch.cuda.synchronize()
                st = app.query()
                if it >= args.warmup:
                    ms.append(st.query_ms)
            med = float(np.median(ms))
            runs.append({"scale": scale, "sources": k, "csr_entries": int(frag.oe_num), "query_ms": med,
                         "query_ms_all": [round(x, 2) for x in ms], "ms_per_source": med / k,
                         "batches": int(st.supersteps), "entries_scanned": int(st.entries_scanned),
                         "bc_ms_per_source": bc_ms, "bc_ms_all": [round(x, 3) for x in one],
                         "speedup_per_source_vs_bc": bc_ms / (med / k)})
            app.close()
        frag.close()
    line = {"bench": "bc_sources", "graph": "R-MAT, edge factor 16, seed 1, undirected, one fragment",
            "steps": args.steps, "warmup": args.warmup, "l2": "flushed (256 MB memset) before every query",
            "runs": runs, "card": card(), "check_scale": args.check_scale, "parity": ok}
    if args.impl == "reference":
        from oracle import refbc
        if not refbc.available():
            raise SystemExit("oracle/_ref/ref_bc_driver is not built (needs the reference sources at build time)")
        frag = pkg.Fragment.rmat(args.ref_scale, 16, seed=1)
        lst = source_list(frag, args.ref_scale, args.ref_sources)
        frag.close()
        rms = []
        for s in lst:
            info = refbc.run_rmat(args.ref_scale, 16, 1, source=int(s), repeat=1)
            rms.append(float(np.median([float(x) for x in info["query_ms"]])))
        line["reference"] = {"scale": args.ref_scale, "sources": lst, "ms_per_source": float(np.mean(rms)),
                             "query_ms_all": [round(x, 1) for x in rms], "threads": info["threads"]}
    print(json.dumps(line), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
