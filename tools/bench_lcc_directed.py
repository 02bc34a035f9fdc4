#!/usr/bin/env python
"""Times the directed local clustering coefficient (csrc/app_lcc_directed.cu) on one GPU and prints one
JSON line.  MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

On the directed R-MAT graph of scale --scale (edge factor 16, seed 1, self loops and duplicates kept,
one fragment built with Fragment.from_edges(..., directed=True)) the app is warmed up, then timed over
--steps queries with the L2 flushed (256 MB memset) in front of each, as bench.py does.  Reported: the
median device query_ms (PEval's oriented rows + the weighted triangle count), the oriented entries read
by the count (entries_scanned) per second, kernel launches per query.  Before timing, the GPU result
at --check-scale is compared bit for bit with the CPU oracle (oracle/lcc_directed_oracle.py):
"parity".  The card's name and power limit are read (query only) in the same run.

--impl reference adds, in the same line, the reference's own CPU app LCCDirected<FRAG_T, uint64_t>
(oracle/_ref/ref_lcc_directed_driver, built by __graft_entry__.build()) timed with
oracle/reflccd.run_rmat on the same directed R-MAT input, generated inside the driver: Query() of a
fresh worker per query, all host threads, --ref-repeat queries.

usage: bench_lcc_directed.py [--scale 24] [--check-scale 16] [--steps 3] [--warmup 1]
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


def directed_rmat(pkg, scale):
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    return 1 << scale, src, dst


def parity(pkg, scale):
    from oracle import lcc_directed_oracle as LO
    n, src, dst = directed_rmat(pkg, scale)
    frag = pkg.Fragment.from_edges(n, src, dst, directed=True)
    app = pkg.App("lcc_directed", frag)
    app.query()
    got = app.result()
    app.close()
    frag.close()
    want, _, _ = LO.lcc_directed_fast(n, src, dst)
    return got.tobytes() == want.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--check-scale", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-repeat", type=int, default=1)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    ok = parity(pkg, args.check_scale)
    n, src, dst = directed_rmat(pkg, args.scale)
    frag = pkg.Fragment.from_edges(n, src, dst, directed=True)
    del src, dst
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    app = pkg.App("lcc_directed", frag)
    rows = []
    for it in range(args.warmup + args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        st = app.query()
        if it >= args.warmup:
            rows.append((st.query_ms, st.entries_scanned, st.kernel_launches, [st.step_ms[i] for i in range(st.n_steps)]))
    out = app.result()
    app.close()
    ms = [r[0] for r in rows]
    med = float(np.median(ms))
    gpu = {"query_ms": med, "query_ms_all": [round(x, 3) for x in ms], "step_ms": [round(x, 3) for x in rows[-1][3]],
           "entries_scanned": int(rows[-1][1]), "entries_per_s": rows[-1][1] / (med * 1e-3),
           "kernel_launches": int(rows[-1][2]), "mean_lcc": float(out.mean())}
    line = {"bench": "lcc_directed",
            "graph": "directed R-MAT scale %d, edge factor 16, seed 1, one fragment" % args.scale,
            "vertices": n, "oe_entries": int(frag.oe_num), "ie_entries": int(frag.ie_num), "steps": args.steps,
            "warmup": args.warmup, "l2": "flushed (256 MB memset) before every query", "gpu": gpu, "card": card(),
            "check_scale": args.check_scale, "parity": ok}
    frag.close()
    if args.impl == "reference":
        from oracle import reflccd
        if not reflccd.available():
            raise SystemExit("oracle/_ref/ref_lcc_directed_driver is not built (needs the reference sources at build time)")
        info = reflccd.run_rmat(args.scale, 16, 1, repeat=args.ref_repeat)
        rms = [float(x) for x in info["query_ms"]]
        line["reference"] = {"query_ms": float(np.median(rms)), "query_ms_all": [round(x, 1) for x in rms],
                             "load_s": info["load_s"], "threads": info["threads"],
                             "hardware_concurrency": info["hardware_concurrency"]}
        line["reference_note"] = ("the reference's unmodified CPU app LCCDirected<FRAG_T, uint64_t> "
                                  "(ParallelWorkerOpt), Query() of a fresh worker per query on the same directed "
                                  "R-MAT input, generated inside the driver")
        line["speedup_vs_reference"] = line["reference"]["query_ms"] / med
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
