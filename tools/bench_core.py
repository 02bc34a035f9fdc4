#!/usr/bin/env python
"""Times core decomposition and k-core (csrc/app_core.cu) on one GPU and prints
one JSON line.  MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

On R-MAT scale --scale (edge factor 16, seed 1, one fragment) every app is
warmed up, then timed over --steps queries with the L2 flushed (256 MB memset)
in front of each, as bench.py does.  Per app: the median device query_ms, CSR
entries scanned per second, sub-rounds and kernel launches per query.  Before
timing, the GPU results at --check-scale are compared bit for bit with the CPU
oracle (oracle/core_oracle.py): "parity".  The card's name and power limit are
read (query only) in the same run.

--impl reference adds, in the same line, the reference's own CPU apps
(oracle/_ref/ref_core_driver, built by __graft_entry__.build()) timed with
oracle/refcore.run_rmat on the same R-MAT input, generated inside the driver:
Query() of a fresh worker per query, all host threads, --ref-repeat queries.
GL_KTIME=1 in the environment also prints, per GPU query, the device time the
fused kernel spent in level steps and in sub-rounds (stderr).

usage: bench_core.py [--scale 24] [--check-scale 20] [--steps 5] [--warmup 2] [--k 16,64]
                     [--impl gpu|reference] [--ref-repeat 1]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                           text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(q[0])
        info["sm_max_mhz"] = float(q[1])
    except Exception:
        pass
    return info


def configs(ks):
    return [("core_decomposition", {})] + [("kcore", {"k": k}) for k in ks]


def parity(pkg, scale, ks):
    from oracle import core_oracle as CO
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    n = 1 << scale
    frag = pkg.Fragment.rmat(scale, 16, seed=1)
    ok = {}
    for kind, cfg in configs(ks):
        app = pkg.App(kind, frag, **cfg)
        app.query()
        got = app.result()
        app.close()
        want = CO.core_decomposition(n, src, dst)[0] if kind == "core_decomposition" else CO.kcore(n, src, dst, cfg["k"])
        ok["%s%s" % (kind, "" if not cfg else "_k%d" % cfg["k"])] = bool(np.array_equal(got, want))
    frag.close()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--check-scale", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--k", default="16,64")
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-repeat", type=int, default=1)
    args = ap.parse_args()
    ks = [int(x) for x in args.k.split(",") if x]
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    checks = parity(pkg, args.check_scale, ks)
    frag = pkg.Fragment.rmat(args.scale, 16, seed=1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    apps = {}
    for kind, cfg in configs(ks):
        app = pkg.App(kind, frag, **cfg)
        rows = []
        for it in range(args.warmup + args.steps):
            flush.zero_()
            torch.cuda.synchronize()
            st = app.query()
            if it >= args.warmup:
                rows.append((st.query_ms, st.entries_scanned, st.supersteps, st.kernel_launches, st.frontier_vertices))
        app.close()
        ms = [r[0] for r in rows]
        med = float(np.median(ms))
        apps["%s%s" % (kind, "" if not cfg else "_k%d" % cfg["k"])] = {
            "query_ms": med, "query_ms_all": [round(x, 3) for x in ms],
            "entries_scanned": int(rows[-1][1]), "entries_per_s": rows[-1][1] / (med * 1e-3),
            "sub_rounds": int(rows[-1][2]), "kernel_launches": int(rows[-1][3]), "vertices_peeled": int(rows[-1][4])}
    line = {"bench": "core", "graph": "R-MAT scale %d, edge factor 16, seed 1, one fragment" % args.scale,
            "vertices": 1 << args.scale, "csr_entries": int(frag.oe_num), "steps": args.steps, "warmup": args.warmup,
            "l2": "flushed (256 MB memset) before every query", "apps": apps, "card": card(),
            "check_scale": args.check_scale, "parity_detail": checks, "parity": all(checks.values())}
    frag.close()
    if args.impl == "reference":
        from oracle import refcore
        if not refcore.available():
            raise SystemExit("oracle/_ref/ref_core_driver is not built (needs the reference sources at build time)")
        ref = {}
        for kind, cfg in configs(ks):
            info = refcore.run_rmat(kind, args.scale, 16, 1, k=cfg.get("k", 0), repeat=args.ref_repeat)
            ms = [float(x) for x in info["query_ms"]]
            ref["%s%s" % (kind, "" if not cfg else "_k%d" % cfg["k"])] = {
                "query_ms": float(np.median(ms)), "query_ms_all": [round(x, 1) for x in ms], "load_s": info["load_s"],
                "threads": info["threads"], "hardware_concurrency": info["hardware_concurrency"]}
        line["reference"] = ref
        line["reference_note"] = ("the reference's unmodified CPU apps (ParallelWorkerOpt), Query() of a fresh worker "
                                  "per query on the same R-MAT input, generated inside the driver")
        line["speedup_vs_reference"] = {k: ref[k]["query_ms"] / apps[k]["query_ms"] for k in apps}
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
