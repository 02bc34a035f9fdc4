#!/usr/bin/env python
"""Times k-clique counting (csrc/app_kclique.cu) on one GPU and prints one JSON
line.  MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

On R-MAT scale --scale (edge factor 16, seed 1, one fragment, self loops and
multi-edges kept in the fragment; the count is on the simple graph underneath)
every k of --k is warmed up, then timed over --steps queries with the L2 flushed
(256 MB memset) in front of each.  Per k: the count, the median device
query_ms, the DAG entries the intersections iterated, the largest candidate set
s and the edges each tier took (warp <= 32, CTA bitmap <= 1024, CTA list
> 1024).  Before timing, the GPU counts at --check-scale are compared with the
CPU oracle (oracle/kclique_oracle.py): "parity".  The card's name and power
limit are read (query only) in the same run.

--impl reference adds the reference's own CPU app (oracle/_ref/ref_kclique_driver,
built by __graft_entry__.build()) on the same R-MAT input at --ref-scale,
simplified inside the driver, next to the GPU time at that scale.

The default, k = 3 at scale 24, shows the largest candidate set R-MAT reaches; on an H100 one query
at k = 4 and scale 24 takes over a minute, so k = 4 and 5 are run at smaller scales (--scale 16 --k 3,4,5).

usage: bench_kclique.py [--scale 24] [--k 3] [--check-scale 12] [--steps 5] [--warmup 2]
                        [--impl gpu|reference] [--ref-scale 16] [--ref-repeat 1]"""
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


def parity(pkg, scale, ks):
    from oracle import kclique_oracle as KO
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    frag = pkg.Fragment.rmat(scale, 16, seed=1)
    ok = {}
    for k in ks:
        app = pkg.App("kclique", frag, k=k)
        app.query()
        ok["k%d" % k] = app.result() == KO.count(1 << scale, src, dst, k)
        app.close()
    frag.close()
    return ok


def time_gpu(pkg, scale, ks, steps, warmup):
    import torch
    frag = pkg.Fragment.rmat(scale, 16, seed=1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    out = {}
    for k in ks:
        app = pkg.App("kclique", frag, k=k)
        ms = []
        for it in range(warmup + steps):
            flush.zero_()
            torch.cuda.synchronize()
            st = app.query()
            if it >= warmup:
                ms.append(st.query_ms)
        count = app.result()
        out["k%d" % k] = {
            "count": count, "query_ms": float(np.median(ms)), "query_ms_all": [round(x, 3) for x in ms],
            "entries_scanned": int(st.entries_scanned), "oriented_edges": int(st.frontier_vertices),
            "max_candidate_set": int(st.step_frontier[0]),
            "tier_items": {"warp": int(st.step_frontier[1]), "cta_bitmap": int(st.step_frontier[2]),
                           "cta_list": int(st.step_frontier[3])}}
        app.close()
        print("[bench_kclique] scale %d k=%d: %r" % (scale, k, out["k%d" % k]), file=sys.stderr, flush=True)
    csr = int(frag.oe_num)
    frag.close()
    return out, csr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--k", default="3")
    ap.add_argument("--check-scale", type=int, default=12)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-scale", type=int, default=16)
    ap.add_argument("--ref-repeat", type=int, default=1)
    args = ap.parse_args()
    ks = [int(x) for x in args.k.split(",") if x]
    pkg = importlib.import_module("libgrape-lite_b200")
    checks = parity(pkg, args.check_scale, ks)
    apps, csr = time_gpu(pkg, args.scale, ks, args.steps, args.warmup)
    line = {"bench": "kclique", "graph": "R-MAT scale %d, edge factor 16, seed 1, one fragment" % args.scale,
            "vertices": 1 << args.scale, "csr_entries": csr, "steps": args.steps, "warmup": args.warmup,
            "l2": "flushed (256 MB memset) before every query", "apps": apps, "card": card(),
            "check_scale": args.check_scale, "parity_detail": checks, "parity": all(checks.values())}
    if args.impl == "reference":
        from oracle import refkclique
        if not refkclique.available():
            raise SystemExit("oracle/_ref/ref_kclique_driver is not built (needs the reference sources at build time)")
        gpu_at = apps if args.ref_scale == args.scale else time_gpu(pkg, args.ref_scale, ks, args.steps, args.warmup)[0]
        ref = {}
        for k in ks:
            info = refkclique.run_rmat(args.ref_scale, k, repeat=args.ref_repeat)
            ms = [float(x) for x in info["query_ms"]]
            ref["k%d" % k] = {"count": int(info["clique_num"]), "query_ms": float(np.median(ms)),
                              "query_ms_all": [round(x, 1) for x in ms], "threads": info["threads"],
                              "hardware_concurrency": info["hardware_concurrency"],
                              "gpu_query_ms": gpu_at["k%d" % k]["query_ms"],
                              "same_count": int(info["clique_num"]) == gpu_at["k%d" % k]["count"]}
        line["reference_scale"] = args.ref_scale
        line["reference"] = ref
        line["reference_note"] = ("the reference's unmodified CPU app (ParallelWorkerOpt, one fragment), Query() of "
                                  "a fresh worker per query on the simplified R-MAT input, generated inside the driver")
        line["parity"] = line["parity"] and all(r["same_count"] for r in ref.values())
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
