#!/usr/bin/env python
"""Times PageRank on a vertex-cut fragment (csrc/app_pagerank_vc.cu) on one GPU and prints one JSON
line.  MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

On the R-MAT graph of scale --scale (edge factor 16, seed 1, built on the device by
VcFragment.rmat: one fragment, every generated edge once) the app runs --rounds rounds; it is warmed
up, then timed over --steps queries with the L2 flushed (256 MB memset) in front of each.  Reported:
the median device query_ms, ms per round (query_ms / rounds), the local CSR entries a round reads
and the algorithmic bytes of a round: per entry a 4-byte column id and an 8-byte gather of curr, per
local vertex its 8-byte row pointer and 8-byte partial sum.  GL_APP_PAGERANK (pull) runs on the
edge-cut fragment of the same edges (Fragment.rmat, which stores each edge in both rows) with the
same rounds, timed the same way.  Before timing, both apps' values at --check-scale are compared
with each other and with the scipy oracle (oracle/pagerank_vc_oracle.py) to 1e-9 relative: "parity".
The card's name and power limit are read (query only) in the same run.  One more query, untimed, runs
under torch.profiler and reports the device time of each kernel summed over the query ("kernel_ms"):
k_vc_pull (rows of up to 4096 entries), k_vc_chunks + k_vc_long (longer rows), k_vc_master and the rest.

--impl reference adds, in the same line, the reference's own CPU app PageRankVC
(oracle/_ref/ref_pagerank_vc_driver, built by __graft_entry__.build()) on the same R-MAT input at
--ref-scale (generated inside the driver, one fragment, all host threads): Query() of a fresh worker.

usage: bench_pagerank_vc.py [--scale 24] [--check-scale 16] [--rounds 10] [--steps 3] [--warmup 1]
                            [--impl gpu|reference] [--ref-scale 22]"""
import argparse
import importlib
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_core import card  # noqa: E402


def parity(pkg, scale, rounds):
    from oracle import pagerank_vc_oracle as V
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    n = 1 << scale
    frag = pkg.VcFragment.rmat(scale, 16, seed=1)
    app = pkg.App("pagerank_vc", frag, pr_delta=0.85, max_round=rounds)
    app.query()
    vc = app.result()
    app.close()
    frag.close()
    ec = pkg.Fragment.rmat(scale, 16, seed=1)
    app = pkg.App("pagerank", ec, pr_pull=1, pr_delta=0.85, max_round=rounds)
    app.query()
    pr = app.result()
    app.close()
    ec.close()
    want = V.pagerank_vc(n, src, dst, 0.85, rounds)
    return bool(np.allclose(vc, want, rtol=1e-9, atol=0) and np.allclose(vc, pr, rtol=1e-9, atol=0))


def timed(app, flush, steps, warmup):
    import torch
    rows = []
    for it in range(warmup + steps):
        flush.zero_()
        torch.cuda.synchronize()
        st = app.query()
        if it >= warmup:
            rows.append((st.query_ms, st.entries_scanned, st.kernel_launches))
    return rows


def profile_kernels(app):
    """Device time per kernel name (ms, summed) over one query under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        app.query()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"\b(k_\w+)", e.name)
            name = m.group(1) if m else e.name.strip()
            out[name] = out.get(name, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--check-scale", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-scale", type=int, default=22)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    ok = parity(pkg, args.check_scale, args.rounds)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    frag = pkg.VcFragment.rmat(args.scale, 16, seed=1)
    info = frag.info
    app = pkg.App("pagerank_vc", frag, pr_delta=0.85, max_round=args.rounds)
    rows = timed(app, flush, args.steps, args.warmup)
    vc = app.result()
    kernel_ms = profile_kernels(app)
    app.close()
    frag.close()
    ms = [r[0] for r in rows]
    med = float(np.median(ms))
    entries, nl = int(info["entries"]), int(info["local_vnum"])
    round_bytes = entries * (4 + 8) + nl * (8 + 8)
    gpu = {"query_ms": med, "query_ms_all": [round(x, 3) for x in ms], "ms_per_round": med / args.rounds,
           "entries_per_round": entries, "bytes_per_round": round_bytes,
           "algorithmic_GBps": round_bytes * args.rounds / (med * 1e-3) / 1e9,
           "kernel_launches": int(rows[-1][2]), "sum": float(vc.sum()), "kernel_ms": kernel_ms}
    ec = pkg.Fragment.rmat(args.scale, 16, seed=1)
    app = pkg.App("pagerank", ec, pr_pull=1, pr_delta=0.85, max_round=args.rounds)
    prow = timed(app, flush, args.steps, args.warmup)
    app.close()
    ec.close()
    pms = float(np.median([r[0] for r in prow]))
    line = {"bench": "pagerank_vc",
            "graph": "R-MAT scale %d, edge factor 16, seed 1, one vertex-cut fragment" % args.scale,
            "vertices": 1 << args.scale, "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
            "l2": "flushed (256 MB memset) before every query", "gpu": gpu,
            "pagerank_pull": {"query_ms": pms, "query_ms_all": [round(r[0], 3) for r in prow],
                              "ms_per_round": pms / args.rounds},
            "card": card(), "check_scale": args.check_scale, "parity": ok}
    if args.impl == "reference":
        from oracle import refprvc
        if not refprvc.available():
            raise SystemExit("oracle/_ref/ref_pagerank_vc_driver is not built (needs the reference sources at build time)")
        info = refprvc.run_rmat(args.ref_scale, 16, 1, 0.85, args.rounds, np_ranks=1)
        line["reference"] = {"scale": args.ref_scale, "query_ms": float(info["query_ms"][-1]),
                             "threads": info["threads"], "load_s": info["load_s"],
                             "hardware_concurrency": info["hardware_concurrency"]}
    print(json.dumps(line), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
