#!/usr/bin/env python
"""Times directed CDLP (csrc/app_cdlp_directed.cu) on one GPU and prints one JSON line.
MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

For every scale of --scales, on the directed R-MAT graph of that scale (edge factor 16, seed 1, self
loops and duplicates kept, one fragment built with Fragment.from_edges(..., directed=True)) the app runs
--rounds rounds: it is warmed up, then timed over --steps queries with the L2 flushed (256 MB memset)
in front of each, as bench.py does.  Reported: the median device query_ms, the in + out entries the
rounds read (entries_scanned) per second, kernel launches per query.  In the same line GL_APP_CDLP runs
the same way on the undirected fragment of the same edges, whose rows hold the same entries, and the
ratio of the two medians is given.  Before timing, the GPU result at --check-scale is compared with
the CPU oracle (tests/cdlp_directed_cases.py: the undirected CDLP of the same edges): "parity".  The
card's name and power limit are read (query only) in the same run.

--impl reference adds, per scale, the reference's own GPU CDLP with --directed 1 (oracle/_ref/ref_gpu_driver,
the reference's grape/cuda compiled for sm_90a, built by __graft_entry__.build()) on the same R-MAT input,
generated inside the driver (--rmat SCALE,16,1,0): the host wall time of Query() per --lb mode, the
first of --ref-repeat repetitions taken as warm-up, as tools/ref_gpu_compare.py does.

usage: bench_cdlp_directed.py [--scales 22,24] [--rounds 10] [--check-scale 16] [--steps 3] [--warmup 1]
                              [--impl gpu|reference] [--ref-lb cm,wm,cta] [--ref-repeat 3]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_core import card  # noqa: E402


def directed_rmat(pkg, scale):
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    return 1 << scale, src, dst


def parity(pkg, scale, rounds):
    from tests.cdlp_directed_cases import oracle
    n, src, dst = directed_rmat(pkg, scale)
    frag = pkg.Fragment.from_edges(n, src, dst, directed=True)
    app = pkg.App("cdlp_directed", frag, max_round=rounds)
    app.query()
    got = app.result()
    app.close()
    frag.close()
    return bool(np.array_equal(got, oracle(n, src, dst, rounds)))


def timed(pkg, kind, frag, rounds, steps, warmup):
    import torch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    app = pkg.App(kind, frag, max_round=rounds)
    rows = []
    for it in range(warmup + steps):
        flush.zero_()
        torch.cuda.synchronize()
        st = app.query()
        if it >= warmup:
            rows.append((st.query_ms, st.entries_scanned, st.kernel_launches))
    out = app.result()
    app.close()
    ms = [r[0] for r in rows]
    med = float(np.median(ms))
    return {"query_ms": med, "query_ms_all": [round(x, 3) for x in ms], "entries_scanned": int(rows[-1][1]),
            "entries_per_s": rows[-1][1] / (med * 1e-3), "kernel_launches": int(rows[-1][2]),
            "distinct_labels": int(len(np.unique(out)))}


def reference(scale, rounds, lbs, repeat):
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_gpu_driver")
    if not os.path.exists(exe):
        raise SystemExit("oracle/_ref/ref_gpu_driver is not built (needs the reference sources at build time)")
    cmd = [exe, "--application", "cdlp", "--directed", "1", "--cdlp_mr", str(rounds), "--rmat",
           "%d,16,1,0" % scale, "--lb", lbs, "--repeat", str(repeat)]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3600)
    if p.returncode != 0:
        return {"error": p.stderr[-600:]}
    by_lb = {}
    for r in (json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")):
        by_lb.setdefault(r["lb"], []).append(r["query_ms"])
    out = {lb: {"query_ms": float(np.median(ms[1:] if len(ms) > 1 else ms)), "query_ms_all": [round(x, 3) for x in ms]}
           for lb, ms in by_lb.items()}
    out["best_lb"] = min(by_lb, key=lambda lb: out[lb]["query_ms"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--check-scale", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-lb", default="cm,wm,cta")
    ap.add_argument("--ref-repeat", type=int, default=3)
    args = ap.parse_args()
    pkg = importlib.import_module("libgrape-lite_b200")
    line = {"bench": "cdlp_directed", "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
            "l2": "flushed (256 MB memset) before every query", "card": card(),
            "check_scale": args.check_scale, "parity": parity(pkg, args.check_scale, args.rounds), "runs": []}
    for scale in (int(x) for x in args.scales.split(",")):
        n, src, dst = directed_rmat(pkg, scale)
        run = {"graph": "directed R-MAT scale %d, edge factor 16, seed 1, one fragment" % scale, "scale": scale,
               "vertices": n, "edges": int(len(src))}
        frag = pkg.Fragment.from_edges(n, src, dst, directed=True)
        run["oe_entries"], run["ie_entries"] = int(frag.oe_num), int(frag.ie_num)
        run["gpu"] = timed(pkg, "cdlp_directed", frag, args.rounds, args.steps, args.warmup)
        frag.close()
        frag = pkg.Fragment.from_edges(n, src, dst)
        del src, dst
        run["cdlp_undirected"] = timed(pkg, "cdlp", frag, args.rounds, args.steps, args.warmup)
        frag.close()
        run["ratio_to_cdlp_undirected"] = run["gpu"]["query_ms"] / run["cdlp_undirected"]["query_ms"]
        if args.impl == "reference":
            run["reference"] = reference(scale, args.rounds, args.ref_lb, args.ref_repeat)
            run["reference_note"] = ("the reference's own GPU CDLP (cuda/cdlp/cdlp.h on its grape/cuda, "
                                     "kBothOutIn) on the same directed R-MAT input, generated inside the "
                                     "driver; host wall time of Query(), median after the first repetition")
            best = run["reference"].get("best_lb")
            if best:
                run["speedup_vs_reference"] = run["reference"][best]["query_ms"] / run["gpu"]["query_ms"]
        line["runs"].append(run)
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
