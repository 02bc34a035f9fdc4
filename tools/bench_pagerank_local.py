#!/usr/bin/env python
"""Times un-normalised PageRank (csrc/app_pagerank_local.cu) on one GPU and prints one JSON line.
MEASUREMENT INFRASTRUCTURE (needs a GPU; writes nothing).

For every scale of --scales, on the undirected R-MAT fragment of that scale (Fragment.rmat: edge factor
16, seed 1, one fragment, as bench.py builds it) the app runs --rounds rounds at d = 0.85: it is warmed
up, then timed over --steps queries with the L2 flushed (256 MB memset) in front of each.  Reported: the
median device query_ms, ms per round, the oe entries a round reads, and the algorithmic bytes of a round
over its time: per oe entry a 4-byte column id and an 8-byte gather of x, per vertex its 8-byte row
pointers (read twice: the tier and the epilogue's degree) and its 8-byte x store.  GL_APP_PAGERANK's f64
pull (pr_pull = 1) runs the same way on the same fragment: the same pull over the same rows per round,
so the two times should be close.  Before timing, the result at --check-scale is compared with the
oracle (tests/pagerank_local_cases.py) to 1e-9 relative: "parity".  The card's name, power limit and
maximum and current SM clock are read (query only) in the same run.

--impl reference adds the reference's CPU PageRankLocal (oracle/_ref/ref_pagerank_local_driver, built
by __graft_entry__.build()) at --ref-scale on the same R-MAT edges, generated inside the driver, on an
undirected fragment: Query() of a fresh worker on all host threads, the median after the first of
--ref-repeat repetitions.  R-MAT's average degree is above 10, so on one fragment the reference takes
its branch that never divides by the degree: the same work per round, but a different output, which is
therefore not compared.

usage: bench_pagerank_local.py [--scales 22,24] [--rounds 10] [--check-scale 16] [--steps 3]
                               [--warmup 1] [--impl gpu|reference] [--ref-scale 22] [--ref-repeat 3]"""
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

DELTA = 0.85


def sm_clock_mhz():
    """The current SM clock of device 0 (a query), or None."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return float(q.stdout.strip())
    except Exception:
        return None


def parity(pkg, scale, rounds):
    from tests.pagerank_local_cases import pagerank_local
    src, dst, _ = pkg.rmat_edges_host(scale, 16, 1, 0)
    n = 1 << scale
    ok = True
    for directed in (False, True):
        frag = pkg.Fragment.from_edges(n, src, dst, directed=directed)
        app = pkg.App("pagerank_local", frag, pr_delta=DELTA, max_round=rounds)
        app.query()
        got = app.result()
        app.close()
        frag.close()
        ok = ok and bool(np.allclose(got, pagerank_local(n, src, dst, DELTA, rounds, directed), rtol=1e-9, atol=0))
    return ok


def timed(pkg, kind, frag, rounds, steps, warmup, **cfg):
    import torch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    app = pkg.App(kind, frag, pr_delta=DELTA, max_round=rounds, **cfg)
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
    return {"query_ms": med, "query_ms_all": [round(x, 3) for x in ms], "ms_per_round": med / rounds,
            "entries_scanned": int(rows[-1][1]), "kernel_launches": int(rows[-1][2]), "sum": float(out.sum()),
            "sm_clock_mhz_after": sm_clock_mhz()}


def reference(scale, rounds, repeat):
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_pagerank_local_driver")
    if not os.path.exists(exe):
        raise SystemExit("oracle/_ref/ref_pagerank_local_driver is not built (needs the reference sources at build time)")
    cmd = [exe, "--rmat", "%d,16,1" % scale, "--directed", "0", "--pr_d", repr(DELTA), "--mr", str(rounds),
           "--repeat", str(repeat)]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3600)
    if p.returncode != 0:
        return {"error": p.stderr[-600:]}
    info = json.loads(p.stdout.strip().splitlines()[-1])
    ms = info["query_ms"]
    return {"scale": scale, "query_ms": float(np.median(ms[1:] if len(ms) > 1 else ms)),
            "query_ms_all": [round(x, 3) for x in ms], "threads": info["threads"],
            "hardware_concurrency": info["hardware_concurrency"], "load_s": info["load_s"],
            "avg_degree": info["avg_degree"],
            "note": "one fragment with avg_degree > 10: the reference's non-dividing branch (the same work per "
                    "round, a different output), so its output is not compared"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--check-scale", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--impl", choices=("gpu", "reference"), default="gpu")
    ap.add_argument("--ref-scale", type=int, default=22)
    ap.add_argument("--ref-repeat", type=int, default=3)
    args = ap.parse_args()
    pkg = importlib.import_module("libgrape-lite_b200")
    line = {"bench": "pagerank_local", "delta": DELTA, "rounds": args.rounds, "steps": args.steps,
            "warmup": args.warmup, "l2": "flushed (256 MB memset) before every query", "card": card(),
            "sm_clock_mhz": sm_clock_mhz(), "check_scale": args.check_scale,
            "parity": parity(pkg, args.check_scale, args.rounds), "runs": []}
    for scale in (int(x) for x in args.scales.split(",")):
        frag = pkg.Fragment.rmat(scale, 16, seed=1)
        n, oe = int(frag.ivnum), int(frag.oe_num)
        run = {"graph": "undirected R-MAT scale %d, edge factor 16, seed 1, one fragment" % scale, "scale": scale,
               "vertices": n, "oe_entries_per_round": oe}
        round_bytes = oe * (4 + 8) + n * (8 + 8 + 8 + 8)
        run["bytes_per_round"] = round_bytes
        run["gpu"] = timed(pkg, "pagerank_local", frag, args.rounds, args.steps, args.warmup)
        run["gpu"]["algorithmic_GBps"] = round_bytes * args.rounds / (run["gpu"]["query_ms"] * 1e-3) / 1e9
        run["pagerank_pull_same_fragment"] = timed(pkg, "pagerank", frag, args.rounds, args.steps, args.warmup,
                                                   pr_pull=1)
        run["pagerank_note"] = ("GL_APP_PAGERANK's f64 pull (pr_pull = 1) on the same fragment: normalised by N, "
                                "dangling mass spread, the same pull over the same rows per round")
        frag.close()
        line["runs"].append(run)
    if args.impl == "reference":
        line["reference"] = reference(args.ref_scale, args.rounds, args.ref_repeat)
    print(json.dumps(line), flush=True)
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
