#!/usr/bin/env python
"""Splits the time of bench.py's headline BFS query (R-MAT scale 24, one GPU, the
fused single-launch query) by level.  MEASUREMENT INFRASTRUCTURE (needs a GPU;
writes nothing).

The configuration is bench.py's with --sweep none: R-MAT --scale, edge factor 16,
seed 1, one fragment, push/pull, fused query, from the maximum-degree vertex;
warmed up, then --steps device-timed queries with the L2 flushed (256 MB memset)
in front of each.  Printed, as a table and then as one JSON line: the median
query time, per level the median time (from the kernel's per-level timestamps),
its mode (0 push, 1 pull), CSR entries scanned and frontier size, and the median
gap = query time - sum of the level times: the launch, the time from the last
level to the end of the kernel and the epilogue (control-block copy, end event).
Entries and modes are those of the last query (they are the same in every query).
GL_KTIME=1 in the environment also prints, per query, the kernel's own split of
the gap (stderr).  The card's name and power limit are read in the same run.

usage: bench_bfs_split.py [--scale 24] [--steps 20] [--warmup 3]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("libgrape-lite_b200")
    frag = pkg.Fragment.rmat(args.scale, 16, seed=1)
    src = int(frag.max_degree_vertex()[0])   # lid == oid on the R-MAT builder (bench.py's source rule)
    app = pkg.App("bfs", frag, None, source_oid=src, direction_opt=1, fuse_supersteps=1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(max(args.warmup, 1)):
        flush.zero_()
        torch.cuda.synchronize()
        app.query()
    q, lv, gap = [], [], []
    for _ in range(args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        st = app.query()
        ms = [st.step_ms[i] for i in range(st.n_steps)]
        q.append(st.query_ms)
        lv.append(ms)
        gap.append(st.query_ms - sum(ms))
        last = dict(mode=[int(st.step_mode[i]) for i in range(st.n_steps)],
                    entries=[int(st.step_entries[i]) for i in range(st.n_steps)],
                    frontier=[int(st.step_frontier[i]) for i in range(st.n_steps)])
    app.close()
    frag.close()
    n = min(len(x) for x in lv)
    med = np.median(np.array([x[:n] for x in lv]), axis=0)
    # step 0 is the seed (inside the kernel's prologue, 0 ms); levels are steps 1..n-1
    levels = [dict(level=i - 1, ms=round(float(med[i]), 4), mode=last["mode"][i], entries=last["entries"][i],
                   frontier=last["frontier"][i]) for i in range(1, n)]
    line = dict(workload="BFS R-MAT scale-%d ef-16 seed 1, 1 fragment, fused query, source %d" % (args.scale, src),
                card=card(), steps=args.steps, ms_per_query=round(float(np.median(q)), 4),
                ms_per_query_range=[round(float(min(q)), 4), round(float(max(q)), 4)],
                gap_ms=round(float(np.median(gap)), 4), levels=levels)
    print("level  mode        ms      entries    frontier")
    for r in levels:
        print("%5d  %4d  %8.4f  %11d  %10d" % (r["level"], r["mode"], r["ms"], r["entries"], r["frontier"]))
    print("query %.4f ms (median of %d), gap (query - sum of levels) %.4f ms" % (line["ms_per_query"], args.steps,
                                                                               line["gap_ms"]))
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
