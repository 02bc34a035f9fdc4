#!/usr/bin/env python
"""Regenerates tests/golden/ref_pagerank_vc_outputs.{json,npz}: what the reference's CPU app PageRankVC
(oracle/_ref/ref_pagerank_vc_driver, built by `make -C oracle/ref -f pagerank_vc.mk` from the reference
sources) computes on the inputs of tests/pagerank_vc_cases.py ref_cases(), at every round count, damping
factor and fragment count listed there, so that the tests compare with the reference where it is not
installed.  The npz holds one f64 array per run in ascending-oid order (for p2p-31 and R-MAT 12 only the
sample_index vertices); the JSON holds each run's sum over all vertices and the runs the reference
aborted (its loader dies at 9 fragments on the smallest graphs).

  python tests/golden/make_ref_pagerank_vc_fixtures.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refprvc  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests import pagerank_vc_cases as P  # noqa: E402

assert refprvc.available(), "build oracle/_ref first: make -C oracle/ref -f pagerank_vc.mk"
arrays, sums, aborted = {}, {}, []
for name, (n, src, dst) in sorted(P.ref_cases().items()):
    idx = P.sample_index(n) if name in P.LARGE else np.arange(n)
    for R in P.REF_ROUNDS:
        for delta in P.REF_DELTAS:
            for fnum in P.REF_FNUMS:
                key = P.ref_key(name, R, delta, fnum)
                try:
                    out = refprvc.run_app(n, src, dst, delta, R, fnum, threads=1)
                except RuntimeError:
                    aborted.append(key)
                    print(key, "aborted", flush=True)
                    continue
                arrays[key] = out[idx]
                sums[key] = float(out.sum())
                print(key, "sum %.17g" % sums[key], flush=True)
np.savez_compressed(os.path.join(G.GOLDEN, "ref_pagerank_vc_outputs.npz"), **arrays)
with open(os.path.join(G.GOLDEN, "ref_pagerank_vc_outputs.json"), "w") as f:
    json.dump({"sums": sums, "aborted": aborted}, f, indent=1, sort_keys=True)
    f.write("\n")
