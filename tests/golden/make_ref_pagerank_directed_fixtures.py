#!/usr/bin/env python
"""Regenerates tests/golden/ref_pagerank_directed_outputs.{json,npz}: what the reference's CPU app
PageRankDirected (oracle/_ref/ref_pagerank_directed_driver, built by
`make -C oracle/ref -f pagerank_directed.mk` from the reference sources) computes on the inputs of tests/pagerank_directed_cases.py: every case at
every (d, R) of REF_DELTAS x ROUNDS, and p2p-31 at d = 0.85, R = 10, so that the tests compare with the
reference where it is not installed.  The npz holds one f64 array per run in vertex-index order; the JSON
holds each run's sum.

  python tests/golden/make_ref_pagerank_directed_fixtures.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import golden_io as G  # noqa: E402
from tests import pagerank_directed_cases as P  # noqa: E402

assert os.path.exists(P.REF_EXE), "build oracle/_ref first: make -C oracle/ref -f pagerank_directed.mk"
cases = P.pagerank_directed_cases()
arrays, sums = {}, {}
for name, delta, R in P.ref_runs():
    n, s, d = cases[name]
    key = P.ref_key(name, delta, R)
    arrays[key] = P.run_ref(n, s, d, delta, R)
    sums[key] = float(arrays[key].sum())
    print(key, "sum %.17g" % sums[key], flush=True)
np.savez_compressed(os.path.join(G.GOLDEN, "ref_pagerank_directed_outputs.npz"), **arrays)
with open(os.path.join(G.GOLDEN, "ref_pagerank_directed_outputs.json"), "w") as f:
    json.dump({"sums": sums}, f, indent=1, sort_keys=True)
    f.write("\n")
