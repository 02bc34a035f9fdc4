#!/usr/bin/env python
"""Regenerates tests/golden/ref_pagerank_local_outputs.{json,npz}: what the reference's CPU app
PageRankLocal (oracle/_ref/ref_pagerank_local_driver, built by
`make -C oracle/ref -f pagerank_local.mk` from the reference sources) computes on the inputs of
tests/pagerank_local_cases.py, on undirected and directed fragments: every case at every (d, R) of
REF_DELTAS x ROUNDS on 1 rank where the reference's avg_degree is at most 10 and on 2 and 3 ranks (the
MPI shim's GL_MPI_NP), the dense case at d = 0.85, R = 10 on 1 rank, and p2p-31 at d = 0.85, R = 10 on
1 rank, so that the tests compare with the reference where it is not installed.  The npz holds one f64
array per run in vertex-index order; the JSON holds each run's sum, the avg_degree the reference
reported on 1 rank, and the multi-rank runs left out because the reference does not complete them
(pagerank_local_cases.every_pair_linked).

  python tests/golden/make_ref_pagerank_local_fixtures.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import golden_io as G  # noqa: E402
from tests import pagerank_local_cases as P  # noqa: E402

assert os.path.exists(P.REF_EXE), "build oracle/_ref first: make -C oracle/ref -f pagerank_local.mk"
cases = P.pagerank_local_cases()
arrays, sums, avg, not_run = {}, {}, {}, []
for name, dr, delta, R, ranks in P.ref_runs(cases):
    n, s, d = cases[name]
    key = P.ref_key(name, dr, delta, R, ranks)
    if not P.every_pair_linked(n, s, d, ranks, dr == "directed"):
        not_run.append(key)
        continue
    arrays[key], a = P.run_ref(n, s, d, delta, R, dr == "directed", ranks)
    sums[key] = float(arrays[key].sum())
    if ranks == 1:
        avg[key] = a
    print(key, "sum %.17g" % sums[key], flush=True)
np.savez_compressed(os.path.join(G.GOLDEN, "ref_pagerank_local_outputs.npz"), **arrays)
with open(os.path.join(G.GOLDEN, "ref_pagerank_local_outputs.json"), "w") as f:
    json.dump({"sums": sums, "avg_degree": avg, "not_run": sorted(not_run),
               "not_run_reason": "not every pair of fragments holds an outer copy of the other's vertices; "
                                 "the reference's PageRankLocal does not complete there"},
              f, indent=1, sort_keys=True)
    f.write("\n")
