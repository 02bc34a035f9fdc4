#!/usr/bin/env python
"""Regenerates tests/golden/ref_bc_sources_outputs.npz: for a few graphs of tests/bc_cases.py and a
source list each, the f64 sum over the list of the f32 centrality c that the reference's CPU app bc
(oracle/_ref/ref_bc_driver, built by `make -C oracle/ref -f bc.mk`) computes with one thread, with
each source's own row skipped, in ascending-oid order.  Keys: "<case>" (the sums) and "<case>_sources"
(the list of oids).

  python tests/golden/make_ref_bc_sources_fixtures.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refbc  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests.bc_sources_cases import ref_cases  # noqa: E402

assert refbc.available(), "build oracle/_ref first: make -C oracle/ref -f bc.mk"
out = {}
for name, (n, src, dst, oids, sources) in ref_cases().items():
    order = np.sort(np.asarray(oids, dtype=np.int64)) if oids is not None else np.arange(n, dtype=np.int64)
    acc = np.zeros(n, dtype=np.float64)
    for s in sources:
        c, _, _ = refbc.run_app(n, src, dst, s, oids=oids, threads=1)
        c = c.astype(np.float64)
        c[order == s] = 0.0   # the source's own row is not a dependency
        acc += c
    out[name] = acc
    out[name + "_sources"] = np.asarray(sources, dtype=np.int64)
    print(name, len(sources), "sources", flush=True)
np.savez_compressed(os.path.join(G.GOLDEN, "ref_bc_sources_outputs.npz"), **out)
