#!/usr/bin/env python
"""Regenerates tests/golden/ref_bc_outputs.json: digests (golden_io.digest) of
the depth, sigma and f32 centrality that the reference's CPU app bc
(oracle/_ref/ref_bc_driver, built by `make -C oracle/ref -f bc.mk` from the
reference sources) computes with ONE thread on the inputs of
tests/bc_cases.py, so that the tests compare with the reference where it is
not installed.  Every value array is in ascending-oid order.

  python tests/golden/make_ref_bc_fixtures.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refbc  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests.bc_cases import bc_cases  # noqa: E402

assert refbc.available(), "build oracle/_ref first: make -C oracle/ref -f bc.mk"
out = {}
for name, (n, src, dst, oids, source) in bc_cases().items():
    c, sigma, depth = refbc.run_app(n, src, dst, source, oids=oids, threads=1)
    reached = depth < np.iinfo(np.int64).max
    out[name] = {"source": int(source), "levels": int(depth[reached].max()) + 1 if reached.any() else 0,
                 "depth": G.digest(depth), "sigma": G.digest(sigma), "c": G.digest(c)}
    print(name, "levels", out[name]["levels"], flush=True)
with open(os.path.join(G.GOLDEN, "ref_bc_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
