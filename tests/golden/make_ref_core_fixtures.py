#!/usr/bin/env python
"""Regenerates tests/golden/ref_core_outputs.json: digests (golden_io.digest)
of what the reference's CPU apps core_decomposition and kcore
(oracle/_ref/ref_core_driver, built by `make -C oracle/ref -f core.mk` from the
reference sources) compute on the inputs of tests/test_core_oracle.py and
tests/test_gpu_core.py, so that those tests compare with the reference where it
is not installed.  Every value array is in ascending-oid order.

  python tests/golden/make_ref_core_fixtures.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refcore  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests.core_cases import core_cases  # noqa: E402

assert refcore.available(), "build oracle/_ref first: make -C oracle/ref -f core.mk"
out = {}
for name, (n, src, dst, oids, ks) in core_cases().items():
    core = refcore.run_app("core_decomposition", n, src, dst, oids=oids)
    mx = int(core.max()) if len(core) else 0
    kk = sorted(set(ks) | {mx, mx + 1})
    out[name] = {"core": G.digest(core), "max_core": mx,
                 "kcore": {str(k): G.digest(refcore.run_app("kcore", n, src, dst, k=k, oids=oids)) for k in kk}}
    print(name, "max core", mx, flush=True)
with open(os.path.join(G.GOLDEN, "ref_core_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
