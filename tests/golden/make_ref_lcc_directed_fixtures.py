#!/usr/bin/env python
"""Regenerates tests/golden/ref_lcc_directed_outputs.json: digests (golden_io.digest) of the tri and
deduplicated-degree arrays that the reference's CPU app LCCDirected (oracle/_ref/ref_lcc_directed_driver,
built by `make -C oracle/ref -f lcc_directed.mk` from the reference sources) computes on the inputs of
tests/lcc_directed_cases.py, so that the tests compare with the reference where it is not installed.
Every array is in ascending-oid order.

  python tests/golden/make_ref_lcc_directed_fixtures.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import reflccd  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests.lcc_directed_cases import lcc_directed_cases  # noqa: E402

assert reflccd.available(), "build oracle/_ref first: make -C oracle/ref -f lcc_directed.mk"
out = {}
for name, (n, src, dst, oids) in lcc_directed_cases().items():
    tri, d = reflccd.run_app(n, src, dst, oids=oids, threads=1)
    out[name] = {"tri": G.digest(tri), "d": G.digest(d), "tri_sum": int(tri.sum())}
    print(name, "tri_sum", out[name]["tri_sum"], flush=True)
with open(os.path.join(G.GOLDEN, "ref_lcc_directed_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
