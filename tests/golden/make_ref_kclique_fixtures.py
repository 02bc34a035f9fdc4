#!/usr/bin/env python
"""Regenerates tests/golden/ref_kclique_outputs.json: {case: {k: count}} of what
the reference's CPU app kclique (oracle/_ref/ref_kclique_driver, built by
`make -C oracle/ref -f kclique.mk` from the reference sources) prints for the
cases of tests/kclique_cases.py, each loaded with self loops and repeated pairs
removed.  k runs over 3, 4, 5 and, where the clique number is at most 8 and
the counts stay small (at most 10^6 at every k), up to the clique number + 1
(count 0); the cases of K_UP_TO run over 3 .. K_UP_TO[case].

  python tests/golden/make_ref_kclique_fixtures.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refkclique  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests.kclique_cases import K_UP_TO, kclique_cases, ks_for  # noqa: E402

assert refkclique.available(), "build oracle/_ref first: make -C oracle/ref -f kclique.mk"
out = {}
for name, (n, src, dst, oids) in kclique_cases().items():
    counts = {k: refkclique.run_app(n, src, dst, k, oids=oids, threads=8) for k in (3, 4, 5)}
    k = 5
    while 0 < counts[k] <= 10 ** 6 and k < 9:   # the clique number is at least k
        k += 1
        counts[k] = refkclique.run_app(n, src, dst, k, oids=oids, threads=8)
    omega = max([j for j, c in counts.items() if c] + [2])
    ks = ks_for(omega) if counts[k] == 0 else [3, 4, 5]
    for j in range(6, K_UP_TO.get(name, 0) + 1):
        if j not in counts:
            counts[j] = refkclique.run_app(n, src, dst, j, oids=oids, threads=8)
        ks = sorted(set(ks) | {j})
    out[name] = {str(j): counts[j] for j in ks}
    print(name, out[name], flush=True)
with open(os.path.join(G.GOLDEN, "ref_kclique_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
