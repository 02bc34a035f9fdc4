#!/usr/bin/env python
"""Regenerates tests/golden/ref_cdlp_directed_outputs.json: digests (golden_io.digest) of the labels, in
ascending-oid order, that the reference's own GPU CDLP (cuda/cdlp/cdlp.h on its grape/cuda, run as
`run_cuda_app --application cdlp --directed 1`: oracle/_ref/ref_gpu_driver, built by
__graft_entry__.build() from the reference sources) computes on the inputs of tests/cdlp_directed_cases.py
after 1, 2, 5 and 10 rounds, one fragment, --lb cm.  Needs a GPU.  Round 0 is not recorded: the
reference's context is left uninitialised there.

  python tests/golden/make_ref_cdlp_directed_fixtures.py
"""
import json
import os
import shutil
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import golden_io as G  # noqa: E402
from tests.cdlp_directed_cases import REF_EXES, cdlp_directed_cases, run_ref_cdlp, write_efile_vfile  # noqa: E402

REF_ROUNDS = (1, 2, 5, 10)
exe = REF_EXES["reference-gpu"]
assert os.path.exists(exe), "build oracle/_ref first: python -c 'import __graft_entry__ as g; g.build()'"
tmp = tempfile.mkdtemp()
jobs = []
for name, (n, src, dst, oids) in sorted(cdlp_directed_cases().items()):
    d = os.path.join(tmp, name)
    os.makedirs(d)
    e, v = write_efile_vfile(d, n, src, dst, oids)
    jobs += [(name, r, e, v) for r in REF_ROUNDS]
with ThreadPoolExecutor(8) as pool:
    labels = list(pool.map(lambda j: run_ref_cdlp(exe, j[2], j[3], j[1]), jobs))
shutil.rmtree(tmp, ignore_errors=True)
out = {}
for (name, r, _, _), lab in zip(jobs, labels):
    out.setdefault(name, {"rounds": {}})["rounds"][str(r)] = G.digest(lab)
    print(name, r, "labels", len(lab), "distinct", len(set(lab.tolist())), flush=True)
with open(os.path.join(G.GOLDEN, "ref_cdlp_directed_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
