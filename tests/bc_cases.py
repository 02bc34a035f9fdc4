"""Inputs on which betweenness centrality is compared with the reference CPU app
(digests in tests/golden/ref_bc_outputs.json, written by
golden/make_ref_bc_fixtures.py): the graphs of tests/core_cases.py from their
maximum-degree vertex, plus p2p-31 from oids 6 and 0, R-MAT 12 from a degree-1
vertex, a source oid that is not in the graph, and a chain of diamonds whose
path counts grow as 3^k past 2^53.  Each case: (n, src, dst, oids or None,
source oid); src / dst are oids when oids is given, vertex indices otherwise."""
import json
import os

import numpy as np

from tests.core_cases import as_indices, core_cases
from tests.golden_io import GOLDEN


def degrees(n, s, d):
    """CSR entries per vertex index (a self loop counts twice)."""
    return np.bincount(np.concatenate([np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64)]), minlength=n)


def max_degree_index(n, s, d):
    """The vertex with the most CSR entries, ties to the smallest index (bench's --source maxdeg)."""
    return int(np.argmax(degrees(n, s, d))) if n else 0


def diamond_chain(k):
    """Joints 0, 4, 8, .. 4k joined by three middle vertices each: sigma(joint i) = 3^i."""
    src, dst = [], []
    for i in range(k):
        j, nxt = 4 * i, 4 * i + 4
        for m in (1, 2, 3):
            src += [j, j + m]
            dst += [j + m, nxt]
    return 4 * k + 1, np.array(src, dtype=np.int64), np.array(dst, dtype=np.int64)


def bc_cases():
    """name -> (n, src, dst, oids, source oid)."""
    cases = {}
    for name, (n, src, dst, oids, _) in core_cases(big=False).items():
        s, d = as_indices(n, src, dst, oids)
        v = max_degree_index(n, s, d)
        if name == "p2p31":
            cases["p2p31_src6"] = (n, src, dst, oids, 6)
            cases["p2p31_src0"] = (n, src, dst, oids, 0)
            continue
        if name == "rmat12":
            deg = degrees(n, s, d)
            cases["rmat12_deg1"] = (n, src, dst, oids, int(np.flatnonzero(deg == 1)[0]))
            cases["rmat12_absent"] = (n, src, dst, oids, 1 << 40)
        cases[name] = (n, src, dst, oids, int(oids[v]) if oids is not None else v)
    n, s, d = diamond_chain(40)
    cases["diamond_chain40"] = (n, s, d, None, 0)
    return cases


def source_index(n, oids, source):
    """The vertex index of a source oid, or None when the oid is not in the graph."""
    if oids is None:
        return int(source) if 0 <= source < n else None
    o = np.sort(np.asarray(oids, dtype=np.int64))
    i = int(np.searchsorted(o, source))
    return i if i < n and o[i] == source else None


def ref_bc_outputs():
    """name -> {"source", "levels", "depth", "sigma", "c": digests} of the reference app's one-thread run."""
    with open(os.path.join(GOLDEN, "ref_bc_outputs.json")) as f:
        return json.load(f)

