"""Source lists for betweenness centrality over many sources, on graphs of tests/bc_cases.py, whose
reference sums are in tests/golden/ref_bc_sources_outputs.npz (golden/make_ref_bc_sources_fixtures.py).
Each case: (n, src, dst, oids or None, list of source oids)."""
import os

import numpy as np

from tests.bc_cases import bc_cases, max_degree_index
from tests.core_cases import as_indices
from tests.golden_io import GOLDEN


def seeded_list(n, src, dst, oids, k, seed):
    """k source oids: the maximum-degree vertex first, then a seeded sample (repeats allowed)."""
    s, d = as_indices(n, src, dst, oids)
    idx = [max_degree_index(n, s, d)] + np.random.default_rng(seed).integers(0, n, size=k - 1).tolist()
    return [int(oids[i]) if oids is not None else int(i) for i in idx]


def ref_cases():
    """name -> (n, src, dst, oids, sources): p2p-31 and R-MAT 12 with 24 seeded sources, the diamond chain
    from every joint, and a shape with parallel edges and self loops from every vertex."""
    cases = bc_cases()
    out = {}
    for name in ("p2p31", "rmat12"):
        n, src, dst, oids, _ = cases[name if name != "p2p31" else "p2p31_src6"]
        out[name] = (n, src, dst, oids, seeded_list(n, src, dst, oids, 24, seed=31))
    n, src, dst, oids, _ = cases["diamond_chain40"]
    out["diamond_chain40"] = (n, src, dst, oids, list(range(0, n, 4)))
    multi = "random5"
    n, src, dst, oids, _ = cases[multi]
    out[multi] = (n, src, dst, oids, list(range(n)) if n <= 200 else seeded_list(n, src, dst, oids, 64, seed=5))
    return out


def ref_bc_sources_outputs():
    """name -> sums (f64, ascending-oid order), and name + "_sources" -> the list."""
    with np.load(os.path.join(GOLDEN, "ref_bc_sources_outputs.npz")) as z:
        return {k: z[k] for k in z.files}
