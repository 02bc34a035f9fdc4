#!/usr/bin/env python
"""Regenerates tests/golden/ref_outputs.{json,npz}: what the reference's CPU
apps (oracle/_ref/ref_driver, built by `make -C oracle ref` from the reference
sources) compute on the inputs of tests/test_ref_golden.py, test_rmat_def.py,
test_shapes_oracle.py and test_gpu_fullsize.py.  Those tests compare with the stored results, so they
run where the reference is not installed.

Exact results are stored as digests (golden_io.digest; WCC labels after
golden_io.canonical_labels, the partition the reference's check compares),
PageRank vectors as float64 values (a seeded sample of them at scale 20).
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import pyoracle, refdriver  # noqa: E402
from tests import golden_io as G  # noqa: E402
from tests import shapes  # noqa: E402
from tests.test_gpu_fullsize import REF_SCALE, pagerank_sample_index  # noqa: E402
from tests.test_ref_golden import _random_graph  # noqa: E402
from tests.test_rmat_def import RMAT_CASES  # noqa: E402
from tests.util import rmat_graph  # noqa: E402

assert refdriver.available(), "build oracle/_ref first: make -C oracle ref"
out, arrays = {}, {}
tmp = tempfile.mkdtemp()


def run(app, path, parse=float, **kw):
    _, text = refdriver.run_app(app, path, **kw)
    return refdriver.parse_output(text, parse)[1]


# test_ref_golden.py: R-MAT scale 12 with self loops and duplicate edges
n, src, dst, w = rmat_graph(12, seed=21, weight_mode=1)
path = os.path.join(tmp, "rmat.bin")
refdriver.write_graph(path, n, src, dst, w.astype(np.float64))
s = int(pyoracle.Graph(n, src, dst, w.astype(np.float64)).max_degree_vertex())
out["rmat12"] = {"source": s,
                 "bfs": G.digest(run("bfs", path, int, source=s, threads=4)),
                 "sssp": G.digest(run("sssp", path, source=s, threads=4)),
                 "wcc": G.digest(run("wcc", path, int, threads=4)),
                 "cdlp5": G.digest(run("cdlp", path, int, mr=5, threads=4)),
                 "lcc": G.digest(run("lcc", path, threads=4))}
arrays["rmat12_pagerank10"] = run("pagerank", path, pr_d=0.85, mr=10, threads=4)

# test_ref_golden.py: random multigraphs
for seed in range(8):
    rng = np.random.RandomState(1000 + seed)
    n = int(rng.randint(20, 400))
    m = int(rng.randint(n // 2, 6 * n))
    src, dst, w = _random_graph(rng, n, m, weighted=True)
    path = os.path.join(tmp, "g.bin")
    refdriver.write_graph(path, n, src, dst, w)
    d = {}
    for directed in (False, True):
        s = int(rng.randint(0, n))
        d["directed%d" % directed] = {
            "source": s,
            "bfs": G.digest(run("bfs", path, int, directed=directed, source=s, threads=3)),
            "sssp": G.digest(run("sssp", path, directed=directed, source=s, threads=3))}
    d["wcc"] = G.digest(run("wcc", path, int, threads=3))
    d["cdlp4"] = G.digest(run("cdlp", path, int, mr=4, threads=3))
    d["lcc"] = G.digest(run("lcc", path, threads=3))
    arrays["multi%d_pagerank7" % seed] = run("pagerank", path, pr_d=0.85, mr=7, threads=3)
    out["multi%d" % seed] = d

# test_rmat_def.py: the edge lists of the reference arm's generator (oracle/rmat_gen.h)
out["rmat_edges"] = {}
for scale, seed, wmode in RMAT_CASES:
    f = os.path.join(tmp, "e.bin")
    refdriver.subprocess.check_call([refdriver.EXE, "--rmat", "%d,16,%d,%d" % (scale, seed, wmode), "--dump-edges", f])
    raw = np.fromfile(f, dtype=np.int64)
    m = 16 << scale
    e = {"src": G.digest(raw[:m]), "dst": G.digest(raw[m:2 * m])}
    if wmode:
        e["w"] = G.digest(raw[2 * m:].view(np.float64))
    out["rmat_edges"]["%d,%d,%d" % (scale, seed, wmode)] = e

# test_shapes_oracle.py: PageRank after 0 and 1 rounds on a star (undirected) and on a
# directed star into a sink, from both CPU PageRank apps of the reference
for name, (n, src, dst, _), directed in (("star5", shapes.star(5), False), ("sink4", shapes.sink_heavy(4), True)):
    path = os.path.join(tmp, "shape.bin")
    refdriver.write_graph(path, n, src, dst)
    for app in ("pagerank", "pagerank_parallel"):
        for mr in (0, 1):
            arrays["%s_%s%d" % (name, app, mr)] = run(app, path, directed=directed, pr_d=0.85, mr=mr, threads=1)

info = refdriver.run_rmat("bfs", 12, 16, 1, repeat=1)
out["rmat12_seed1_bfs_info"] = {"source": int(info["source"]), "traversed_edges": int(info["traversed_edges"])}

# test_gpu_fullsize.py: R-MAT scale 20, the reference generating its input itself
out["scale%d" % REF_SCALE] = {}
for app in ("bfs", "sssp", "wcc", "pagerank", "cdlp"):
    f = os.path.join(tmp, "out.txt")
    info = refdriver.run_rmat(app, REF_SCALE, 16, 1, repeat=1, out=f)
    oids, vals = refdriver.parse_output(open(f).read(), float if app in ("sssp", "pagerank") else int)
    assert np.array_equal(oids, np.arange(1 << REF_SCALE))
    d = {"source": int(info["source"])}
    if app == "pagerank":
        arrays["scale%d_pagerank10_sample" % REF_SCALE] = vals[pagerank_sample_index(len(vals))]
    else:
        d["digest"] = G.digest(G.canonical_labels(vals) if app == "wcc" else vals)
    out["scale%d" % REF_SCALE][app] = d

with open(os.path.join(G.GOLDEN, "ref_outputs.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
np.savez_compressed(os.path.join(G.GOLDEN, "ref_outputs.npz"), **arrays)
print("wrote ref_outputs.json, ref_outputs.npz")
