"""Runs oracle/_ref/ref_pagerank_vc_driver — the UNMODIFIED reference CPU app PageRankVC on
ImmutableVertexcutFragment, compiled against the shims (oracle/ref/pagerank_vc.mk).
TEST / MEASUREMENT ONLY."""
import glob
import json
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(_HERE, "_ref", "ref_pagerank_vc_driver")


def available():
    return os.path.exists(EXE)


def _run(cmd, np_ranks, timeout):
    env = dict(os.environ, GL_MPI_NP=str(int(np_ranks)))
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout,
                       env=env)
    if p.returncode != 0:
        raise RuntimeError("ref_pagerank_vc_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
    return json.loads(p.stdout.strip().splitlines()[-1])


def run_app(n, src, dst, delta=0.85, max_round=10, np_ranks=1, threads=1, timeout=3600):
    """The reference app on (n, src, dst) at np_ranks fragments -> one f64 per vertex 0..n-1 (every
    vertex is the master of exactly one fragment)."""
    with tempfile.TemporaryDirectory() as d:
        efile = os.path.join(d, "g.e")
        with open(efile, "w") as f:
            for a, b in zip(np.asarray(src, dtype=np.int64).tolist(), np.asarray(dst, dtype=np.int64).tolist()):
                f.write("%d %d\n" % (a, b))
        prefix = os.path.join(d, "out")
        _run(["--efile", efile, "--vnum", str(int(n)), "--pr_d", repr(float(delta)), "--pr_mr", str(int(max_round)),
              "--threads", str(int(threads)), "--out", prefix], np_ranks, timeout)
        out = np.full(n, np.nan)
        seen = np.zeros(n, dtype=np.int64)
        for path in glob.glob(prefix + ".*"):
            for line in open(path):
                oid, val = line.split()
                out[int(oid)] = float(val)
                seen[int(oid)] += 1
        if not np.all(seen == 1):
            raise RuntimeError("reference output does not cover every vertex exactly once")
        return out


def run_rmat(scale, edgefactor=16, seed=1, delta=0.85, max_round=10, np_ranks=1, repeat=1, threads=0,
             timeout=3600):
    """Times the reference app on the R-MAT graph generated inside the driver -> info dict."""
    return _run(["--rmat", "%d,%d,%d" % (scale, edgefactor, seed), "--pr_d", repr(float(delta)),
                 "--pr_mr", str(int(max_round)), "--repeat", str(int(repeat)), "--threads", str(int(threads))],
                np_ranks, timeout)
