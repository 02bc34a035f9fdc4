"""Runs oracle/_ref/ref_lcc_directed_driver — the UNMODIFIED reference CPU app
LCCDirected<FRAG_T, uint64_t> compiled against the shims (oracle/ref/lcc_directed.mk).
TEST / MEASUREMENT ONLY."""
import json
import os
import subprocess
import tempfile

import numpy as np

from . import refdriver

_HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(_HERE, "_ref", "ref_lcc_directed_driver")


def available():
    return os.path.exists(EXE)


def _run(cmd, timeout):
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError("ref_lcc_directed_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
    return json.loads(p.stdout.strip().splitlines()[-1])


def parse(text):
    """`oid tricnt deduped_degree` lines -> (tri int64, d int64) in ascending-oid order."""
    rows = np.array([[int(x) for x in l.split()] for l in text.splitlines() if l.strip()], dtype=np.int64)
    rows = rows.reshape(-1, 3)
    k = np.argsort(rows[:, 0], kind="stable")
    return rows[k, 1], rows[k, 2]


def run_app(n, src, dst, oids=None, threads=1, timeout=3600):
    """The reference app on the directed graph (n, src, dst) -> (tri, d) in ascending-oid order."""
    with tempfile.TemporaryDirectory() as d:
        g = os.path.join(d, "g.bin")
        out = os.path.join(d, "out.txt")
        refdriver.write_graph(g, n, src, dst, None, oids)
        _run(["--graph", g, "--threads", str(int(threads)), "--out", out], timeout)
        return parse(open(out).read())


def run_rmat(scale, edgefactor=16, seed=1, repeat=1, threads=0, timeout=3600):
    """Times the reference app on the directed R-MAT graph generated inside the driver
    (oracle/rmat_gen.h).  -> info dict (query_ms list, threads, load_s, ...)."""
    return _run(["--rmat", "%d,%d,%d" % (scale, edgefactor, seed), "--repeat", str(int(repeat)),
                 "--threads", str(int(threads))], timeout)
