"""Runs oracle/_ref/ref_bc_driver — the UNMODIFIED reference CPU app bc
(StagedBCBFS then StagedBC) compiled against the shims (oracle/ref/bc.mk).
TEST / MEASUREMENT ONLY."""
import json
import os
import subprocess
import tempfile

import numpy as np

from . import refdriver

_HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(_HERE, "_ref", "ref_bc_driver")


def available():
    return os.path.exists(EXE)


def _run(cmd, timeout):
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError("ref_bc_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
    return json.loads(p.stdout.strip().splitlines()[-1])


def parse(text):
    """`oid c sigma depth` lines -> (c float32, sigma float64, depth int64) in ascending-oid order."""
    rows = [l.split() for l in text.splitlines() if l.strip()]
    oid = np.array([int(r[0]) for r in rows], dtype=np.int64)
    c = np.array([float.fromhex(r[1]) for r in rows], dtype=np.float64).astype(np.float32)
    sigma = np.array([float(r[2]) for r in rows], dtype=np.float64)
    depth = np.array([int(r[3]) for r in rows], dtype=np.int64)
    k = np.argsort(oid, kind="stable")
    return c[k], sigma[k], depth[k]


def run_app(n, src, dst, source, oids=None, threads=1, timeout=3600):
    """The reference app on the undirected graph (n, src, dst) from the source OID
    -> (c, sigma, depth) in ascending-oid order.  threads=1 is the order the replay
    oracle reproduces bit for bit."""
    with tempfile.TemporaryDirectory() as d:
        g = os.path.join(d, "g.bin")
        out = os.path.join(d, "out.txt")
        refdriver.write_graph(g, n, src, dst, None, oids)
        _run(["--graph", g, "--source", str(int(source)), "--threads", str(int(threads)), "--out", out], timeout)
        return parse(open(out).read())


def run_rmat(scale, edgefactor=16, seed=1, source="maxdeg", repeat=1, threads=0, timeout=3600):
    """Times the reference app on bench's synthetic input, generated inside the driver
    (oracle/rmat_gen.h).  -> info dict (query_ms list, threads, source, load_s, ...)."""
    return _run(["--rmat", "%d,%d,%d" % (scale, edgefactor, seed), "--source", str(source),
                 "--repeat", str(int(repeat)), "--threads", str(int(threads))], timeout)
