"""Runs oracle/_ref/ref_core_driver — the UNMODIFIED reference CPU apps
core_decomposition and kcore compiled against the shims (oracle/ref/core.mk).
TEST / MEASUREMENT ONLY."""
import json
import os
import subprocess
import tempfile

import numpy as np

from . import refdriver

_HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(_HERE, "_ref", "ref_core_driver")


def available():
    return os.path.exists(EXE)


def _run(cmd, timeout):
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError("ref_core_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
    return json.loads(p.stdout.strip().splitlines()[-1])


def run_app(app, n, src, dst, k=0, oids=None, threads=4, timeout=3600):
    """The reference app on the undirected graph (n, src, dst) -> its partial_result in
    ascending-oid order (int64).  app: "core_decomposition" | "kcore" (k = --kcore_k)."""
    with tempfile.TemporaryDirectory() as d:
        g = os.path.join(d, "g.bin")
        out = os.path.join(d, "out.txt")
        refdriver.write_graph(g, n, src, dst, None, oids)
        _run(["--app", app, "--graph", g, "--k", str(int(k)), "--threads", str(int(threads)), "--out", out], timeout)
        return refdriver.parse_output(open(out).read(), int)[1]


def run_rmat(app, scale, edgefactor=16, seed=1, k=0, repeat=1, threads=0, timeout=3600):
    """Times the reference app on bench's synthetic input, generated inside the driver
    (oracle/rmat_gen.h).  -> info dict (query_ms list, threads, load_s, ...)."""
    return _run(["--app", app, "--rmat", "%d,%d,%d" % (scale, edgefactor, seed), "--k", str(int(k)),
                 "--repeat", str(int(repeat)), "--threads", str(int(threads))], timeout)
