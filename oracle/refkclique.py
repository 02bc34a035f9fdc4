"""Runs oracle/_ref/ref_kclique_driver — the UNMODIFIED reference CPU app kclique
compiled against the shims (oracle/ref/kclique.mk).  TEST / MEASUREMENT ONLY."""
import json
import os
import subprocess
import tempfile

from . import refdriver

_HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(_HERE, "_ref", "ref_kclique_driver")


def available():
    return os.path.exists(EXE)


def _run(cmd, timeout):
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError("ref_kclique_driver failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
    return json.loads(p.stdout.strip().splitlines()[-1])


def run_app(n, src, dst, k, oids=None, simple=True, threads=4, timeout=3600):
    """The reference app's clique_num on the undirected graph (n, src, dst), one fragment;
    simple=True drops self loops and repeated pairs before loading."""
    with tempfile.TemporaryDirectory() as d:
        g = os.path.join(d, "g.bin")
        refdriver.write_graph(g, n, src, dst, None, oids)
        info = _run(["--graph", g, "--k", str(int(k)), "--simple", "1" if simple else "0",
                     "--threads", str(int(threads))], timeout)
        return int(info["clique_num"])


def run_rmat(scale, k, edgefactor=16, seed=1, repeat=1, threads=0, timeout=3600):
    """Times the reference app on the simplified R-MAT input generated inside the driver
    (oracle/rmat_gen.h).  -> info dict (clique_num, query_ms list, threads, load_s, ...)."""
    return _run(["--rmat", "%d,%d,%d" % (scale, edgefactor, seed), "--k", str(int(k)), "--simple", "1",
                 "--repeat", str(int(repeat)), "--threads", str(int(threads))], timeout)
