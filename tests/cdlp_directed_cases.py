"""Inputs on which directed CDLP (GL_APP_CDLP_DIRECTED) is checked against the oracle and against the
reference's own GPU CDLP run with --directed 1 (label digests in tests/golden/ref_cdlp_directed_outputs.json,
written by golden/make_ref_cdlp_directed_fixtures.py).

Each case: (n, src, dst, oids or None); src / dst are oids when oids is given, vertex indices otherwise.
Edges are directed.  The cases are every graph of tests/directed_cases.py (outer copies seen only
through in-edges, the cycle, stars across the cut, ...), the multigraphs, the in-only vertex and the
inward / outward star rings of tests/lcc_directed_cases.py, and graphs made for the vote kernel:
  tie_halves   a vertex whose best in-label and best out-label tie in count (the smaller must win,
               whichever half it is in);
  sum_wins     a label present in both halves that wins only on its summed count;
  threshold    rows of kCdlpdWarpRow - 1, kCdlpdWarpRow and kCdlpdWarpRow + 1 entries (the warp / CTA
               cut of csrc/app_cdlp_directed.cu) with the split between in and out varied;
  reciprocal   every edge in both directions.

The oracle: directed CDLP on an edge list E is the undirected CDLP (oracle/oracle.cc, orc_cdlp) on the
undirected graph built from E, whose row of u is oe(u) + ie(u) as a multiset (a self loop is added
twice there, as it appears once in oe and once in ie); tests/test_cdlp_directed_oracle.py proves that
identity against brute force."""
import json
import os
from collections import Counter

import numpy as np

from tests import directed_cases as D
from tests import golden_io as G
from tests import lcc_directed_cases as LC
from tests.golden_io import GOLDEN

# csrc/app_cdlp_directed.cu kCdlpdWarpRow: rows with more in + out entries are voted by a CTA
WARP_ROW = 1024
ROUNDS = (0, 1, 2, 5, 10)


def tie_halves():
    """Vertex 10: in-edges 5 -> 10 twice, out-edges 10 -> 3 twice: 3 (out) and 5 (in) tie, 3 wins.
    Vertex 11: in-edges 2 -> 11 twice, out-edges 11 -> 7 twice: 2 (in) wins.  Vertex 12: in 4, 9 and
    out 4, 9: each label counts twice across the halves, 4 wins."""
    s = [5, 5, 10, 10, 2, 2, 11, 11, 4, 9, 12, 12]
    d = [10, 10, 3, 3, 11, 11, 7, 7, 12, 12, 4, 9]
    return 13, np.array(s, np.int64), np.array(d, np.int64)


def sum_wins():
    """Vertex 0: in-labels 1, 1, 1, 9, 9 and out-labels 2, 2, 2, 9, 9: 1 and 2 count 3 in one half each,
    9 counts 2 in each half and wins on its sum of 4 although it is the largest label."""
    s = [1, 1, 1, 9, 9, 0, 0, 0, 0, 0]
    d = [0, 0, 0, 0, 0, 2, 2, 2, 9, 9]
    return 10, np.array(s, np.int64), np.array(d, np.int64)


def threshold(seed=7):
    """Centres 200 .. whose in + out rows hold WARP_ROW - 1, WARP_ROW and WARP_ROW + 1 entries, split
    as (all out), (1 in), (half in), (all but 1 in), (all in); their neighbours are drawn with
    repetition from a pool 0 .. 199 that carries a random multigraph of its own, so counts differ."""
    rng = np.random.default_rng(seed)
    pool = 200
    n, s, d = LC.multigraph(pool, 800, seed)
    srcs, dsts = [s], [d]
    c = pool
    for total in (WARP_ROW - 1, WARP_ROW, WARP_ROW + 1):
        for k_in in (0, 1, total // 2, total - 1, total):
            ins = rng.integers(0, pool, k_in)
            outs = rng.integers(0, pool, total - k_in)
            srcs += [ins, np.full(total - k_in, c)]
            dsts += [np.full(k_in, c), outs]
            c += 1
    return c, np.concatenate(srcs).astype(np.int64), np.concatenate(dsts).astype(np.int64)


def _strip(shape):
    n, s, d = shape[:3]
    return n, np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64), None


def cdlp_directed_cases():
    """name -> (n, src, dst, oids or None)."""
    oids, src, dst, _ = G.load_p2p31()
    cases = {"p2p31": (len(oids), src, dst, oids)}
    for name in D.CASES:
        if name != "p2p31":
            cases[name] = _strip(D.build(name))
    for seed in (1, 2):
        cases["multigraph%d" % seed] = _strip(LC.multigraph(300, 3000, seed))
    cases["only_in"] = _strip(LC.only_in())
    cases["in_star4097"] = _strip(LC.star_ring(4097, True))
    cases["out_star4097"] = _strip(LC.star_ring(4097, False))
    cases["tie_halves"] = _strip(tie_halves())
    cases["sum_wins"] = _strip(sum_wins())
    cases["threshold"] = _strip(threshold())
    cases["reciprocal"] = _strip(LC.reciprocal(120, 0.1, 3))
    return cases


as_indices = LC.as_indices


def oracle(n, s, d, rounds, rank=None):
    """Directed CDLP labels per vertex index, as vertex indices: the undirected CDLP of the same edges.
    rank (optional): the position of every vertex in the order ties break in (gid order); default the
    index order."""
    from oracle import pyoracle
    if rank is None:
        return pyoracle.Graph(n, s, d).cdlp(rounds)
    by_rank = np.empty(n, dtype=np.int64)
    by_rank[rank] = np.arange(n)
    lab = pyoracle.Graph(n, rank[s], rank[d]).cdlp(rounds)
    return by_rank[lab[rank]]


def brute(n, s, d, rounds):
    """The definition, one round at a time: labels per vertex index after each round 0 .. rounds,
    from a Counter over the labels of the in-row followed by the out-row."""
    s = np.asarray(s, np.int64)
    d = np.asarray(d, np.int64)
    order = np.argsort(d, kind="stable")
    in_rp = np.concatenate([[0], np.cumsum(np.bincount(d, minlength=n))])
    in_col = s[order]
    order = np.argsort(s, kind="stable")
    out_rp = np.concatenate([[0], np.cumsum(np.bincount(s, minlength=n))])
    out_col = d[order]
    label = np.arange(n, dtype=np.int64)
    out = [label.copy()]
    for _ in range(rounds):
        new = label.copy()
        for v in range(n):
            row = np.concatenate([in_col[in_rp[v]:in_rp[v + 1]], out_col[out_rp[v]:out_rp[v + 1]]])
            if len(row) == 0:
                continue
            c = Counter(label[row].tolist())
            top = max(c.values())
            new[v] = min(x for x, k in c.items() if k == top)
        label = new
        out.append(label.copy())
    return out


# the reference's GPU CDLP behind run_cuda_app's command line: on this repository's compat headers, and
# on the reference's own grape/cuda (both built by __graft_entry__.build() when its sources are present)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_EXES = {"compat": os.path.join(ROOT, "oracle", "_ref", "compat", "run_compat_app"),
            "reference-gpu": os.path.join(ROOT, "oracle", "_ref", "ref_gpu_driver")}


def write_efile_vfile(d, n, src, dst, oids):
    """The case as p2p-31-style text files (`src dst 1` and `oid 0` lines, ids as oids); paths."""
    vid = np.arange(n, dtype=np.int64) if oids is None else np.sort(np.asarray(oids, dtype=np.int64))
    e, v = os.path.join(d, "g.e"), os.path.join(d, "g.v")
    with open(e, "w") as f:
        f.writelines("%d %d 1\n" % (a, b) for a, b in zip(np.asarray(src).tolist(), np.asarray(dst).tolist()))
    with open(v, "w") as f:
        f.writelines("%d 0\n" % x for x in vid.tolist())
    return e, v


def run_ref_cdlp(exe, efile, vfile, rounds, lb="cm", np_=1, timeout=900):
    """run_cuda_app --application cdlp --directed 1 --cdlp_mr rounds on the files, on np_ ranks (the MPI
    shim's GL_MPI_NP); the labels in ascending-oid order (int64) from every result_frag_* file."""
    import shutil
    import subprocess
    import tempfile
    out = tempfile.mkdtemp()
    try:
        cmd = [exe, "--application", "cdlp", "--directed", "1", "--cdlp_mr", str(rounds), "--efile", efile,
               "--vfile", vfile, "--out_prefix", out, "--lb", lb]
        env = dict(os.environ, GL_MPI_NP=str(np_), GL_MPI_TIMEOUT_S="300")
        p = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=timeout)
        if p.returncode != 0:
            raise RuntimeError("%s failed (%d): %s" % (" ".join(cmd), p.returncode, p.stderr[-2000:]))
        rows = []
        for f in range(np_):
            with open(os.path.join(out, "result_frag_%d" % f)) as fh:
                rows += [tuple(int(x) for x in line.split()[:2]) for line in fh if line.strip()]
    finally:
        shutil.rmtree(out, ignore_errors=True)
    rows.sort()
    return np.array([r[1] for r in rows], dtype=np.int64)


def ref_cdlp_directed_outputs():
    """name -> {"rounds": {str(R): digest of the labels in ascending-oid order}} of the reference's run."""
    with open(os.path.join(GOLDEN, "ref_cdlp_directed_outputs.json")) as f:
        return json.load(f)
