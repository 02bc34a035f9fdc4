"""The un-normalised PageRank oracle (tests/pagerank_local_cases.py) on the CPU: against a plain
per-vertex loop, against the reference's own PageRankLocal (the fixtures, on 1, 2 and 3 ranks, and the
live oracle/_ref/ref_pagerank_local_driver when it was built), the reference's one-fragment
non-dividing branch on the dense case, and the row lengths the cases are built to reach."""
import os

import numpy as np
import pytest

from tests import pagerank_local_cases as P

CASES = P.pagerank_local_cases()
SMALL = sorted(k for k in CASES if k != "p2p31")
RUNS = P.ref_runs(CASES)


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("dr", P.DIRS)
def test_oracle_equals_plain_loop(name, dr):
    n, s, d = CASES[name]
    for delta in P.DELTAS:
        for R in P.ROUNDS:
            got = P.pagerank_local(n, s, d, delta, R, dr == "directed")
            want = P.plain_loop(n, s, d, delta, R, dr == "directed")
            assert np.allclose(got, want, rtol=1e-12, atol=0), (delta, R)


def test_fixture_runs():
    """Every run of ref_runs is in the npz, except the multi-rank runs the reference does not complete,
    which are exactly those where some fragment holds no outer copy of another's vertices."""
    meta, arrays = P.ref_pagerank_local_outputs()
    keys = {P.ref_key(*r) for r in RUNS}
    unlinked = {P.ref_key(*r) for r in RUNS
                if not P.every_pair_linked(*CASES[r[0]], r[4], r[1] == "directed")}
    assert set(meta["not_run"]) == unlinked
    assert set(arrays) == keys - unlinked
    assert all(k.endswith("np1") for k in meta["avg_degree"])
    # every case but the single-vertex and edgeless ones has multi-rank fixtures on both fragment kinds
    for name in ("mixed", "tier_rows", "long_rows", "random", "dense"):
        for dr in P.DIRS:
            assert P.ref_key(name, dr, 0.85, 10, 2) in arrays


def test_oracle_matches_reference_fixtures():
    meta, arrays = P.ref_pagerank_local_outputs()
    for name, dr, delta, R, ranks in RUNS:
        key = P.ref_key(name, dr, delta, R, ranks)
        if key not in arrays:
            continue
        n, s, d = CASES[name]
        ref = arrays[key]
        assert ref.shape == (n,) and meta["sums"][key] == pytest.approx(float(ref.sum()), rel=1e-12)
        if ranks == 1:
            avg = P.avg_degree(n, s, d, dr == "directed")
            assert meta["avg_degree"][key] == avg, key
            if avg > 10:
                continue      # test_dense_one_fragment_differs
        got = P.pagerank_local(n, s, d, delta, R, dr == "directed")
        assert np.allclose(got, ref, rtol=1e-9, atol=0), key


@pytest.mark.parametrize("dr", P.DIRS)
def test_dense_one_fragment_differs(dr):
    """On one fragment with avg_degree > 10 the reference never divides by the degree after PEval
    (pagerank_local.h's fnum() == 1 arm); on 2 and 3 fragments the same graph follows the definition."""
    meta, arrays = P.ref_pagerank_local_outputs()
    name, delta, R = P.DENSE
    n, s, d = CASES[name]
    assert P.avg_degree(n, s, d, dr == "directed") > 10
    ref = arrays[P.ref_key(name, dr, delta, R, 1)]
    undivided = P.pagerank_local(n, s, d, delta, R, dr == "directed", divide=False)
    defined = P.pagerank_local(n, s, d, delta, R, dr == "directed")
    assert np.allclose(ref, undivided, rtol=1e-9, atol=0)
    assert not np.allclose(ref, defined, rtol=1e-3, atol=0)
    assert ref.min() > 10 * defined.max()    # grown, not a PageRank
    for ranks in (2, 3):
        assert np.allclose(arrays[P.ref_key(name, dr, delta, R, ranks)], defined, rtol=1e-9, atol=0)


def test_undirected_is_n_times_normalised_pagerank():
    """Without zero-degree vertices, c(v) = N x the normalised rank of GL_APP_PAGERANK's pull (no dangling
    mass): the CPU check of the relation the GPU test makes against the app itself."""
    n, s, d = CASES["random"]
    r, c = P.rows(n, s, d, False)
    deg = np.bincount(r, minlength=n).astype(np.float64)
    keep = deg > 0
    remap = np.cumsum(keep) - 1
    n2, s2, d2 = int(keep.sum()), remap[s], remap[d]
    r2, c2 = P.rows(n2, s2, d2, False)
    deg2 = np.bincount(r2, minlength=n2).astype(np.float64)
    assert deg2.min() > 0
    x = np.full(n2, 1.0 / n2)
    for _ in range(10):
        x = (1 - 0.85) / n2 + 0.85 * np.bincount(r2, weights=(x / deg2)[c2], minlength=n2)
    got = P.pagerank_local(n2, s2, d2, 0.85, 10, False)
    assert np.allclose(got, n2 * x, rtol=1e-12, atol=0)


def test_cases_reach_the_tier_cuts():
    for dr in P.DIRS:
        n, s, d = CASES["tier_rows"]
        deg = np.bincount(P.rows(n, s, d, dr == "directed")[0], minlength=n)
        assert {32, 33, P.CHUNK, P.CHUNK + 1} <= set(deg[:4].tolist())
        n, s, d = CASES["long_rows"]
        deg = np.bincount(P.rows(n, s, d, dr == "directed")[0], minlength=n)
        assert deg.max() > 2 * P.CHUNK
    n, s, d = CASES["mixed"]
    outd, ind = np.bincount(s, minlength=n), np.bincount(d, minlength=n)
    assert ((outd == 0) & (ind > 0)).any() and ((outd == 0) & (ind == 0)).any()
    assert outd[3] == 1 and s[d == 3].tolist() == [3]
    assert (5 in s[s == d]) and outd[5] > 1


@pytest.mark.skipif(not os.path.exists(P.REF_EXE), reason="oracle/_ref/ref_pagerank_local_driver not built (needs the reference sources)")
@pytest.mark.parametrize("name", SMALL)
def test_live_reference(name):
    """The live driver against the oracle at d = 0, 1 (not in the fixtures) and bit for bit against the
    fixtures at d = 0.85, R = 10."""
    n, s, d = CASES[name]
    _, arrays = P.ref_pagerank_local_outputs()
    for dr in P.DIRS:
        directed = dr == "directed"
        for ranks in P.REF_RANKS:
            if not P.every_pair_linked(n, s, d, ranks, directed):
                continue
            if ranks == 1 and P.avg_degree(n, s, d, directed) > 10:
                continue
            for delta, R in ((0.0, 2), (1.0, 10)):
                ref, _ = P.run_ref(n, s, d, delta, R, directed, ranks)
                assert np.allclose(ref, P.pagerank_local(n, s, d, delta, R, directed), rtol=1e-9, atol=0)
            key = P.ref_key(name, dr, 0.85, 10, ranks)
            ref, _ = P.run_ref(n, s, d, 0.85, 10, directed, ranks)
            assert ref.tobytes() == arrays[key].tobytes(), key
