"""The directed PageRank oracle (tests/pagerank_directed_cases.py) on the CPU: against a plain per-vertex
loop on the small cases, against the reference's own PageRankDirected (the fixtures, and the live
oracle/_ref/ref_pagerank_directed_driver when it was built), the sum of the group's results, and the row lengths the cases
are built to reach."""
import os

import numpy as np
import pytest

from tests import pagerank_directed_cases as P

CASES = P.pagerank_directed_cases()
SMALL = sorted(k for k in CASES if k != "p2p31")


@pytest.mark.parametrize("name", SMALL)
def test_oracle_equals_plain_loop(name):
    n, s, d = CASES[name]
    for delta in P.DELTAS:
        for R in P.ROUNDS:
            got = P.pagerank_directed(n, s, d, delta, R)
            want = P.plain_loop(n, s, d, delta, R)
            assert np.allclose(got, want, rtol=1e-12, atol=0), (delta, R)


@pytest.mark.parametrize("name", sorted(CASES))
def test_results_sum_to_one(name):
    n, s, d = CASES[name]
    for delta in P.DELTAS:
        for R in P.ROUNDS:
            got = P.pagerank_directed(n, s, d, delta, R)
            if R <= 0:
                assert not got.any()
            else:
                assert abs(got.sum() - 1.0) <= 1e-12, (delta, R, got.sum())


def test_oracle_matches_reference_fixtures():
    meta, arrays = P.ref_pagerank_directed_outputs()
    assert set(arrays) == {P.ref_key(*r) for r in P.ref_runs()}
    for name, delta, R in P.ref_runs():
        n, s, d = CASES[name]
        key = P.ref_key(name, delta, R)
        ref = arrays[key]
        assert ref.shape == (n,) and meta["sums"][key] == pytest.approx(float(ref.sum()), rel=1e-12)
        got = P.pagerank_directed(n, s, d, delta, R)
        if R <= 0:
            assert not ref.any(), key      # the reference's zero-initialised result
        else:
            assert np.allclose(got, ref, rtol=1e-9, atol=0), key


def test_p2p31_differs_from_the_pagerank_parallel_golden():
    """GL_APP_PAGERANK's directed golden file (pagerank_parallel.h: a sink is reset to base) sums to about
    0.46 on p2p-31; the Graphalytics definition sums to 1."""
    from tests import golden_io as G
    golden = np.array([float(v) for _, v in G.golden_pairs("p2p-31-PR-directed")])
    n, s, d = CASES["p2p31"]
    got = P.pagerank_directed(n, s, d, 0.85, 10)
    assert len(golden) == n and abs(golden.sum() - 0.462) < 0.01
    assert abs(got.sum() - 1.0) <= 1e-12
    sinks_with_in = (np.bincount(s, minlength=n) == 0) & (np.bincount(d, minlength=n) > 0)
    assert sinks_with_in.sum() == 46199


def test_cases_reach_the_tier_cuts():
    n, s, d = CASES["tier_rows"]
    ind = np.bincount(d, minlength=n)
    assert {32, 33, P.CHUNK, P.CHUNK + 1} <= set(ind.tolist())
    n, s, d = CASES["long_rows"]
    assert np.bincount(d, minlength=n).max() > 2 * P.CHUNK
    assert np.bincount(s, minlength=n).max() > P.CHUNK
    n, s, d = CASES["mixed"]
    outd, ind = np.bincount(s, minlength=n), np.bincount(d, minlength=n)
    assert ((outd == 0) & (ind > 0)).any() and ((outd == 0) & (ind == 0)).any()
    loops = s == d
    assert any(outd[v] == 1 for v in s[loops])


@pytest.mark.skipif(not os.path.exists(P.REF_EXE), reason="oracle/_ref/ref_pagerank_directed_driver not built (needs the reference sources)")
@pytest.mark.parametrize("name", sorted(CASES))
def test_live_reference(name):
    n, s, d = CASES[name]
    runs = [(0.85, 10)] if name == "p2p31" else [(dl, r) for dl in P.DELTAS for r in P.ROUNDS]
    for delta, R in runs:
        ref = P.run_ref(n, s, d, delta, R)
        got = P.pagerank_directed(n, s, d, delta, R)
        if R <= 0:
            assert not ref.any()
        else:
            assert np.allclose(got, ref, rtol=1e-9, atol=0), (delta, R)
