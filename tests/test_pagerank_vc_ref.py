"""The PageRankVC oracle (oracle/pagerank_vc_oracle.py) against the reference's own PageRankVC on
ImmutableVertexcutFragment: against the stored outputs (tests/golden/ref_pagerank_vc_outputs.*) at 1, 4
and 9 fragments, and against the live driver (oracle/_ref/ref_pagerank_vc_driver) when it is built.
The reference sums with f64 atomics in thread order, so values agree to 1e-9 relative, not bit for bit;
with max_round <= 0 both give 0.0 everywhere."""
import numpy as np
import pytest

from oracle import pagerank_vc_oracle as V
from oracle import refprvc
from tests import pagerank_vc_cases as P

META, ARRAYS = P.ref_pagerank_vc_outputs()
CASES = P.ref_cases()
RUNS = [(name, R, d, F) for name in sorted(CASES) for R in P.REF_ROUNDS for d in P.REF_DELTAS for F in P.REF_FNUMS]


def want(name, R, delta):
    n, s, d = CASES[name]
    return V.pagerank_vc(n, s, d, delta, R)


def test_fixtures_cover_every_run():
    keys = {P.ref_key(*r) for r in RUNS}
    assert set(ARRAYS) | set(META["aborted"]) == keys
    assert not set(ARRAYS) & set(META["aborted"])
    # the reference's loader aborts only at 9 fragments, and only on graphs below 9 x 2 vertices
    assert all(k.endswith("|F9") and CASES[k.split("|")[0]][0] < 18 for k in META["aborted"])


@pytest.mark.parametrize("name,R,delta,F", [r for r in RUNS if P.ref_key(*r) in ARRAYS])
def test_oracle_equals_reference_fixture(name, R, delta, F):
    key = P.ref_key(name, R, delta, F)
    w = want(name, R, delta)
    idx = P.sample_index(len(w)) if name in P.LARGE else np.arange(len(w))
    if R <= 0:
        assert not ARRAYS[key].any() and META["sums"][key] == 0.0
    np.testing.assert_allclose(ARRAYS[key], w[idx], rtol=1e-9, atol=0)
    np.testing.assert_allclose(META["sums"][key], w.sum(), rtol=1e-9)


def test_p2p31_has_the_isolated_oid_0():
    n, s, d = CASES["p2p31"]
    assert n == 62587 and not ((s == 0) | (d == 0)).any()
    key = P.ref_key("p2p31", 10, 0.85, 1)
    base_only = ARRAYS[key][0]   # an isolated vertex ends at base
    np.testing.assert_allclose(base_only, want("p2p31", 10, 0.85)[0], rtol=1e-12)


LIVE = [("n_103", F) for F in P.REF_FNUMS] + [("star_9000", 9), ("mid_row", 4), ("loops_dups", 4),
                                              ("p2p31", 4)]


@pytest.mark.skipif(not refprvc.available(), reason="oracle/_ref/ref_pagerank_vc_driver is not built")
@pytest.mark.parametrize("name,F", LIVE)
@pytest.mark.parametrize("R", [0, 10])
def test_oracle_equals_live_reference(name, F, R):
    n, s, d = CASES[name]
    got = refprvc.run_app(n, s, d, 0.85, R, F, threads=2)
    np.testing.assert_allclose(got, want(name, R, 0.85), rtol=1e-9, atol=0)
