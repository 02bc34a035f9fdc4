"""CPU: the oracle of directed CDLP (tests/cdlp_directed_cases.py `oracle`: the undirected CDLP of the
same edges) against the definition counted out by brute force over the in-row followed by the out-row,
on every case after 0, 1, 2, 5 and 10 rounds; against the digests of the reference's own GPU CDLP run
with --directed 1 (tests/golden/ref_cdlp_directed_outputs.json); and the statistics model
(oracle/stats_model.py cdlp over the combined row pointer ie_rp + oe_rp) split into fragment shares."""
import numpy as np
import pytest

from oracle import pyoracle
from oracle import stats_model as M
from tests import golden_io as G
from tests.cdlp_directed_cases import ROUNDS, as_indices, brute, cdlp_directed_cases, oracle, ref_cdlp_directed_outputs

CASES = cdlp_directed_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_is_the_definition(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    by_round = brute(n, s, d, max(ROUNDS))
    for r in ROUNDS:
        got = oracle(n, s, d, r)
        assert np.array_equal(got, by_round[r]), (name, r, np.flatnonzero(got != by_round[r])[:10])


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_the_reference(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    vid = np.arange(n, dtype=np.int64) if oids is None else np.sort(np.asarray(oids, dtype=np.int64))
    ref = ref_cdlp_directed_outputs()[name]["rounds"]
    assert sorted(ref, key=int) == ["1", "2", "5", "10"]
    for r, want in ref.items():
        assert G.digest(vid[oracle(n, s, d, int(r))]) == want, (name, r)


def test_the_vote_cases_do_what_they_are_made_for():
    n, s, d, _ = CASES["tie_halves"]
    assert oracle(n, s, d, 1)[[10, 11, 12]].tolist() == [3, 2, 4]
    n, s, d, _ = CASES["sum_wins"]
    assert oracle(n, s, d, 1)[0] == 9
    # an in-only vertex updates (GL_APP_CDLP would keep its label)
    n, s, d, _ = CASES["only_in"]
    assert np.bincount(s, minlength=n)[0] == 0 and oracle(n, s, d, 1)[0] != 0


@pytest.mark.parametrize("name", ["p2p31", "cycle", "rmat12", "only_in", "threshold"])
@pytest.mark.parametrize("fnum", [1, 2, 3])
def test_stats_shares(name, fnum):
    """Per-round entries of a fragment = the ie and oe entries of its inner rows; the shares add up to
    the one-fragment value."""
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    g = pyoracle.Graph(n, s, d, directed=True)
    rp = g.csr(False)[0].astype(np.int64) + g.csr(True)[0].astype(np.int64)
    chunk = -(-n // fnum)
    total = 0
    for fid in range(fnum):
        st = M.cdlp(rp, 5, fid, fnum)
        lo, hi = min(n, fid * chunk), min(n, (fid + 1) * chunk)
        own = int(np.count_nonzero((s >= lo) & (s < hi)) + np.count_nonzero((d >= lo) & (d < hi)))
        assert st.supersteps == 6 and st.step_entries == [0] + [own] * 5
        assert st.touched_vertices == (hi - lo) * 5
        total += st.entries_scanned
    assert total == M.cdlp(rp, 5).entries_scanned == 5 * 2 * len(s)
