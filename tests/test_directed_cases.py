"""CPU: every directed case of tests/directed_cases.py reaches the fragment
geometry it is listed for at 2 and 3 fragments, and the oracle the
several-fragment directed tests compare with still reproduces the reference's
directed golden files."""
import numpy as np
import pytest

from tests import directed_cases as D
from tests import shapes as S
from tests.test_oracle_golden import p2p, test_bfs, test_pagerank_directed, test_sssp  # noqa: F401


@pytest.mark.parametrize("fnum", D.FNUMS)
@pytest.mark.parametrize("name", list(D.CASES))
def test_case_reaches_its_geometry(name, fnum):
    n, src, dst, _ = D.build(name)
    got = D.claims(name, n, src, dst, fnum)
    assert got, "case %s lists no geometry" % name
    missed = [what for what, ok in got if not ok]
    assert not missed, "%s at fnum=%d: %s" % (name, fnum, missed)


def test_shrunk_cases_lose_their_geometry():
    """The claims are tied to the thresholds the cases are sized for: a shrunk case fails them."""
    small = {"sink4097": S.sink_heavy(10), "source4097": S.source_heavy(10), "reversed_path": D.reversed_path(200),
             "cycle": D.cycle(100), "star_last": S.star(100, True), "hub_block": S.hub_block(4)}
    for name, (n, src, dst, _) in small.items():
        for fnum in D.FNUMS:
            assert not all(ok for _, ok in D.claims(name, n, src, dst, fnum)), (name, fnum)


def test_geometry_on_a_hand_checked_graph():
    # 0 -> 3, 4 -> 1, 5 -> 2, 2 -> 2; fnum 2 splits {0, 1, 2} | {3, 4, 5}
    geo = D.geometry(6, np.array([0, 4, 5, 2]), np.array([3, 1, 2, 2]), 2)
    g0, g1 = geo
    assert (g0["lo"], g0["hi"], g1["lo"], g1["hi"]) == (0, 3, 3, 6)
    assert list(g0["oe_outer"]) == [3] and list(g0["ie_outer"]) == [4, 5] and list(g0["ie_only"]) == [4, 5]
    assert list(g0["outer"]) == [3, 4, 5] and list(g0["in_from"]) == [1]
    assert list(g0["dangling_cross"]) == [1]          # 2 has an out-edge (its self loop)
    assert list(g1["oe_outer"]) == [1, 2] and list(g1["ie_outer"]) == [0] and list(g1["ie_only"]) == [0]
    assert list(g1["dangling_cross"]) == [3]


def test_sources_and_ok_line_count():
    n, src, dst, _ = D.build("reversed_path")
    s = D.sources(n, src, dst, 3)
    assert s["last_frag"] == n - 1 and s["unknown"] >= n
    assert s["ie_only"] in D.geometry(n, src, dst, 3)[0]["ie_only"]
    per = {real: len(D.BFS_CONFIGS) * len(D.BFS_SOURCES) + len(D.BFS_SOURCES_FUSED)
           + len(D.SSSP_SOURCES) * len(D.SSSP_REAL if real else D.SSSP_INT)
           + len(D.WCC_KINDS) + len(D.PR_CONFIGS) + 1 for real in (False, True)}
    nreal = sum(1 for _, real in D.CASES.values() if real)
    assert D.ok_lines_expected() == (len(D.CASES) - nreal) * per[False] + nreal * per[True] + 13
