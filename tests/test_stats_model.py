"""The host model of the query statistics (oracle/stats_model.py) on graphs small
enough to count by hand: the expected numbers are written out here."""
import numpy as np
import pytest

from oracle import stats_model as M


def csr(n, edges, directed=False):
    """Rows in input order of the entries: edge (u, v) is an entry of u's row and,
    undirected, one of v's (a self loop gives two entries)."""
    rows = [[] for _ in range(n)]
    for u, v in edges:
        rows[u].append(v)
        if not directed:
            rows[v].append(u)
    rp = np.zeros(n + 1, dtype=np.int64)
    rp[1:] = np.cumsum([len(r) for r in rows])
    return rp, np.array([v for r in rows for v in r], dtype=np.int64)


PATH5 = csr(5, [(0, 1), (1, 2), (2, 3), (3, 4)])
STAR4 = csr(5, [(0, 1), (0, 2), (0, 3), (0, 4)])
# two triangles 0-1-2 and 3-4-5 joined by 2-3
BOWTIE = csr(6, [(0, 1), (1, 2), (0, 2), (3, 4), (4, 5), (3, 5), (2, 3)])
# 0-1 three times, a self loop at 1, 1-2, and the isolated vertex 3
MULTI = csr(4, [(0, 1), (0, 1), (0, 1), (1, 1), (1, 2)])


def test_bfs_push_path():
    s = M.bfs_push(*PATH5, 0)
    assert s.supersteps == 6 and s.n_steps == 6
    assert s.step_frontier == [0, 1, 1, 1, 1, 1]
    assert s.step_entries == [0, 1, 2, 2, 2, 1]
    assert s.step_mode == [0] * 6
    assert (s.entries_scanned, s.frontier_vertices, s.touched_vertices) == (8, 5, 4)
    s = M.bfs_push(*PATH5, 2)
    assert s.supersteps == 4
    assert s.step_frontier == [0, 1, 2, 2] and s.step_entries == [0, 2, 4, 2]
    assert s.touched_vertices == 4


def test_bfs_push_star():
    s = M.bfs_push(*STAR4, 0)
    assert s.step_frontier == [0, 1, 4] and s.step_entries == [0, 4, 4] and s.supersteps == 3
    s = M.bfs_push(*STAR4, 3)
    assert s.step_frontier == [0, 1, 1, 3] and s.step_entries == [0, 1, 4, 3] and s.supersteps == 4
    assert s.touched_vertices == 4


def test_bfs_push_bowtie():
    s = M.bfs_push(*BOWTIE, 0)
    # levels {0}, {1, 2}, {3}, {4, 5}
    assert s.step_frontier == [0, 1, 2, 1, 2]
    assert s.step_entries == [0, 2, 5, 3, 4]
    assert (s.entries_scanned, s.frontier_vertices, s.touched_vertices, s.supersteps) == (14, 6, 5, 5)


def test_bfs_push_multigraph():
    s = M.bfs_push(*MULTI, 0)
    # row 0: three entries; row 1: 3 + 2 (the loop) + 1; row 2: one; vertex 3 is not reached
    assert s.step_frontier == [0, 1, 1, 1]
    assert s.step_entries == [0, 3, 6, 1]
    assert s.touched_vertices == 2
    s = M.bfs_push(*MULTI, 3)   # an isolated source
    assert s.step_frontier == [0, 1] and s.step_entries == [0, 0] and s.supersteps == 2
    assert s.touched_vertices == 0


def test_bfs_source_not_in_graph():
    s = M.bfs_push(*PATH5, None)
    assert s.supersteps == 1 and s.entries_scanned == 0 and s.frontier_vertices == 0 and s.touched_vertices == 0


def test_bfs_pull_bounds():
    # star from a leaf: expanding {leaf} finds the centre; 4 rows of 7 entries are not yet reached
    # (one probe and the row each); expanding {centre} finds 3 leaves, whose 3 rows of one entry are left
    assert M.bfs_pull_bounds(*STAR4, 3) == [(1, 11), (3, 6), (0, 0)]


def test_direction_rule():
    # star of 4 leaves from the centre: level 0 has 4 of the 8 entries, 4 > (8 - 4) / 14: pull at once;
    # level 1 (4 vertices, 5 * 24 > 5) stays in the pull phase
    assert M.bfs_direction_modes([1, 4], [4, 4], 8, 5, 5) == [M.PULL, M.PULL]
    # a path: one or two of 1998 entries per level never exceed a 14th of the rest until the very end
    sizes, ents = [1] * 1000, [1] + [2] * 998 + [1]
    modes = M.bfs_direction_modes(sizes, ents, 1998, 1000, 1000)
    assert modes[:900] == [M.PUSH] * 900
    first_pull = modes.index(M.PULL)
    # m_f = 2 > m_u // 14 first holds with m_u = 27: 1 + 2 * d entries seen, 1998 - 27 = 1971 -> level 985
    assert first_pull == 985
    # pull, then the frontier drops below vnum / beta with many vertices left: back to push for good
    modes = M.bfs_direction_modes([1, 100, 2, 1, 1], [1000, 5000, 4, 2, 2], 20000, 10000, 10000, beta=200)
    assert modes == [M.PUSH, M.PULL, M.PUSH, M.PUSH, M.PUSH]
    # a larger divisor keeps the second level in the pull phase
    assert M.bfs_direction_modes([1, 100, 2], [1000, 5000, 4], 20000, 10000, 10000, beta=10000)[:3] == [0, 1, 1]


def test_dense_apps():
    s = M.pagerank(BOWTIE[0], 3)
    assert s.supersteps == 5 and s.step_entries == [0, 14, 14, 14, 0] and s.step_frontier == [0, 6, 6, 6, 0]
    assert s.step_mode == [0, 2, 2, 2, 0] and s.touched_vertices == 18
    s = M.pagerank(BOWTIE[0], 0)
    assert s.supersteps == 2 and s.entries_scanned == 0 and s.touched_vertices == 0
    s = M.cdlp(MULTI[0], 2)
    assert s.supersteps == 3 and s.step_entries == [0, 10, 10] and s.step_frontier == [0, 4, 4]
    assert M.cdlp(MULTI[0], 0).supersteps == 1 and M.cdlp(MULTI[0], 1).supersteps == 2
    assert M.cdlp(MULTI[0], 1).step_entries == [0, 10]


def test_lcc():
    # bow tie: degrees 2 2 3 3 2 2.  N+(0) = {}, N+(1) = {0}, N+(2) = {0, 1}, N+(3) = {2, 4, 5},
    # N+(4) = {}, N+(5) = {4}: the DAG entries (v, u) read |N+(u)| = (1,0):0 (2,0):0 (2,1):1
    # (3,2):2 (3,4):0 (3,5):1 (5,4):0
    s = M.lcc(*BOWTIE)
    assert s.step_entries == [0, 4, 0] and s.step_frontier == [0, 6, 0] and s.supersteps == 3
    # a star: only the centre has DAG entries, and they lead to the leaves' empty DAG rows
    assert M.lcc(*STAR4).step_entries[1] == 0


def test_kcore_entries():
    deg = np.diff(BOWTIE[0])
    assert M.kcore_entries(BOWTIE[0], deg, 3) == 8          # values 2 2 3 3 2 2: the four corners' rows
    assert M.kcore_entries(BOWTIE[0], deg, 1) == 0


@pytest.mark.parametrize("fnum", [2, 3])
def test_fragment_shares_add_up(fnum):
    for rp, col in (PATH5, STAR4, BOWTIE, MULTI):
        n = len(rp) - 1
        ranges = [M.fragment_range(n, f, fnum) for f in range(fnum)]
        assert ranges[0][0] == 0 and ranges[-1][1] == n
        assert all(ranges[i][1] == ranges[i + 1][0] for i in range(fnum - 1))
        for source in range(n):
            one = M.bfs_push(rp, col, source)
            parts = [M.bfs_push(rp, col, source, f, fnum) for f in range(fnum)]
            assert all(p.supersteps == one.supersteps for p in parts)
            assert [sum(x) for x in zip(*[p.step_frontier for p in parts])] == one.step_frontier
            assert [sum(x) for x in zip(*[p.step_entries for p in parts])] == one.step_entries
        for make in (M.pagerank, M.cdlp):
            one = make(rp, 3)
            parts = [make(rp, 3, f, fnum) for f in range(fnum)]
            assert sum(p.entries_scanned for p in parts) == one.entries_scanned
            assert sum(p.frontier_vertices for p in parts) == one.frontier_vertices
            assert sum(p.touched_vertices for p in parts) == one.touched_vertices


def test_fragment_range_is_ceil_chunks():
    assert [M.fragment_range(5, f, 3) for f in range(3)] == [(0, 2), (2, 4), (4, 5)]
    assert [M.fragment_range(4, f, 3) for f in range(3)] == [(0, 2), (2, 4), (4, 4)]
    assert M.fragment_range(0, 0, 2) == (0, 0)
