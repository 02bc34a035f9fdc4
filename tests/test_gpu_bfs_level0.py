"""Level 0 of the fused single-fragment BFS: the source's row split statically over every warp of
the cooperative grid (bfs_source_row_push, app_bfs.cu), each warp taking up to K_SRC_GROUPS
32-entry groups per pass.  The source rows sit on that split's thresholds -- empty, around one
group, one group per warp, K groups per warp (one pass or two) -- or carry a self loop and parallel
edges across a warp's slice boundary.  Every query is checked against the CPU oracle's depths, and
the size of level 1 against the distinct non-source neighbours in the fragment's CSR."""
import numpy as np
import pytest

from oracle import pyoracle
from tests.util import pkg

pytestmark = pytest.mark.gpu

K_SRC_GROUPS = 8     # kSrcGroups in app_bfs.cu
CTAS_PER_SM = 4      # k_bfs_fused's occupancy (GL_BFS_FUSED_CTAS): its grid is SMs x 4 CTAs of 8 warps
WARPS_PER_CTA = 8
FILL_MULT = 64       # parallel edges per filler pair

# push-only (the fragment's order), push/pull in the fragment's order, push/pull in hub-first order
CFGS = [dict(direction_opt=0, reserved={1: 1}), dict(direction_opt=1, reserved={1: 1}),
        dict(direction_opt=1, reserved={1: 2})]


def _warps():
    return pkg().device_info()["sm_count"] * CTAS_PER_SM * WARPS_PER_CTA


def _star(leaves, copies=None, self_loop=False, tail=0, hub=0):
    """Vertex 0 joined to the leaves 1..leaves (leaf i + 1 `copies[i]` times), optionally with a self
    loop, a path of `tail` vertices hanging off leaf 1 and a disconnected star of `hub` leaves.  Then
    disconnected filler pairs of FILL_MULT parallel edges with 16x the source row's entries, so that
    level 0 is a push level also with direction_opt = 1.  Returns (n, src, dst)."""
    rep = np.ones(leaves, dtype=np.int64) if copies is None else np.asarray(copies, dtype=np.int64)
    src = [np.zeros(int(rep.sum()), dtype=np.int64)]
    dst = [np.repeat(np.arange(1, leaves + 1, dtype=np.int64), rep)]
    row = int(rep.sum())
    n = leaves + 1
    if self_loop:
        src.append(np.zeros(1, dtype=np.int64))
        dst.append(np.zeros(1, dtype=np.int64))
        row += 2
    if tail:
        p = np.arange(n, n + tail, dtype=np.int64)
        src.append(np.concatenate([[1], p[:-1]]))
        dst.append(p)
        n += tail
    if hub:
        src.append(np.full(hub, n, dtype=np.int64))
        dst.append(np.arange(n + 1, n + 1 + hub, dtype=np.int64))
        n += hub + 1
    pairs = (16 * row + 128 + 2 * FILL_MULT - 1) // (2 * FILL_MULT)
    a = n + 2 * np.arange(pairs, dtype=np.int64)
    src.append(np.repeat(a, FILL_MULT))
    dst.append(np.repeat(a + 1, FILL_MULT))
    n += 2 * pairs
    return n, np.concatenate(src), np.concatenate(dst)


def _check(graph, cfgs=CFGS, queries=1, source=0):
    """Queries every configuration `queries` times on one app; returns the source's CSR row."""
    n, src, dst = graph
    frag = pkg().Fragment.from_edges(n, src, dst)
    g = pyoracle.Graph(n, src, dst, None)
    rp, col, _ = frag.csr(0)
    row = col[int(rp[source]):int(rp[source + 1])].astype(np.int64)
    distinct = len(np.unique(row[row != source]))
    want, _ = g.bfs(source)
    for cfg in cfgs:
        app = pkg().App("bfs", frag, source_oid=source, fuse_supersteps=1, **cfg)
        for q in range(queries):
            st = app.query()
            got = app.result()
            assert np.array_equal(got, want), (cfg, q, np.flatnonzero(got != want)[:8])
            assert st.step_frontier[2] == distinct, (cfg, q, st.step_frontier[2], distinct)
            # level 0 pushed the source row
            assert st.step_mode[1] == 0 and st.step_entries[1] == len(row), (cfg, q, st.step_entries[1], len(row))
        app.close()
    frag.close()
    return row


@pytest.mark.parametrize("leaves", [0, 1, 31, 32, 33])
def test_short_source_rows(leaves):
    """No entry, one entry, and rows around one 32-entry group."""
    assert len(_check(_star(leaves))) == leaves


@pytest.mark.parametrize("groups_per_warp", [1, K_SRC_GROUPS])
@pytest.mark.parametrize("delta", [-1, 1])
def test_source_rows_on_the_split_thresholds(groups_per_warp, delta):
    """warps x 32 +- 1 entries: one group per warp or two for some; warps x K x 32 +- 1: one pass of K
    groups per warp or a second pass.  Vertex 0's row starts at entry 0: the groups are the row's."""
    leaves = _warps() * 32 * groups_per_warp + delta
    assert len(_check(_star(leaves))) == leaves


def test_self_loop_and_parallel_edges_across_slices():
    """Every leaf two or three times and a self loop: runs of equal entries straddle boundaries
    between the warps' slices (checked on the fragment's order), and the source's own entries never
    count."""
    warps = _warps()
    leaves = warps * 32
    row = _check(_star(leaves, copies=2 + np.arange(leaves) % 2, self_loop=True))
    assert np.count_nonzero(row == 0) >= 1
    per = min(-(-((len(row) + 31) // 32) // warps), K_SRC_GROUPS)
    bounds = np.arange(32 * per, len(row), 32 * per)
    assert per >= 2 and np.count_nonzero(row[bounds - 1] == row[bounds]) > 0, per


def test_hub_first_source_below_the_maximum_degree():
    """Hub-first order forced on a small graph whose largest row is not the source's: the source
    keeps a lid other than 0 and its row starts inside a group."""
    _check(_star(1000, hub=3000), cfgs=[dict(direction_opt=d, reserved={1: 2}) for d in (0, 1)])


def test_three_queries_on_one_app():
    _check(_star(_warps() * 32 + 1), queries=3)


def test_query_after_a_spilled_query():
    """A ring of 4 level bitmaps: the first launch parks after level 2, the relaunch resumes from the
    parked state; the next query starts from a fresh seed again."""
    cfgs = [dict(c, reserved={**c["reserved"], 3: 4}) for c in CFGS]
    _check(_star(_warps() * 32 + 1, tail=12), cfgs=cfgs, queries=2)
