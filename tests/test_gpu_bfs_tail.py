"""Fused single-fragment BFS in hub-first order: the pull's stage 2 starts after
the hub neighbour, the sweeps stop at the last vertex with an edge, and the tail
levels walk a candidate list instead of the bitmap.  Every depth must match the
CPU oracle exactly, also when the level ring parks and relaunches the query
while the list is in use, and on the paths that keep the old pull (directed
graphs, fragment order)."""
import numpy as np
import pytest

from oracle import pyoracle
from tests.util import pkg, rmat_graph

pytestmark = pytest.mark.gpu


def _sources(g, n):
    rp, _, _ = g.csr()
    deg = np.diff(rp.astype(np.int64))
    low = int(np.flatnonzero(deg == 1)[0])         # a degree-1 vertex: mostly a stage-1 miss
    iso = np.flatnonzero(deg == 0)
    return [int(g.max_degree_vertex()), low, int(iso[-1]) if len(iso) else n - 1]


@pytest.mark.parametrize("scale", [16, 20])
@pytest.mark.parametrize("ring", [0, 4, 5])
def test_bfs_hub_first_tail_vs_oracle(scale, ring):
    """R-MAT graphs whose unreachable remainder is far below the list capacity: the tail levels
    run from the candidate list by themselves.  A ring of 4 or 5 level bitmaps parks the query every
    few levels, so that some relaunches fall into list mode (the list is rebuilt by a sweep)."""
    n, src, dst, _ = rmat_graph(scale, seed=1)
    g = pyoracle.Graph(n, src, dst, None)
    frag = pkg().Fragment.rmat(scale, 16, seed=1)
    reserved = {1: 2}          # hub-first order also below 2^16 vertices
    if ring:
        reserved[3] = ring
    sources = _sources(g, n)
    for source in sources:
        app = pkg().App("bfs", frag, source_oid=source, direction_opt=1, fuse_supersteps=1, reserved=reserved)
        st = app.query()
        want, _ = g.bfs(source)
        assert np.array_equal(app.result(), want), "source %d" % source
        if source == sources[0]:
            assert any(st.step_mode[i] == 1 for i in range(st.n_steps))     # pull levels really ran
        app.query()                    # the lists and their counters reset between queries
        assert np.array_equal(app.result(), want)
        app.close()
    frag.close()


@pytest.mark.parametrize("fuse", [0, 1])
def test_bfs_fragment_order_keeps_full_pull(fuse):
    """cfg.reserved[1] = 1 keeps the fragment's own order: hub_nbr is the true highest-degree
    neighbour, not the first entry of the row, so stage 2 scans whole rows and sweeps cover every
    vertex."""
    scale = 16
    n, src, dst, _ = rmat_graph(scale, seed=2)
    g = pyoracle.Graph(n, src, dst, None)
    frag = pkg().Fragment.rmat(scale, 16, seed=2)
    for source in _sources(g, n):
        app = pkg().App("bfs", frag, source_oid=source, fuse_supersteps=fuse, reserved={1: 1})
        app.query()
        want, _ = g.bfs(source)
        assert np.array_equal(app.result(), want), "source %d" % source
        app.close()
    frag.close()


@pytest.mark.parametrize("ring", [0, 4])
def test_bfs_directed_keeps_full_pull(ring):
    """Directed graph: the pull walks the ie rows, which are not in hub-first order."""
    scale = 16
    n, src, dst, _ = rmat_graph(scale, seed=9)
    g = pyoracle.Graph(n, src, dst, None, directed=True)
    frag = pkg().Fragment.from_edges(n, src, dst, directed=True)
    rp, _, _ = frag.csr(0)
    source = int(np.argmax(np.diff(rp.astype(np.int64))))
    app = pkg().App("bfs", frag, source_oid=source, direction_opt=1, fuse_supersteps=1,
                    reserved={3: ring} if ring else {})
    st = app.query()
    want, _ = g.bfs(source)
    assert np.array_equal(app.result(), want)
    assert any(st.step_mode[i] == 1 for i in range(st.n_steps))
    app.close()
    frag.close()
