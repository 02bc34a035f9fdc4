"""Betweenness centrality (csrc/app_bc.cu) on the threshold graphs of
tests/bc_shapes.py, bit for bit against the order-exact oracle
(oracle/bc_oracle.py bc_rows) on the fragment's own CSR.

For every graph, every source of bc_shapes.sources() and direction_opt 0 and 1:
depth, path_num and centrality equal bc_rows exactly; the two direction_opt
runs and a second query are byte-identical; and the per-step statistics equal
the host replicas of bc_shapes (the push / pull rule of every forward level,
the entries every step reads).  Each graph first checks, on the fragment's CSR,
that it reaches the branch it is there for."""
import numpy as np
import pytest

from oracle import bc_oracle as BO
from tests import bc_shapes as B
from tests.util import pkg

pytestmark = pytest.mark.gpu


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8).tobytes()


def check_exact(got, want):
    """got: the app's BC_DTYPE result; want: (c, sigma, depth) of bc_rows."""
    c, sigma, depth = want
    assert np.array_equal(got["depth"], depth), np.flatnonzero(got["depth"] != depth)[:8]
    bad = np.flatnonzero(got["path_num"].view(np.uint64) != sigma.view(np.uint64))
    assert len(bad) == 0, ("path_num", bad[:8], got["path_num"][bad[:8]], sigma[bad[:8]])
    want_c = c.astype(np.float64)
    bad = np.flatnonzero(got["centrality"].view(np.uint64) != want_c.view(np.uint64))
    assert len(bad) == 0, ("centrality", bad[:8], got["centrality"][bad[:8]], want_c[bad[:8]])


def check_steps(st, n, rp, col, depth, direction_opt):
    """The step statistics of one single-fragment query against the host replicas."""
    cap = pkg().GL_MAX_STEP_STATS
    fwd = B.forward_steps(n, rp, col, depth, direction_opt)
    back = B.backward_entries(rp, depth)
    L1 = len(fwd)
    assert st.n_steps == min(2 * L1, cap)
    modes = [int(st.step_mode[i]) for i in range(st.n_steps)]
    entries = [int(st.step_entries[i]) for i in range(st.n_steps)]
    want_m = ([m for m, _ in fwd] + [2] * L1)[:cap]
    want_e = ([e for _, e in fwd] + back[::-1])[:cap]
    assert modes == want_m, [(i, a, b) for i, (a, b) in enumerate(zip(modes, want_m)) if a != b][:8]
    assert entries == want_e, [(i, a, b) for i, (a, b) in enumerate(zip(entries, want_e)) if a != b][:8]
    return modes


@pytest.mark.parametrize("name", sorted(B.BC_SHAPES))
def test_bc_shape(name):
    build, root = B.BC_SHAPES[name]
    n, s, d, _ = build()
    frag = pkg().Fragment.from_edges(n, s, d)
    assert frag.ivnum == n
    rp, col, _ = frag.csr(0)
    rp, col = rp.astype(np.int64), col.astype(np.int64)
    srcs = B.sources(n, rp, col, root)
    checks = B.reach_checks(name, n, rp, col, srcs[0])
    assert all(ok for _, ok in checks), [what for what, ok in checks if not ok]
    pulled = {}
    for source in srcs:
        want = BO.bc_rows(n, rp, col, source if 0 <= source < n else None)
        runs = []
        for dopt in (0, 1):
            app = pkg().App("bc", frag, source_oid=source, direction_opt=dopt)
            st = app.query()
            got = app.result()
            check_exact(got, want)
            modes = check_steps(st, n, rp, col, want[2], dopt)
            pulled[(source, dopt)] = 1 in modes
            app.query()   # a second query on the same app
            assert app.result().tobytes() == got.tobytes(), (source, dopt, "second query")
            app.close()
            runs.append(got.tobytes())
        assert runs[0] == runs[1], (source, "direction_opt 0 and 1 differ")
    assert not any(p for (_, dopt), p in pulled.items() if dopt == 0)
    if name == "star70000":
        # from the centre and from a leaf, direction_opt = 1 reaches a pull level
        assert pulled[(0, 1)] and pulled[(1, 1)]
    frag.close()
