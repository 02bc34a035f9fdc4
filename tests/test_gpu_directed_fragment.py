"""GPU: every fragment of a 2-, 3- and 8-way directed split stores exactly the
adjacency the edge list gives it, entry by entry against numpy.

On a directed fragment `oe` holds the out-edges and `ie` the in-edges of the
inner vertices, and the outer vertex set is the union of the outer columns of
both.  The reverse adjacency of the outer vertices (`ov_ie`, csr(2)) is the
transpose of the outer part of `oe` only: an outer vertex the fragment sees only
through an in-edge has an empty row there, which wcc_opt relies on when it
decides which rows it may skip."""
import numpy as np
import pytest

from tests import directed_cases as D
from tests import shapes as S
from tests.util import pkg

pytestmark = pytest.mark.gpu


def _rmat11():
    src, dst, w = pkg().rmat_edges_host(11, 16, 31, 1)
    return 1 << 11, src, dst, w.astype(np.float64)


def _check_rows(rp, col, w, lid2g, ivnum, lo, rows_g, nbr_g, w_g, n):
    """Row r of the fragment CSR (rp, col, w) holds the entries (rows_g == lo + r, nbr_g, w_g):
    inner neighbours first, then outer ones, each part ascending by global id; weights follow
    their entry (a multi-edge's copies may carry their weights in any order)."""
    rows = np.repeat(np.arange(ivnum, dtype=np.int64), np.diff(rp).astype(np.int64))
    assert np.array_equal(np.diff(rp).astype(np.int64), np.bincount(rows_g - lo, minlength=ivnum))
    inner = (nbr_g >= lo) & (nbr_g < lo + ivnum)
    order = np.lexsort((w_g, nbr_g, ~inner, rows_g))
    got_g = lid2g[col]
    assert np.array_equal(got_g, nbr_g[order])
    assert np.array_equal(col < ivnum, inner[order])
    key = col.astype(np.int64) + rows * (1 << 33)
    assert np.all(np.diff(key) >= 0)
    got_w = w.astype(np.float64)
    mine = np.lexsort((got_w, got_g, rows))
    assert np.array_equal(got_w[mine], w_g[order][np.lexsort((w_g[order], nbr_g[order], rows_g[order] - lo))])


@pytest.mark.parametrize("case", ["rmat11", "sink4097"])
@pytest.mark.parametrize("fnum", [2, 3, 8])
def test_directed_split_layout(case, fnum):
    n, src, dst, w = _rmat11() if case == "rmat11" else S.sink_heavy(4097)
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    w32 = np.asarray(w, dtype=np.float32)
    wd = w32.astype(np.float64)
    chunk = D.chunk_of(n, fnum)
    geo = D.geometry(n, src, dst, fnum)
    oe_sum = ie_sum = 0
    ie_only_rows = 0
    for fid in range(fnum):
        g = geo[fid]
        lo, hi = g["lo"], g["hi"]
        f = pkg().Fragment.from_edges(n, src, dst, w32, directed=True, fid=fid, fnum=fnum)
        assert (f.fid, f.fnum, f.directed, f.ivnum) == (fid, fnum, 1, hi - lo)
        ovgid = f.ovgid()
        off = f.fid_offset
        owner = (ovgid >> off).astype(np.int64)
        glob_outer = owner * chunk + (ovgid & ((1 << off) - 1)).astype(np.int64)
        # the outer vertices: the distinct non-inner endpoints of both CSRs, ascending, grouped by owner
        assert f.ovnum == len(g["outer"])
        assert np.all(np.diff(ovgid.astype(np.int64)) > 0) and np.all(owner != fid)
        assert np.array_equal(glob_outer, g["outer"])
        lid2g = np.concatenate([np.arange(lo, hi), glob_outer])
        s_in = (src >= lo) & (src < hi)
        d_in = (dst >= lo) & (dst < hi)
        rp, col, fw = f.csr(0)
        _check_rows(rp, col, fw, lid2g, f.ivnum, lo, src[s_in], dst[s_in], wd[s_in], n)
        irp, icol, iw = f.csr(1)
        _check_rows(irp, icol, iw, lid2g, f.ivnum, lo, dst[d_in], src[d_in], wd[d_in], n)
        assert (f.oe_num, f.ie_num) == (int(s_in.sum()), int(d_in.sum()))
        oe_sum += f.oe_num
        ie_sum += f.ie_num
        # ov_ie: the transpose of the outer part of oe only
        vrp, vcol, _ = f.csr(2)
        rows = np.repeat(np.arange(f.ivnum, dtype=np.int64), np.diff(rp).astype(np.int64))
        is_outer = col >= f.ivnum
        pairs = np.stack([col[is_outer].astype(np.int64) - f.ivnum, rows[is_outer]], 1)
        pairs = pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))]
        vdeg = np.diff(vrp).astype(np.int64)
        assert np.array_equal(vdeg, np.bincount(pairs[:, 0], minlength=f.ovnum))
        assert np.array_equal(vcol.astype(np.int64), pairs[:, 1])
        only = np.isin(glob_outer, g["ie_only"])
        assert np.all(vdeg[only] == 0) and np.all(vdeg[~only] > 0)
        ie_only_rows += int(only.sum())
        f.close()
    assert oe_sum == len(src) and ie_sum == len(src)
    assert ie_only_rows > 0           # the split has outer vertices seen only through in-edges
