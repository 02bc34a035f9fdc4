"""Host model of `gl_frag_desc` for any partition of a graph into fragments.

The library's own builders (`gl_frag_build_from_edges`, `gl_frag_build_rmat`) cut the vertices into
contiguous blocks of ceil(n / fnum) ascending oids and number each block in oid order.  A host that
calls `gl_frag_create` may partition and number the vertices any way it likes; the reference's edge-file
loader, for one, hashes every vertex to fid `oid % fnum` and numbers them in order of first appearance
in the edge list (grape/fragment/basic_efile_fragment_loader.h, grape/vertex_map/partitioner.h).

Here a partition is two arrays over the vertex indices 0..n-1 of a graph: `owner[v]`, the fid that holds
v, and `key[v]`: inside each fragment the lids follow ascending `key`.  `describe` turns a graph and a
partition into what every fid passes to `gl_frag_create`, meeting the header's preconditions: rows in lid
order, each row sorted by neighbour lid (so inner neighbours first), outer lids in ascending gid order.
It also returns the gid rank of every vertex, `off[fid] + lid` with `off` the prefix sum of the ivnums:
the vertex's position in gid order, which is the order the apps break label ties in.

Plain numpy; every rank of a fragment group computes the same partition from the same seeds."""
import numpy as np

SEED = 20261017


def fid_offset(fnum):
    """IdParser::fid_offset_ of the library (gid = fid << fid_offset | lid)."""
    return 31 if fnum == 1 else 32 - int(fnum - 1).bit_length()


# ------------------------------------------------------------------ partitions --------------------------------
def blocks(n, fnum):
    """The library's builders: contiguous blocks of ceil(n / fnum) indices, lids in index order."""
    chunk = max(-(-n // fnum), 1)
    return np.arange(n, dtype=np.int64) // chunk, np.arange(n, dtype=np.int64)


def first_appearance(n, src, dst):
    """Position of every vertex in the order it first appears over (src[0], dst[0], src[1], dst[1], ...);
    vertices without edges come last, in index order."""
    seq = np.stack([np.asarray(src, np.int64), np.asarray(dst, np.int64)], 1).ravel()
    seen, first = np.unique(seq, return_index=True)
    key = np.full(n, len(seq), dtype=np.int64) + np.arange(n)
    key[seen] = first
    out = np.empty(n, dtype=np.int64)
    out[np.argsort(key, kind="stable")] = np.arange(n)
    return out


def hash_owner(oids, fnum):
    """HashPartitioner with libstdc++'s std::hash<int64_t> (the identity): fid = size_t(oid) % fnum."""
    return (np.asarray(oids, np.int64).astype(np.uint64) % np.uint64(fnum)).astype(np.int64)


def hash_part(n, src, dst, oids, fnum):
    """The reference's edge-file loader: `oid % fnum`, lids in order of first appearance."""
    return hash_owner(oids, fnum), first_appearance(n, src, dst)


def map_sizes(vnum, fnum):
    """MapPartitioner::Init(fnum, oid_list): list position i goes to fid i / ceil(vnum / fnum)."""
    per = max(-(-vnum // fnum), 1)
    return np.bincount(np.arange(vnum) // per, minlength=fnum)


def map_part(n, fnum, seed=SEED):
    """MapPartitioner::Init over a seeded permutation of the vertex list; lids in list order."""
    perm = np.random.default_rng([seed, n, fnum]).permutation(n)
    per = max(-(-n // fnum), 1)
    owner = np.empty(n, dtype=np.int64)
    key = np.empty(n, dtype=np.int64)
    owner[perm] = np.arange(n) // per
    key[perm] = np.arange(n)
    return owner, key


def degrees(n, src, dst):
    return np.bincount(np.concatenate([np.asarray(src, np.int64), np.asarray(dst, np.int64)]), minlength=n)


def skew_part(n, src, dst, oids, fnum, hubs=16, seed=SEED):
    """The `hubs` highest-degree vertices (ties: smaller oid) alone in fid fnum-1, the rest by
    oid % (fnum-1); lids in a seeded permutation."""
    assert fnum >= 2
    deg = degrees(n, src, dst)
    top = np.lexsort((np.asarray(oids, np.int64), -deg))[:hubs]
    owner = hash_owner(oids, fnum - 1)
    owner[top] = fnum - 1
    return owner, np.random.default_rng([seed, n, fnum, 1]).permutation(n).astype(np.int64)


def hollow_part(n, oids, fnum=3, empty_fid=1, seed=SEED):
    """No vertex on fid `empty_fid`: the vertices are hashed over the other fids; lids in a seeded
    permutation."""
    others = np.array([f for f in range(fnum) if f != empty_fid], dtype=np.int64)
    owner = others[hash_owner(oids, len(others))]
    return owner, np.random.default_rng([seed, n, fnum, 2]).permutation(n).astype(np.int64)


def partition(name, n, src, dst, oids, fnum):
    if name == "blocks":
        return blocks(n, fnum)
    if name == "hash":
        return hash_part(n, src, dst, oids, fnum)
    if name == "map":
        return map_part(n, fnum)
    if name == "skew":
        return skew_part(n, src, dst, oids, fnum)
    if name == "hollow":
        return hollow_part(n, oids, fnum)
    raise KeyError(name)


# ------------------------------------------------------------------ descriptors -------------------------------
class Layout:
    """`describe`'s result.  Per vertex index: owner, lid, gid, rank (gid rank).  `frags[fid]` is a dict
    with ivnum, ovnum, total_vnum, oe = (rp, col, w), ie = (rp, col, w) or None, ovgid (uint32),
    inner_oids (lid order), inner (vertex indices in lid order), ovie = (rp, col), the transpose of the
    outer part of oe, and outer (vertex indices of the outer lids)."""

    def __init__(self, n, fnum, owner, lid, gid, rank, frags):
        self.n, self.fnum = n, fnum
        self.owner, self.lid, self.gid, self.rank, self.frags = owner, lid, gid, rank, frags
        self.by_rank = np.empty(n, dtype=np.int64)
        self.by_rank[rank] = np.arange(n)

    def global_csr(self):
        """The fragments' oe rows, concatenated in fid order, with every neighbour written as its gid rank
        (each row keeps the fragment's entry order)."""
        rps, cols = [], []
        for f in self.frags:
            rp, col, _ = f["oe"]
            lid2v = np.concatenate([f["inner"], f["outer"]]).astype(np.int64)
            rps.append(np.diff(rp.astype(np.int64)))
            cols.append(self.rank[lid2v[col.astype(np.int64)]])
        rp = np.concatenate([[0], np.cumsum(np.concatenate(rps))]).astype(np.int64)
        return rp, np.concatenate(cols).astype(np.int64)


def _csr(rows, cols, w, nrows):
    order = np.lexsort((cols, rows))
    rp = np.zeros(nrows + 1, dtype=np.uint64)
    rp[1:] = np.cumsum(np.bincount(rows, minlength=nrows))
    return rp, cols[order].astype(np.uint32), None if w is None else w[order]


def describe(n, src, dst, w, oids, directed, owner, key, fnum):
    """Every fid's gl_frag_desc for the graph (src, dst: vertex indices; w: per-edge weights or None;
    oids: per vertex index) cut by (owner, key)."""
    src = np.asarray(src, np.int64)
    dst = np.asarray(dst, np.int64)
    oids = np.asarray(oids, np.int64)
    owner = np.asarray(owner, np.int64)
    assert len(owner) == n and owner.min(initial=0) >= 0 and owner.max(initial=0) < fnum
    fo = fid_offset(fnum)
    lid = np.empty(n, dtype=np.int64)
    inner = []
    for f in range(fnum):
        vs = np.flatnonzero(owner == f)
        vs = vs[np.argsort(key[vs], kind="stable")]
        lid[vs] = np.arange(len(vs))
        inner.append(vs)
    ivnums = np.array([len(v) for v in inner], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(ivnums)])
    gid = (owner << fo) | lid
    rank = off[owner] + lid
    if directed:
        csrs = {"oe": (src, dst, w), "ie": (dst, src, w)}
    else:
        csrs = {"oe": (np.concatenate([src, dst]), np.concatenate([dst, src]),
                       None if w is None else np.concatenate([w, w]))}
    frags = []
    for f in range(fnum):
        iv = int(ivnums[f])
        mine = {k: owner[r] == f for k, (r, _, _) in csrs.items()}
        nbs = np.concatenate([csrs[k][1][mine[k]] for k in csrs])
        outer = np.unique(nbs[owner[nbs] != f])
        outer = outer[np.argsort(gid[outer], kind="stable")]
        local = np.empty(n, dtype=np.int64)
        local[inner[f]] = np.arange(iv)
        local[outer] = iv + np.arange(len(outer))
        d = {"fid": f, "ivnum": iv, "ovnum": len(outer), "total_vnum": n, "inner": inner[f], "outer": outer,
             "inner_oids": oids[inner[f]], "ovgid": gid[outer].astype(np.uint32), "ie": None}
        for k, (r, c, ww) in csrs.items():
            sel = mine[k]
            d[k] = _csr(lid[r[sel]], local[c[sel]], None if ww is None else ww[sel], iv)
        rp, col, _ = d["oe"]
        rows = np.repeat(np.arange(iv), np.diff(rp.astype(np.int64)))
        out = col.astype(np.int64) >= iv
        o_rp, o_col, _ = _csr(col[out].astype(np.int64) - iv, rows[out], None, len(outer))
        d["ovie"] = (o_rp, o_col)
        frags.append(d)
    return Layout(n, fnum, owner, lid, gid, rank, frags)


def from_layout(pkg, layout, fid, directed):
    """Creates fragment `fid` of a layout through gl_frag_create (Fragment.from_csr)."""
    d = layout.frags[fid]
    rp, col, w = d["oe"]
    ie = d["ie"] if directed else None
    return pkg.Fragment.from_csr(d["ivnum"], rp, col, w, ovgid=d["ovgid"] if d["ovnum"] else None,
                                 total_vnum=layout.n, fid=fid, fnum=layout.fnum, directed=directed, ie=ie,
                                 inner_oids=d["inner_oids"])


def same_weights(rp, col, w_a, w_b):
    """Weights equal as multisets per (row, col): duplicate edges may carry different weights in any order."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(np.asarray(rp, np.int64)))
    a = np.lexsort((np.asarray(w_a, np.float64), col, rows))
    b = np.lexsort((np.asarray(w_b, np.float64), col, rows))
    return np.array_equal(np.asarray(w_a, np.float64)[a], np.asarray(w_b, np.float64)[b])


def min_label_wcc(n, src, dst, order):
    """Weakly connected components labelled by the member with the smallest `order` value; returns the
    label's vertex index per vertex (plain union-find)."""
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for a, b in zip(np.asarray(src, np.int64), np.asarray(dst, np.int64)):
        ra, rb = find(a), find(b)
        if ra != rb:
            if order[ra] < order[rb]:
                parent[rb] = ra
            else:
                parent[ra] = rb
    return np.array([find(v) for v in range(n)], dtype=np.int64)
