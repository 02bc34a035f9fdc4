"""Host model of the query statistics (gl_query_stats) — TEST INFRASTRUCTURE ONLY.

Plain level-synchronous numpy code over a CSR (row pointers `rp`, columns `col`, the
arrays pyoracle.Graph.csr() and Fragment.csr(0) return): what each app must report in
entries_scanned, frontier_vertices, touched_vertices, supersteps and the per-step
arrays.  It is the executable form of the "Query statistics" text beside
gl_query_stats in include/grape_b200.h; nothing here looks at how a kernel counts.

Step index: step 0 is PEval; the k-th set of counters an app records (k = 0, 1, ...)
is reported as step k + 1.  Every function returns a Stats whose step arrays are
already laid out that way (index 0 is PEval's, all zero unless said otherwise).

Fragments: fragment `fid` of `fnum` owns the contiguous block of vertices
[fid * chunk, min(n, (fid + 1) * chunk)), chunk = ceil(n / fnum), as the fragment
builders partition.  With fnum > 1 the functions return that fragment's share: the
rows it owns; the shares of all fragments add up to the one-fragment values.
"""
import numpy as np

GL_MAX_STEP_STATS = 512
PUSH, PULL, DENSE = 0, 1, 2


class Stats:
    """supersteps and totals of one query, and the per-step lists (index = step)."""

    def __init__(self, supersteps, step_entries, step_frontier, step_mode, touched):
        self.supersteps = int(supersteps)
        self.step_entries = [int(x) for x in step_entries]
        self.step_frontier = [int(x) for x in step_frontier]
        self.step_mode = [int(x) for x in step_mode]
        self.entries_scanned = sum(self.step_entries)
        self.frontier_vertices = sum(self.step_frontier)
        self.touched_vertices = None if touched is None else int(touched)
        self.n_steps = min(self.supersteps, GL_MAX_STEP_STATS)

    def __repr__(self):
        return ("Stats(supersteps=%d entries=%d frontier=%d touched=%d step_entries=%s step_frontier=%s step_mode=%s)"
                % (self.supersteps, self.entries_scanned, self.frontier_vertices, self.touched_vertices,
                   self.step_entries[:12], self.step_frontier[:12], self.step_mode[:12]))


def fragment_range(n, fid=0, fnum=1):
    """[first, last) of the vertices fragment fid of fnum owns."""
    chunk = (n + fnum - 1) // fnum if n else 0
    return min(n, fid * chunk), min(n, (fid + 1) * chunk)


def _degrees(rp):
    return np.diff(np.asarray(rp, dtype=np.int64))


def _own(n, fid, fnum):
    lo, hi = fragment_range(n, fid, fnum)
    own = np.zeros(n, dtype=bool)
    own[lo:hi] = True
    return own


def bfs_levels(rp, col, source):
    """The BFS levels from vertex index `source` (None: not in the graph): a list of
    sorted vertex arrays, level d = the vertices at depth d."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    n = len(rp) - 1
    if source is None:
        return []
    seen = np.zeros(n, dtype=bool)
    seen[source] = True
    level = np.array([source], dtype=np.int64)
    levels = []
    while len(level):
        levels.append(level)
        lens = rp[level + 1] - rp[level]
        starts = np.repeat(rp[level] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
        nbrs = col[starts + np.arange(int(lens.sum()), dtype=np.int64)]
        nxt = np.unique(nbrs)
        nxt = nxt[~seen[nxt]]
        seen[nxt] = True
        level = nxt
    return levels


def bfs_push(rp, col, source, fid=0, fnum=1):
    """BFS with direction_opt = 0.  Step i >= 1 expands level i - 1: step_frontier =
    the level's size, step_entries = the row lengths of the level, mode push.  The
    step that expands the last level finds nothing and ends the query, so
    supersteps = levels + 1.  touched_vertices = vertices given a depth by an
    expansion: every reached vertex but the source (one fragment; on several the count also covers
    outer copies a fragment reaches and is not modelled: None).
    A source that is not in the graph: one superstep (PEval), all counters zero."""
    deg = _degrees(rp)
    n = len(deg)
    own = _own(n, fid, fnum)
    levels = bfs_levels(rp, col, source)
    ent = [0] + [int(deg[l[own[l]]].sum()) for l in levels]
    fro = [0] + [int(own[l].sum()) for l in levels]
    reached = sum(len(l) for l in levels)
    steps = len(levels) + 1
    return Stats(steps, ent, fro, [PUSH] * steps, max(reached - 1, 0) if fnum == 1 else None)


def bfs_direction_modes(level_sizes, level_entries, m_total, vnum, nz_total, beta=24):
    """The push / pull choice of every level of a direction-optimising BFS that knows
    the exact entry counts and keeps the per-frontier tail rule (the stepwise query
    on one fragment).  A restatement of the library's own rule (bfs_next_phase), not an
    independent derivation: comparing step_mode with it shows that the query feeds the
    rule the level sizes, entry counts and unvisited totals defined here.  With n_f / m_f the vertices / CSR entries of the level to
    expand, m_u the entries of the rows not yet reached and `unvisited` the vertices
    with at least one entry not yet reached:
      * in the initial push phase a level is pulled once m_f > m_u / 14;
      * a pull phase goes on while n_f >= floor(vnum / beta) (written
        (n_f + 1) * beta > vnum) or while unvisited <= 64 * n_f;
      * after that every level is pushed."""
    modes, phase = [], 0
    seen_entries, seen_cnt = 0, 0
    for n_f, m_f in zip(level_sizes, level_entries):
        seen_entries += m_f
        seen_cnt += n_f
        m_u = max(m_total - seen_entries, 0)
        unvisited = max(nz_total - seen_cnt, 0)
        if phase == 0:
            phase = 1 if m_f > m_u // 14 else 0
        elif phase == 1:
            if not ((n_f + 1) * beta > vnum or unvisited <= 64 * n_f):
                phase = 2
        modes.append(PULL if phase == 1 else PUSH)
    return modes


def bfs_pull_bounds(rp, col, source):
    """Per level d: (vertices of level d + 1, entries a pull step over level d may read at most).
    A pull step reads at least one entry per vertex it finds; every vertex with a non-empty row
    that is unlabelled when the step begins costs at most one probe of its highest-degree
    neighbour plus its whole row."""
    deg = _degrees(rp)
    levels = bfs_levels(rp, col, source)
    left, left_rows = int(deg.sum()), int(np.count_nonzero(deg))
    out = []
    for d, l in enumerate(levels):
        left -= int(deg[l].sum())
        left_rows -= int(np.count_nonzero(deg[l]))
        found = len(levels[d + 1]) if d + 1 < len(levels) else 0
        out.append((found, left + left_rows))
    return out


def dense_rounds(rp, rounds, final_rounds, fid=0, fnum=1):
    """An app of `rounds` dense rounds: each one reads every CSR entry of the
    fragment's rows once and writes every inner vertex once (step_frontier = ivnum,
    mode dense); `final_rounds` more supersteps follow that read nothing (the round
    that notices max_round is reached)."""
    deg = _degrees(rp)
    lo, hi = fragment_range(len(deg), fid, fnum)
    m, iv = int(deg[lo:hi].sum()), hi - lo
    steps = 1 + rounds + final_rounds
    pad = [0] * final_rounds
    return Stats(steps, [0] + [m] * rounds + pad, [0] + [iv] * rounds + pad, [0] + [DENSE] * rounds + pad, iv * rounds)


def pagerank(rp, max_round, fid=0, fnum=1):
    """PageRank, push or pull, f32 or f64 gather: PEval sets 1/N, rounds 1..max_round
    each read the whole CSR, and one more superstep ends the query:
    supersteps = max_round + 2."""
    return dense_rounds(rp, max_round, 1, fid, fnum)


def cdlp(rp, max_round, fid=0, fnum=1):
    """CDLP: round 1 runs inside PEval (its counters are step 1's, by the step-index
    rule), rounds 2..max_round in the following supersteps, and the superstep that
    sees max_round reached ends the query: supersteps = max_round + 1 (1 when
    max_round = 0)."""
    return dense_rounds(rp, max_round, 0, fid, fnum)


def lcc(rp, col):
    """LCC on one fragment: PEval builds the degree-ordered DAG N+ (u in N+(v) when
    deg u < deg v, or the degrees tie and u < v; one entry per CSR entry), step 1
    counts triangles: for every DAG entry (v, u) it reads the DAG row of u.  Step 2
    ends the query."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    deg = _degrees(rp)
    n = len(deg)
    row = np.repeat(np.arange(n, dtype=np.int64), deg)
    keep = (deg[col] < deg[row]) | ((deg[col] == deg[row]) & (row > col))
    out_deg = np.bincount(row[keep], minlength=n)
    entries = int(out_deg[col[keep]].sum())
    return Stats(3, [0, entries, 0], [0, n, 0], [0, DENSE, 0], n)


def kcore_entries(rp, value, k):
    """k-core on one fragment: one step; the peel reads the whole row of every vertex
    it removes: the vertices whose result value is below k."""
    deg = _degrees(rp)
    return int(deg[np.asarray(value) < k].sum())


def bfs_push_cut_items(rp, col, source, fid, fnum):
    """Vertices fragment fid reports to their owners during a push-only BFS: a fragment learns that an
    outer vertex is visited only by reaching it itself, so it reports, once, every vertex it does not own
    that has an entry in the row of one of its reached vertices."""
    rp = np.asarray(rp, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    own = _own(len(rp) - 1, fid, fnum)
    levels = bfs_levels(rp, col, source)
    if not levels:
        return 0
    mine = np.concatenate(levels)
    mine = mine[own[mine]]
    lens = rp[mine + 1] - rp[mine]
    starts = np.repeat(rp[mine] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    nbrs = np.unique(col[starts + np.arange(int(lens.sum()), dtype=np.int64)])
    return int(np.count_nonzero(~own[nbrs]))
