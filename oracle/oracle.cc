// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// A plain-C++ CPU restatement of the six LDBC apps of alibaba/libgrape-lite
// (reference @ e7c4465) used as the parity checker for the CUDA path.  Only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
// reference legs may load this library; the product (libgrape-lite_b200/)
// never does.
//
// Parity pin: every function below is checked against the reference's bundled
// golden vectors dataset/p2p-31-{BFS,BFS-directed,SSSP,SSSP-directed,PR,
// PR-directed,CDLP,LCC,WCC} (tests/test_oracle_golden.py, comparison rules of
// misc/app_tests.sh:6-40), and -- when oracle/_ref is built -- against the
// unmodified reference CPU apps on R-MAT graphs and on randomised multigraphs
// (tests/test_ref_golden.py).
//
// Citations are to files under /root/reference.
//
// Graph model.  Vertices are indexed 0..n-1 in ascending oid order (this is
// the lid order of a 1-fragment ImmutableEdgecutFragment:
// grape/fragment/basic_fragment_loader.h:95-105).  Rows are sorted by
// neighbour index (grape/graph/immutable_csr.h:104-131); multi-edges and self
// loops are kept; an undirected edge (u,v) adds v to row u AND u to row v,
// also when u == v (grape/fragment/csr_edgecut_fragment_base.h:462-478,
// parse_iter_out_undirected).
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

struct Csr {
  std::vector<uint64_t> rp;   // n+1
  std::vector<uint32_t> col;  // neighbour index
  std::vector<double> w;      // optional
};

struct Graph {
  int64_t n = 0;
  int directed = 0;
  std::vector<int64_t> oid;  // sorted ascending, size n
  Csr out;                   // out adjacency (undirected: the symmetrised one)
  Csr in;                    // directed only
  bool weighted = false;
};

void build_csr(int64_t n, int64_t m, const uint32_t* s, const uint32_t* d,
               const double* w, bool both, Csr& csr) {
  csr.rp.assign(n + 1, 0);
  for (int64_t i = 0; i < m; ++i) {
    csr.rp[s[i] + 1]++;
    if (both) csr.rp[d[i] + 1]++;
  }
  for (int64_t v = 0; v < n; ++v) csr.rp[v + 1] += csr.rp[v];
  uint64_t tot = csr.rp[n];
  csr.col.resize(tot);
  if (w) csr.w.resize(tot);
  std::vector<uint64_t> pos(csr.rp.begin(), csr.rp.end() - 1);
  for (int64_t i = 0; i < m; ++i) {
    uint64_t p = pos[s[i]]++;
    csr.col[p] = d[i];
    if (w) csr.w[p] = w[i];
    if (both) {
      p = pos[d[i]]++;
      csr.col[p] = s[i];
      if (w) csr.w[p] = w[i];
    }
  }
  // sort each row by neighbour index (stable on (col) only, as
  // immutable_csr.h:104-131 sorts Nbr by neighbour lid).
#pragma omp parallel
  {
    std::vector<std::pair<uint32_t, double>> tmp;
#pragma omp for schedule(dynamic, 1024)
    for (int64_t v = 0; v < n; ++v) {
      uint64_t b = csr.rp[v], e = csr.rp[v + 1];
      if (e - b < 2) continue;
      if (!w) {
        std::sort(csr.col.begin() + b, csr.col.begin() + e);
      } else {
        tmp.resize(e - b);
        for (uint64_t i = b; i < e; ++i) tmp[i - b] = {csr.col[i], csr.w[i]};
        std::stable_sort(tmp.begin(), tmp.end(),
                         [](const std::pair<uint32_t, double>& a,
                            const std::pair<uint32_t, double>& b2) {
                           return a.first < b2.first;
                         });
        for (uint64_t i = b; i < e; ++i) {
          csr.col[i] = tmp[i - b].first;
          csr.w[i] = tmp[i - b].second;
        }
      }
    }
  }
}

}  // namespace

extern "C" {

// Build from an edge list of oids. `oids` may be NULL, meaning oids = 0..n-1.
// Edges naming an oid that is not a vertex are dropped (the reference loader
// does the same: basic_fragment_loader.h ignores edges with unknown ends).
void* orc_graph_build(int64_t n, const int64_t* oids, int64_t m,
                      const int64_t* src, const int64_t* dst, const double* w,
                      int directed) {
  Graph* g = new Graph;
  g->n = n;
  g->directed = directed;
  g->oid.resize(n);
  if (oids) {
    std::copy(oids, oids + n, g->oid.begin());
    std::sort(g->oid.begin(), g->oid.end());
  } else {
    std::iota(g->oid.begin(), g->oid.end(), (int64_t) 0);
  }
  std::vector<uint32_t> s, d;
  std::vector<double> ww;
  s.reserve(m);
  d.reserve(m);
  if (w) ww.reserve(m);
  auto index_of = [&](int64_t o) -> int64_t {
    if (!oids) return (o >= 0 && o < n) ? o : -1;
    auto it = std::lower_bound(g->oid.begin(), g->oid.end(), o);
    if (it == g->oid.end() || *it != o) return -1;
    return it - g->oid.begin();
  };
  for (int64_t i = 0; i < m; ++i) {
    int64_t a = index_of(src[i]), b = index_of(dst[i]);
    if (a < 0 || b < 0) continue;
    s.push_back((uint32_t) a);
    d.push_back((uint32_t) b);
    if (w) ww.push_back(w[i]);
  }
  int64_t mm = (int64_t) s.size();
  g->weighted = w != nullptr;
  const double* wp = w ? ww.data() : nullptr;
  if (directed) {
    build_csr(n, mm, s.data(), d.data(), wp, false, g->out);
    build_csr(n, mm, d.data(), s.data(), wp, false, g->in);
  } else {
    build_csr(n, mm, s.data(), d.data(), wp, true, g->out);
  }
  return g;
}

void orc_graph_free(void* h) { delete (Graph*) h; }
int64_t orc_graph_n(void* h) { return ((Graph*) h)->n; }
uint64_t orc_graph_entries(void* h) { return ((Graph*) h)->out.rp.back(); }
const int64_t* orc_graph_oids(void* h) { return ((Graph*) h)->oid.data(); }
// raw CSR access (used by the fragment-layout parity test)
const uint64_t* orc_graph_rp(void* h, int in) {
  Graph* g = (Graph*) h;
  return in ? g->in.rp.data() : g->out.rp.data();
}
const uint32_t* orc_graph_col(void* h, int in) {
  Graph* g = (Graph*) h;
  return in ? g->in.col.data() : g->out.col.data();
}
const double* orc_graph_w(void* h, int in) {
  Graph* g = (Graph*) h;
  const Csr& c = in ? g->in : g->out;
  return c.w.empty() ? nullptr : c.w.data();
}
int64_t orc_graph_index_of(void* h, int64_t oid) {
  Graph* g = (Graph*) h;
  auto it = std::lower_bound(g->oid.begin(), g->oid.end(), oid);
  if (it == g->oid.end() || *it != oid) return -1;
  return it - g->oid.begin();
}
// vertex of maximum out-degree (ties -> smallest index); bench source rule
// (SURVEY.md §8(d)).
int64_t orc_graph_max_degree_vertex(void* h) {
  Graph* g = (Graph*) h;
  int64_t best = 0;
  uint64_t bd = 0;
  for (int64_t v = 0; v < g->n; ++v) {
    uint64_t dgr = g->out.rp[v + 1] - g->out.rp[v];
    if (dgr > bd) {
      bd = dgr;
      best = v;
    }
  }
  return best;
}

// ---------------------------------------------------------------- BFS ------
// examples/analytical_apps/bfs/bfs.h:44-212 (level-synchronous; PEval sets
// depth 0 / 1, IncEval expands curr_inner_updated; unreachable =
// numeric_limits<int64_t>::max(), bfs_context.h).  Directed graphs follow
// outgoing edges.  Returns the number of supersteps (levels expanded).
int orc_bfs(void* h, int64_t source_index, int64_t* depth) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  const int64_t INF = INT64_MAX;
  for (int64_t v = 0; v < n; ++v) depth[v] = INF;
  if (source_index < 0 || source_index >= n) return 0;
  std::vector<uint32_t> curr, next;
  depth[source_index] = 0;
  curr.push_back((uint32_t) source_index);
  int64_t d = 0;
  int steps = 0;
  const Csr& c = g->out;
  while (!curr.empty()) {
    next.clear();
    ++steps;
    for (uint32_t u : curr) {
      for (uint64_t e = c.rp[u]; e < c.rp[u + 1]; ++e) {
        uint32_t v = c.col[e];
        if (depth[v] == INF) {
          depth[v] = d + 1;
          next.push_back(v);
        }
      }
    }
    ++d;
    curr.swap(next);
  }
  return steps;
}

// --------------------------------------------------------------- SSSP ------
// examples/analytical_apps/sssp/sssp.h:51-169: frontier Bellman-Ford in fp64
// (run_app.cc:49 loads EDATA=double): PEval relaxes the source's edges,
// IncEval relaxes every vertex in curr_modified until no vertex changes.
// Unreachable = DBL_MAX (printed "infinity", sssp_context.h:60-70).
int orc_sssp(void* h, int64_t source_index, double* dist) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  for (int64_t v = 0; v < n; ++v) dist[v] = DBL_MAX;
  if (source_index < 0 || source_index >= n) return 0;
  const Csr& c = g->out;
  std::vector<uint8_t> in_next(n, 0);
  std::vector<uint32_t> curr, next;
  dist[source_index] = 0;
  curr.push_back((uint32_t) source_index);
  int steps = 0;
  while (!curr.empty()) {
    ++steps;
    next.clear();
    for (uint32_t v : curr) {
      double dv = dist[v];
      for (uint64_t e = c.rp[v]; e < c.rp[v + 1]; ++e) {
        uint32_t u = c.col[e];
        double nd = dv + (c.w.empty() ? 1.0 : c.w[e]);
        if (nd < dist[u]) {
          dist[u] = nd;
          if (!in_next[u]) {
            in_next[u] = 1;
            next.push_back(u);
          }
        }
      }
    }
    for (uint32_t u : next) in_next[u] = 0;
    curr.swap(next);
  }
  return steps;
}

// ---------------------------------------------------------------- WCC ------
// examples/analytical_apps/wcc/wcc.h:128-226: comp_id[v] = own id, then push
// min along outgoing (and, when directed, incoming) edges until fixpoint.
// Labels are the minimum vertex INDEX of the component; since indices are in
// ascending-oid order, oid[label] is the CPU app's min-oid label
// (wcc.h:139-153) and the index is the GPU app's min-gid label
// (cuda/wcc/wcc.h:110-111) for an order-preserving partitioner.
int orc_wcc(void* h, uint32_t* label) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  std::vector<uint8_t> in_next(n, 0);
  std::vector<uint32_t> curr(n), next;
  for (int64_t v = 0; v < n; ++v) {
    label[v] = (uint32_t) v;
    curr[v] = (uint32_t) v;
  }
  int steps = 0;
  auto relax = [&](const Csr& c, uint32_t u) {
    uint32_t lu = label[u];
    for (uint64_t e = c.rp[u]; e < c.rp[u + 1]; ++e) {
      uint32_t v = c.col[e];
      if (lu < label[v]) {
        label[v] = lu;
        if (!in_next[v]) {
          in_next[v] = 1;
          next.push_back(v);
        }
      }
    }
  };
  while (!curr.empty()) {
    ++steps;
    next.clear();
    for (uint32_t u : curr) {
      relax(g->out, u);
      if (g->directed) relax(g->in, u);
    }
    for (uint32_t v : next) in_next[v] = 0;
    curr.swap(next);
  }
  return steps;
}

// ----------------------------------------------------------- PageRank ------
// mode 0: examples/analytical_apps/pagerank/pagerank.h:52-154 (undirected
//   pull; result pre-divided by degree; base=(1-d)/N + d*dangling_sum/N;
//   dangling_sum_next = base * N_dangling; exactly max_round updates; final
//   multiply by degree).
// mode 1: examples/analytical_apps/cuda/pagerank/pagerank.h:137-249 restated
//   in fp64 (push; dangling sum from actual ranks; next = (1-d)/N +
//   d*dangling/N + sum_u d*rank[u]/deg[u]).
// mode 2: examples/analytical_apps/pagerank/pagerank_parallel.h:52-205
//   (directed; pulls along incoming edges; a vertex with out-degree 0 keeps
//   rank = base -- the reference's own quirk, pinned by p2p-31-PR-directed).
void orc_pagerank(void* h, double delta, int max_round, int mode,
                  double* rank) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  const Csr& oe = g->out;
  const Csr& ie = g->directed ? g->in : g->out;
  // max_round <= 0: pagerank.h:52-55 returns from PEval before it writes a
  // rank, so the CPU app prints its zero-initialised result; modes 1 and 2 run
  // their initialisation and return 1/N (pagerank_parallel.h:108-116 multiplies
  // the PEval values p/deg back by the degree in the first IncEval).
  if (max_round <= 0 && mode == 0) {
    for (int64_t v = 0; v < n; ++v) rank[v] = 0;
    return;
  }
  const double p = 1.0 / (double) n;
  std::vector<double> res(n), nxt(n);
  std::vector<int64_t> deg(n);
  int64_t dangling = 0;
  for (int64_t v = 0; v < n; ++v) {
    deg[v] = (int64_t) (oe.rp[v + 1] - oe.rp[v]);
    if (deg[v] == 0) ++dangling;
  }
  if (mode == 1) {
    for (int64_t v = 0; v < n; ++v) res[v] = p;
    for (int it = 0; it < max_round; ++it) {
      double ds = 0;
      for (int64_t v = 0; v < n; ++v)
        if (deg[v] == 0) ds += res[v];
      double base = (1.0 - delta) / (double) n + delta * ds / (double) n;
      for (int64_t v = 0; v < n; ++v) nxt[v] = base;
      for (int64_t u = 0; u < n; ++u) {
        if (!deg[u]) continue;
        double send = delta * res[u] / (double) deg[u];
        for (uint64_t e = oe.rp[u]; e < oe.rp[u + 1]; ++e)
          nxt[oe.col[e]] += send;
      }
      res.swap(nxt);
    }
    for (int64_t v = 0; v < n; ++v) rank[v] = res[v];
    return;
  }
  for (int64_t v = 0; v < n; ++v) res[v] = deg[v] > 0 ? p / (double) deg[v] : p;
  double dangling_sum = p * (double) dangling;
  for (int step = 1; step <= max_round; ++step) {
    double base =
        (1.0 - delta) / (double) n + delta * dangling_sum / (double) n;
    dangling_sum = base * (double) dangling;
#pragma omp parallel for schedule(dynamic, 1024)
    for (int64_t u = 0; u < n; ++u) {
      double cur = 0;
      for (uint64_t e = ie.rp[u]; e < ie.rp[u + 1]; ++e)
        cur += res[ie.col[e]];
      nxt[u] = deg[u] > 0 ? (delta * cur + base) / (double) deg[u] : base;
    }
    res.swap(nxt);
  }
  for (int64_t v = 0; v < n; ++v)
    rank[v] = deg[v] != 0 ? res[v] * (double) deg[v] : res[v];
}

// --------------------------------------------------------------- CDLP ------
// examples/analytical_apps/cdlp/cdlp.h:45-161 + cdlp_utils.h:35-73:
// labels = oid, synchronous; new label = most frequent label among the
// OUT-neighbours (multi-edges count), ties -> smallest label; vertices
// without out-edges keep their label; exactly max_round propagations.
void orc_cdlp(void* h, int max_round, int64_t* labels) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  const Csr& c = g->out;
  for (int64_t v = 0; v < n; ++v) labels[v] = g->oid[v];
  std::vector<int64_t> nl(n);
  for (int step = 1; step <= max_round; ++step) {
#pragma omp parallel
    {
      std::vector<int64_t> loc;
#pragma omp for schedule(dynamic, 1024)
      for (int64_t v = 0; v < n; ++v) {
        uint64_t b = c.rp[v], e = c.rp[v + 1];
        if (b == e) {
          nl[v] = labels[v];
          continue;
        }
        loc.clear();
        for (uint64_t i = b; i < e; ++i) loc.push_back(labels[c.col[i]]);
        std::sort(loc.begin(), loc.end());
        int64_t best = 0, cur = loc[0];
        int bc = 0, cc = 1;
        for (size_t i = 1; i < loc.size(); ++i) {
          if (loc[i] != loc[i - 1]) {
            if (cc > bc) {
              best = cur;
              bc = cc;
            }
            cur = loc[i];
            cc = 1;
          } else {
            ++cc;
          }
        }
        nl[v] = (cc > bc) ? cur : best;
      }
    }
    for (int64_t v = 0; v < n; ++v) labels[v] = nl[v];
  }
}

// ---------------------------------------------------------------- LCC ------
// examples/analytical_apps/lcc/lcc.h:48-233 + lcc_context.h:52-66 on an
// undirected graph: degree = CSR entries of the row (multi-edges count);
// orientation keeps u in N+(v) iff deg u < deg v, or equal degree and
// gid(v) > gid(u) (gid order = index order here); for every v, every u in
// N+(v) (with multiplicity), every w in N+(u) (with multiplicity): if w is in
// set(N+(v)) then tricnt[u,v,w] += 1; lcc = 2*tri/(d*(d-1)), 0 when d < 2.
// `tri` (optional) receives the integer triangle counters.
void orc_lcc(void* h, double* lcc, int64_t* tri_out) {
  Graph* g = (Graph*) h;
  const int64_t n = g->n;
  const Csr& c = g->out;
  std::vector<int64_t> deg(n);
  for (int64_t v = 0; v < n; ++v) deg[v] = (int64_t) (c.rp[v + 1] - c.rp[v]);
  std::vector<uint64_t> orp(n + 1, 0);
  for (int64_t v = 0; v < n; ++v) {
    uint64_t k = 0;
    for (uint64_t e = c.rp[v]; e < c.rp[v + 1]; ++e) {
      uint32_t u = c.col[e];
      if (deg[u] < deg[v] || (deg[u] == deg[v] && (uint32_t) v > u)) ++k;
    }
    orp[v + 1] = orp[v] + k;
  }
  std::vector<uint32_t> ocol(orp[n]);
  for (int64_t v = 0; v < n; ++v) {
    uint64_t k = orp[v];
    for (uint64_t e = c.rp[v]; e < c.rp[v + 1]; ++e) {
      uint32_t u = c.col[e];
      if (deg[u] < deg[v] || (deg[u] == deg[v] && (uint32_t) v > u))
        ocol[k++] = u;
    }
  }
  std::vector<int64_t> tri(n, 0);
#pragma omp parallel for schedule(dynamic, 256)
  for (int64_t v = 0; v < n; ++v) {
    const uint32_t* vb = ocol.data() + orp[v];
    const uint32_t* ve = ocol.data() + orp[v + 1];
    for (const uint32_t* pu = vb; pu != ve; ++pu) {
      uint32_t u = *pu;
      for (uint64_t e = orp[u]; e < orp[u + 1]; ++e) {
        uint32_t w = ocol[e];
        if (std::binary_search(vb, ve, w)) {
#pragma omp atomic
          tri[u]++;
#pragma omp atomic
          tri[v]++;
#pragma omp atomic
          tri[w]++;
        }
      }
    }
  }
  for (int64_t v = 0; v < n; ++v) {
    if (tri_out) tri_out[v] = tri[v];
    if (deg[v] < 2) {
      lcc[v] = 0.0;
    } else {
      lcc[v] = 2.0 * (double) tri[v] / (double) (deg[v] * (deg[v] - 1));
    }
  }
}

int orc_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

}  // extern "C"
