// app_bc.cu — single-source betweenness centrality on an undirected graph.
//
// Behaviour follows examples/analytical_apps/bc/staged_bc_bfs.h then bc/staged_bc.h
// (CPU apps sharing one BCContext, LoadStrategy::kOnlyOut).  Per vertex: depth
// (BFS level from the source), sigma (f64 number of shortest paths) and c (f32
// centrality).
//  * sigma(s) = 1; every depth-1 vertex has sigma = 1 however many parallel edges
//    join it to s; a vertex at depth d >= 2 has sigma = sum of sigma(u) over the
//    entries (v, u) of its row with depth(u) = d - 1 (one term per copy of a
//    parallel edge; a self loop never qualifies).
//  * Backward, level d = L .. 0: cacc = f32(sum of double(t[v]) over the entries
//    (u, v) of u's row with depth(v) = d + 1); d > 0: c = f32(double(cacc) * sigma),
//    t = f32((1.0 / sigma) * (1.0 + double(c))); the source keeps c = cacc.
// Every sum is a gather over the vertex's own row in a fixed order: a row of up
// to kBcShort entries is summed sequentially by one thread; a longer row is cut
// into kBcChunk-entry chunks, a warp sums a chunk with lane stride 32 and a fixed
// shuffle tree, and the chunk sums are added in chunk order.  The same graph
// therefore gives bit-identical results on every run; sigma is exact (and equal
// to the reference's) while it stays below 2^53.
//
//  * One fragment: the whole query is ONE cooperative launch (k_bc_fused).  The
//    reached vertices are kept in one level list (vertices grouped by level, level
//    offsets in `loff`).  Forward level d: discovery (push: CAS on the depth of the
//    neighbours of the level d-1 list through queue_scan_phase / hub_scan_phase;
//    pull: unvisited vertices probe their rows up to the first level d-1
//    neighbour), grid.sync, then the sigma gather over the level d list.  Backward:
//    one gather over each level's list, deepest first.  No step sweeps all
//    vertices except a pull discovery.
//  * Several fragments: one level per superstep through the worker loop, pull
//    only: every unvisited inner vertex gathers over its whole row, inner and
//    outer entries alike; the outer copies' depth / sigma / t are refreshed by
//    the dense mirror sync before each step, and the level size is all-reduced.
#include <cooperative_groups.h>

#include "apps_common.cuh"

namespace gl {
namespace {

namespace cg = cooperative_groups;

constexpr uint32_t kBcUnvis = 0xFFFFFFFFu;
constexpr uint32_t kBcShort = 32;     // rows up to this length: one thread, sequential sum
constexpr uint32_t kBcChunk = 1024;   // longer rows: chunks of this many entries, one warp per chunk
constexpr int kBcMaxStat = GL_MAX_STEP_STATS;
#define GL_BC_FUSED_CTAS 4

GL_DEV unsigned long long bc_global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// append v to q among the currently active lanes (one atomic per warp)
GL_DEV void bc_append_active(uint32_t* q, unsigned int* n, uint32_t v) {
  const uint32_t m = __activemask();
  const uint32_t leader = __ffs(m) - 1;
  uint32_t base = 0;
  if (lane_id() == leader) base = atomicAdd(n, (unsigned int) __popc(m));
  base = __shfl_sync(m, base, leader);
  q[base + __popc(m & ((1u << lane_id()) - 1))] = v;
}

// t of a vertex below the deepest level, from its gathered sum (staged_bc.h:59-63)
GL_DEV void bc_finish_back(uint32_t u, double s, bool source, const double* sigma, float* c, float* t) {
  const float cacc = (float) s;
  if (source) {   // the source is never multiplied
    c[u] = cacc;
    return;
  }
  const double sg = __ldcg(sigma + u);
  const float cv = (float) ((double) cacc * sg);
  c[u] = cv;
  t[u] = (float) ((1.0 / sg) * (1.0 + (double) cv));
}

// The two gathers.  term(v): the contribution of one row entry; finish(u, s): the vertex's result.
struct GatherSigma {   // level d >= 2: sigma[u] = sum of sigma[v] with depth[v] = d - 1
  const uint32_t* depth;
  double* sigma;
  uint32_t prev;
  GL_DEV double term(uint32_t v) const { return __ldcg(depth + v) == prev ? __ldcg(sigma + v) : 0.0; }
  GL_DEV void finish(uint32_t u, double s) const { sigma[u] = s; }
};
struct GatherBack {    // level d: sum of t[v] with depth[v] = d + 1
  const uint32_t* depth;
  const double* sigma;
  float* t;
  float* c;
  uint32_t next;
  bool source_level;
  GL_DEV double term(uint32_t v) const { return __ldcg(depth + v) == next ? (double) __ldcg(t + v) : 0.0; }
  GL_DEV void finish(uint32_t u, double s) const { bc_finish_back(u, s, source_level, sigma, c, t); }
};

// push discovery: the first CAS on an unvisited endpoint appends it to the level list
struct OpBcDiscover {
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* depth;
  uint32_t* out;
  unsigned int* out_n;
  uint32_t d;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  GL_DEV void edge(uint32_t, Meta, uint32_t v, W, ScanAcc& acc) const {
    if (__ldcg(depth + v) != kBcUnvis) return;
    if (atomicCAS(depth + v, kBcUnvis, d) != kBcUnvis) return;
    bc_append_active(out, out_n, v);
    acc.next_count++;
  }
};

// ---------------------------------------------------------------------------
// One fragment: the whole query in one cooperative launch.
// ---------------------------------------------------------------------------
struct BcLong {   // a long row of a gather: its chunks are [base, base + n) of the chunk arrays
  uint32_t v, base, n, pad;
};

// Counters of one step.  Step t uses c[t % 3]; thread 0 zeroes c[(t + 2) % 3] after the grid.sync that
// ends step t, one grid.sync before step t + 2 uses it.
struct BcStep {
  ScanCtrl sc;                 // push discovery
  unsigned int found;          // vertices appended to the level list
  unsigned int nlong, nchunk;  // long rows of the gather and their chunks
  unsigned int pad;
  unsigned long long m_lvl;    // row entries of the level's vertices
  unsigned long long scanned;  // entries read by the pull probes and the gather
};
struct BcFusedCtl {
  BcStep c[3];
  unsigned long long levels;   // levels 0..L of the forward pass: L + 1 (0: the source is absent)
  unsigned long long reached, scanned, fwd_ns, bwd_ns;
  unsigned long long fscan[kBcMaxStat], bscan[kBcMaxStat];   // entries read per forward / backward level
  unsigned char mode[kBcMaxStat];                             // forward level: 0 push, 1 pull discovery
};

struct BcFusedArgs {
  EdgeRange er;
  uint32_t n;
  uint32_t src;   // kBcUnvis: not in this fragment
  unsigned long long m;
  int direction_opt;
  uint32_t* depth;
  double* sigma;
  float* t;
  float* c;
  uint32_t* list;   // [n]: the reached vertices grouped by level
  uint32_t* loff;   // [n + 2]: level d is list[loff[d], loff[d + 1])
  BcLong* lng;      // [n]
  uint32_t* chunk_item;   // [chunk_cap]: the long row a chunk belongs to
  double* part;           // [chunk_cap]: chunk sums
  BcFusedCtl* ctl;
  HubItem* hubs;
  uint32_t hub_cap, hub_deg;
};

GL_DEV uint32_t row_len(const uint64_t* rp, uint32_t v) { return (uint32_t) (rp[v + 1] - rp[v]); }

// Gather over the level list [b, e): rows of up to kBcShort entries are summed by one thread; longer ones are
// registered as chunks, summed per chunk by a warp, and the chunk sums added in chunk order.  Ends without a
// trailing grid.sync; the caller's end of step provides it.
template <class G>
GL_DEV void gather_level(cg::grid_group& grid, const BcFusedArgs& a, const G& g, uint32_t b, uint32_t e,
                         BcStep* C, uint32_t gtid, uint32_t nthr) {
  const uint64_t* rp = a.er.rp;
  const uint32_t* col = a.er.col;
  unsigned long long scanned = 0, m_lvl = 0;
  for (uint32_t i = b + gtid; i < e; i += nthr) {
    const uint32_t u = a.list[i];
    const uint64_t r0 = rp[u], r1 = rp[u + 1];
    const uint32_t deg = (uint32_t) (r1 - r0);
    m_lvl += deg;
    if (deg <= kBcShort) {
      double s = 0.0;
      for (uint64_t j = r0; j < r1; ++j) s += g.term(col[j]);
      scanned += deg;
      g.finish(u, s);
    } else {
      const uint32_t nc = (deg + kBcChunk - 1) / kBcChunk;
      const uint32_t item = atomicAdd(&C->nlong, 1u);
      const uint32_t base = atomicAdd(&C->nchunk, nc);
      a.lng[item] = BcLong{u, base, nc, 0};
      for (uint32_t k = 0; k < nc; ++k) a.chunk_item[base + k] = item;
    }
  }
  grid.sync();
  const uint32_t nchunk = ((volatile BcStep*) C)->nchunk;
  if (nchunk) {
    const uint32_t nwarps = nthr >> 5;
    for (uint32_t ck = gtid >> 5; ck < nchunk; ck += nwarps) {
      const BcLong L = a.lng[a.chunk_item[ck]];
      const uint64_t c0 = rp[L.v] + (uint64_t) (ck - L.base) * kBcChunk;
      const uint64_t c1 = min(c0 + kBcChunk, rp[L.v + 1]);
      double s = 0.0;
      for (uint64_t j = c0 + lane_id(); j < c1; j += 32) s += g.term(col[j]);
      s = warp_sum(s);   // xor butterfly: every lane ends with the same, order-fixed sum
      if (lane_id() == 0) {
        a.part[ck] = s;
        scanned += c1 - c0;
      }
    }
    grid.sync();
    const uint32_t nlong = ((volatile BcStep*) C)->nlong;
    for (uint32_t i = gtid; i < nlong; i += nthr) {
      const BcLong L = a.lng[i];
      double s = 0.0;
      for (uint32_t k = 0; k < L.n; ++k) s += __ldcg(a.part + L.base + k);
      g.finish(L.v, s);
    }
  }
  scanned = warp_sum(scanned);
  m_lvl = warp_sum(m_lvl);
  if (lane_id() == 0) {
    if (scanned) atomicAdd(&C->scanned, scanned);
    if (m_lvl) atomicAdd(&C->m_lvl, m_lvl);
  }
}

__global__ void __launch_bounds__(kTB, GL_BC_FUSED_CTAS) k_bc_fused(BcFusedArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ ScanSmem<uint32_t> sm;
  __shared__ uint32_t s_item;
  BcFusedCtl* ctl = a.ctl;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nthr = gridDim.x * blockDim.x;
  uint32_t t = 0;
  auto end_step = [&]() {
    grid.sync();
    if (gtid == 0) ctl->c[(t + 2) % 3] = BcStep();
    ++t;
  };
  const unsigned long long t0 = gtid == 0 ? bc_global_ns() : 0;
  const bool has_src = a.src != kBcUnvis;
  if (gtid == 0) {
    a.loff[0] = 0;
    a.loff[1] = has_src ? 1 : 0;
    if (has_src) {
      a.depth[a.src] = 0;
      a.sigma[a.src] = 1.0;
      a.list[0] = a.src;
    }
  }
  end_step();
  if (!has_src) return;   // nothing is reached; every count in ctl stays 0
  // forward: level d + 1 from level d = list[lb, le)
  uint32_t d = 0, lb = 0, le = 1, phase = 0;
  unsigned long long m_f = row_len(a.er.rp, a.src), visited_m = m_f;
  for (;;) {
    const uint32_t n_f = le - lb;
    if (a.direction_opt) {
      // Beamer's rule, as the BFS app: pull while the frontier's entries outweigh the unvisited ones
      if (phase == 0) phase = m_f > (a.m - visited_m) / 14 ? 1u : 0u;
      else phase = (unsigned long long) (n_f + 1) * 24 > a.n ? 1u : 0u;
    }
    BcStep* C = &ctl->c[t % 3];
    uint32_t* out = a.list + le;
    const uint32_t nd = d + 1;
    unsigned long long pscan = 0;
    if (phase == 0) {
      OpBcDiscover op{a.depth, out, &C->found, nd};
      ScanAcc acc;
      queue_scan_phase<OpBcDiscover>(sm, ArraySrc{a.list + lb}, n_f, a.er, op, &C->sc, a.hubs, a.hub_cap,
                                     a.hub_deg, acc);
      grid.sync();
      hub_scan_phase<OpBcDiscover>(&s_item, a.er, op, &C->sc, a.hubs, a.hub_cap, acc);
    } else {
      // pull: an unvisited vertex probes its row up to the first level-d neighbour
      for (uint32_t base = blockIdx.x * blockDim.x; base < a.n; base += nthr) {   // warp-uniform bound
        const uint32_t v = base + threadIdx.x;
        bool hit = false;
        if (v < a.n && __ldcg(a.depth + v) == kBcUnvis) {
          const uint64_t r1 = a.er.rp[v + 1];
          for (uint64_t j = a.er.rp[v]; j < r1; ++j) {
            ++pscan;
            if (__ldcg(a.depth + a.er.col[j]) == d) {
              hit = true;
              break;
            }
          }
          if (hit) a.depth[v] = nd;
        }
        queue_append_warp(out, &C->found, hit, v);
      }
      pscan = warp_sum(pscan);
      if (lane_id() == 0 && pscan) atomicAdd(&C->scanned, pscan);
    }
    grid.sync();
    const uint32_t found = ((volatile BcStep*) C)->found;
    if (found == 0) {
      end_step();
      break;
    }
    // sigma of the new level
    if (nd == 1) {
      unsigned long long m_lvl = 0;
      for (uint32_t i = gtid; i < found; i += nthr) {
        const uint32_t u = out[i];
        a.sigma[u] = 1.0;   // staged_bc_bfs.h:68-76: one path per depth-1 vertex, parallel edges or not
        m_lvl += row_len(a.er.rp, u);
      }
      m_lvl = warp_sum(m_lvl);
      if (lane_id() == 0 && m_lvl) atomicAdd(&C->m_lvl, m_lvl);
    } else {
      gather_level(grid, a, GatherSigma{a.depth, a.sigma, d}, le, le + found, C, gtid, nthr);
    }
    end_step();
    const volatile BcStep* V = C;
    if (gtid == 0) {
      a.loff[nd + 1] = le + found;
      if (nd < (uint32_t) kBcMaxStat) {
        ctl->fscan[nd] = V->sc.scanned + V->scanned;
        ctl->mode[nd] = (unsigned char) phase;
      }
      ctl->scanned += V->sc.scanned + V->scanned;
    }
    m_f = V->m_lvl;
    visited_m += m_f;
    lb = le;
    le += found;
    d = nd;
  }
  unsigned long long t1 = 0;
  if (gtid == 0) {
    t1 = bc_global_ns();
    ctl->fwd_ns = t1 - t0;
    ctl->levels = d + 1;
    ctl->reached = le;
  }
  // backward: level d = L .. 0 over its part of the list
  for (int lv = (int) d; lv >= 0; --lv) {
    BcStep* C = &ctl->c[t % 3];
    const uint32_t b = __ldcg(a.loff + lv), e = __ldcg(a.loff + lv + 1);
    gather_level(grid, a, GatherBack{a.depth, a.sigma, a.t, a.c, (uint32_t) lv + 1, lv == 0}, b, e, C, gtid, nthr);
    end_step();
    if (gtid == 0) {
      const unsigned long long s = ((volatile BcStep*) C)->scanned;
      if (lv < kBcMaxStat) ctl->bscan[lv] = s;
      ctl->scanned += s;
    }
  }
  if (gtid == 0) ctl->bwd_ns = bc_global_ns() - t1;
}

// ---------------------------------------------------------------------------
// Several fragments: one level per superstep.
// ---------------------------------------------------------------------------
__global__ void k_bc_seed(uint32_t src, uint32_t* depth, double* sigma) {
  depth[src] = 0;
  sigma[src] = 1.0;
}

// forward level d + 1: every unvisited inner vertex gathers over its whole row
__global__ void k_bc_pull_multi(const uint64_t* rp, const uint32_t* col, uint32_t n, uint32_t d, uint32_t* depth,
                                double* sigma, ScanCtrl* ctrl) {
  unsigned long long scanned = 0, found = 0;
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    if (depth[u] != kBcUnvis) continue;
    const uint64_t r0 = rp[u], r1 = rp[u + 1];
    double s = 0.0;
    bool hit = false;
    for (uint64_t j = r0; j < r1; ++j) {
      const uint32_t v = col[j];
      if (depth[v] == d) {
        hit = true;
        s += sigma[v];
      }
    }
    scanned += r1 - r0;
    if (hit) {
      depth[u] = d + 1;   // read by other threads only as "== d": no conflict
      sigma[u] = d == 0 ? 1.0 : s;
      ++found;
    }
  }
  scanned = warp_sum(scanned);
  found = warp_sum(found);
  if (lane_id() == 0) {
    if (scanned) atomicAdd(&ctrl->scanned, scanned);
    if (found) atomicAdd(&ctrl->next_count, found);
  }
}

// backward level d: the inner vertices at depth d gather t over their rows
__global__ void k_bc_back_multi(const uint64_t* rp, const uint32_t* col, uint32_t n, uint32_t d, const uint32_t* depth,
                                const double* sigma, float* t, float* c, ScanCtrl* ctrl) {
  unsigned long long scanned = 0, found = 0;
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    if (depth[u] != d) continue;
    const uint64_t r0 = rp[u], r1 = rp[u + 1];
    double s = 0.0;
    for (uint64_t j = r0; j < r1; ++j) {
      const uint32_t v = col[j];
      if (depth[v] == d + 1) s += (double) t[v];
    }
    scanned += r1 - r0;
    ++found;
    bc_finish_back(u, s, d == 0, sigma, c, t);
  }
  scanned = warp_sum(scanned);
  found = warp_sum(found);
  if (lane_id() == 0) {
    if (scanned) atomicAdd(&ctrl->scanned, scanned);
    if (found) atomicAdd(&ctrl->next_count, found);
  }
}

__global__ void k_bc_out(const uint32_t* depth, const double* sigma, const float* c, uint32_t n, gl_bc_value* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t d = depth[i];
  gl_bc_value r;
  if (d == kBcUnvis) {
    r.centrality = 0.0;
    r.path_num = 0.0;
    r.depth = INT64_MAX;
  } else {
    r.centrality = (double) c[i];
    r.path_num = sigma[i];
    r.depth = (int64_t) d;
  }
  out[i] = r;
}

struct BcApp : gl_app {
  DevBuf<uint32_t> depth, list, loff, chunk_item;
  DevBuf<double> sigma, part;
  DevBuf<float> t, c;
  DevBuf<BcLong> lng;
  DevBuf<gl_bc_value> out;
  DevBuf<BcFusedCtl> d_ctl;
  PinnedBuf<BcFusedCtl> h_ctl;
  cudaEvent_t ev_done = nullptr;
  int fused_grid = 0;
  uint32_t src = kBcUnvis;
  uint32_t tvnum = 0;
  // several fragments
  int dir = 0;       // 0 forward, 1 backward
  int64_t lvl = 0;   // forward: the deepest level found so far; backward: the level of the next step
  uint64_t reached = 0;   // this fragment's vertices found by the forward rounds

  ~BcApp() override {
    if (ev_done) cudaEventDestroy(ev_done);
  }

  size_t ResultElemBytes() const override { return sizeof(gl_bc_value); }

  int Setup() override {
    // the reference app "can work on undirected graph" only: on a directed one its backward pass is not BC
    if (fv.directed) {
      set_error("bc needs an undirected fragment");
      return GL_ERR_ARG;
    }
    if (gl_frag_oid2lid(frag, cfg.source_oid, &src) != GL_OK) src = kBcUnvis;
    tvnum = fv.ivnum + fv.ovnum;
    const uint32_t tv = std::max<uint32_t>(tvnum, 1), iv = std::max<uint32_t>(fv.ivnum, 1);
    GL_CUDA(depth.alloc(tv));
    GL_CUDA(sigma.alloc(tv));
    GL_CUDA(t.alloc(tv));
    GL_CUDA(c.alloc(iv));
    GL_CUDA(out.alloc(iv));
    if (fv.fnum == 1) {
      // a long row (> kBcShort entries) has at most deg / kBcShort chunks
      const uint64_t chunk_cap = fv.oe_num / kBcShort + 1;
      GL_CUDA(list.alloc(iv));
      GL_CUDA(loff.alloc((size_t) iv + 2));
      GL_CUDA(lng.alloc(iv));
      GL_CUDA(chunk_item.alloc(chunk_cap));
      GL_CUDA(part.alloc(chunk_cap));
      GL_CUDA(d_ctl.alloc(1));
      GL_CUDA(h_ctl.alloc(1));
      return GL_OK;
    }
    GL_TRY(mm.Init(comm, fv, 8));
    return mm.BuildMirrorPlan(eng.stream, fv);
  }

  int Init() override {
    cudaStream_t s = eng.stream;
    dir = 0;
    lvl = 0;
    reached = 0;
    GL_CUDA(cudaMemsetAsync(depth, 0xFF, sizeof(uint32_t) * std::max<uint32_t>(tvnum, 1), s));
    if (fv.fnum == 1) {
      GL_CUDA(cudaMemsetAsync(d_ctl, 0, sizeof(BcFusedCtl), s));
    } else {
      // outer copies of unreached vertices read sigma = 0 and t = 0 through the mirror sync
      GL_CUDA(cudaMemsetAsync(sigma, 0, sizeof(double) * std::max<uint32_t>(tvnum, 1), s));
      GL_CUDA(cudaMemsetAsync(t, 0, sizeof(float) * std::max<uint32_t>(tvnum, 1), s));
    }
    return GL_OK;
  }

  int PEval() override {
    cudaStream_t s = eng.stream;
    if (fv.fnum > 1) {
      if (src != kBcUnvis) GL_LAUNCH(k_bc_seed, 1, 1, s, src, depth, sigma);
      mm.ForceContinue();
      return GL_OK;
    }
    BcFusedArgs a;
    a.er = EdgeRange{fv.oe_rp, fv.oe_col, nullptr};
    a.n = fv.ivnum;
    a.src = src;
    a.m = fv.oe_num;
    a.direction_opt = cfg.direction_opt;
    a.depth = depth;
    a.sigma = sigma;
    a.t = t;
    a.c = c;
    a.list = list;
    a.loff = loff;
    a.lng = lng;
    a.chunk_item = chunk_item;
    a.part = part;
    a.ctl = d_ctl;
    a.hubs = eng.hubs;
    a.hub_cap = eng.hub_cap;
    a.hub_deg = eng.hub_deg;
    if (!fused_grid) fused_grid = persistent_grid(k_bc_fused, eng.sm_count);
    void* args[] = {&a};
    GL_CUDA(cudaLaunchCooperativeKernel((void*) k_bc_fused, dim3(fused_grid), dim3(kTB), args, 0, s));
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaMemcpyAsync(h_ctl, d_ctl, sizeof(BcFusedCtl), cudaMemcpyDeviceToHost, s));
    if (!ev_done) GL_CUDA(cudaEventCreate(&ev_done));
    GL_CUDA(cudaEventRecord(ev_done, s));   // the query's last device operation
    GL_CUDA(cudaStreamSynchronize(s));
    if (getenv("GL_KTIME"))
      fprintf(stderr, "[gl-ktime] bc: %llu levels, forward %.3f ms, backward %.3f ms (thread 0, device timer)\n",
              h_ctl->levels, h_ctl->fwd_ns * 1e-6, h_ctl->bwd_ns * 1e-6);
    q_entries += h_ctl->scanned;
    q_frontier += h_ctl->reached;
    query_end = ev_done;
    return GL_OK;   // no ForceContinue: the query ends with this round
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    const int grid = (int) std::min<uint32_t>((fv.ivnum + 255) / 256, eng.sm_count * 8);
    GL_TRY(eng.reset_ctrl());
    if (dir == 0) {
      // forward level lvl + 1 from the owners' current depth and sigma
      GL_TRY(mm.SyncValuesToGhosts(s, depth, 4));
      GL_TRY(mm.SyncValuesToGhosts(s, sigma, 8));
      if (fv.ivnum)
        GL_LAUNCH(k_bc_pull_multi, grid, 256, s, fv.oe_rp, fv.oe_col, fv.ivnum, (uint32_t) lvl, depth, sigma, eng.ctrl);
      GL_TRY(eng.fetch_ctrl());
      int64_t found = (int64_t) eng.h_ctrl->next_count;
      note_step(eng.h_ctrl->scanned, (uint32_t) found, 1);
      reached += (uint64_t) found;
      GL_TRY(mm.AllReduceI64(&found, 1, 0));
      if (found) ++lvl;
      else dir = 1;   // lvl is the deepest level: the backward pass starts there
      mm.ForceContinue();
      return GL_OK;
    }
    // backward level lvl, from the t of level lvl + 1
    GL_TRY(mm.SyncValuesToGhosts(s, t, 4));
    if (fv.ivnum)
      GL_LAUNCH(k_bc_back_multi, grid, 256, s, fv.oe_rp, fv.oe_col, fv.ivnum, (uint32_t) lvl, depth, sigma, t, c,
                eng.ctrl);
    GL_TRY(eng.fetch_ctrl());
    note_step(eng.h_ctrl->scanned, (uint32_t) eng.h_ctrl->next_count, 2);
    if (--lvl >= 0) mm.ForceContinue();
    return GL_OK;
  }

  void FillStats(gl_query_stats* st) override {
    if (fv.fnum > 1) {
      // the forward steps count this fragment's share of each level; the source counts in level 0
      st->frontier_vertices = reached + (src != kBcUnvis ? 1 : 0);
      return;
    }
    const uint32_t L1 = (uint32_t) h_ctl->levels;   // levels 0..L: L + 1
    st->supersteps = (int) (2 * L1);
    st->frontier_vertices = h_ctl->reached;
    st->entries_scanned = h_ctl->scanned;
    const int n = (int) std::min<uint32_t>(2 * L1, GL_MAX_STEP_STATS);
    st->n_steps = n;
    if (!n) return;
    std::vector<uint32_t> off(L1 + 1);
    if (cudaMemcpy(off.data(), loff.get(), sizeof(uint32_t) * (L1 + 1), cudaMemcpyDeviceToHost) != cudaSuccess) return;
    // steps 0..L: forward levels 0..L; steps L+1..2L+1: backward levels L..0
    for (int i = 0; i < n; ++i) {
      const bool fwd = i < (int) L1;
      const uint32_t lv = fwd ? (uint32_t) i : 2 * L1 - 1 - (uint32_t) i;
      st->step_ms[i] = 0.f;
      st->step_frontier[i] = off[lv + 1] - off[lv];
      st->step_mode[i] = fwd ? (lv < (uint32_t) kBcMaxStat ? h_ctl->mode[lv] : 0) : 2;
      st->step_entries[i] = lv < (uint32_t) kBcMaxStat ? (fwd ? h_ctl->fscan[lv] : h_ctl->bscan[lv]) : 0;
    }
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_LAUNCH(k_bc_out, (fv.ivnum + 255) / 256, 256, eng.stream, depth, sigma, c, fv.ivnum, out);
    GL_CUDA(cudaMemcpyAsync(host_out, out, sizeof(gl_bc_value) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_bc() { return new BcApp; }

}  // namespace gl
