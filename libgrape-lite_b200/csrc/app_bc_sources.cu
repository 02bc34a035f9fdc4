// app_bc_sources.cu — betweenness centrality summed over a list of sources (undirected graphs).
//
// For every source s of the list: depth_s / sigma_s as GL_APP_BC, then the backward pass in f64:
// cacc = sum of t_s(w) over the entries (v, w) of v's row with depth_s(w) = depth_s(v) + 1,
// delta_s(v) = cacc * sigma_s(v), t_s(v) = (1 / sigma_s(v)) * (1 + delta_s(v)); bc(v) is the left fold
// of delta_s(v) over the list.
//
// Sources run in batches of B <= 32, lane b of a warp owning source b of the batch.  Every per-vertex
// state is B lanes wide and vertex-major (sigma[v * B + b], t[v * B + b], depth[v * B + b]), next to
// two u32 lane masks per vertex: `vis` (reached) and the level mask (forward: at the current level;
// backward: at the level below the one being processed).  A gather over a row reads each entry's mask
// once as a broadcast and, where a lane's bit is set, that lane's sigma or t: one coalesced read of up
// to 256 B per entry instead of B scattered 8-byte reads.
//
// Every sum is a gather in a fixed order: a warp walks a row of up to kBcsChunk entries sequentially;
// a longer row is cut into kBcsChunk-entry chunks, each summed sequentially by one warp into a B-wide
// partial, and the partials are added in chunk order.  Nothing depends on the batch a source runs in,
// so the result is bit-identical for every B; there are no floating-point atomics.
//
//  * One fragment: each batch is ONE cooperative launch (k_bcs_batch): seed, forward levels, backward
//    levels, then every vertex adds its B lanes to bc in lane order.  Batches are enqueued back to
//    back with no host synchronisation.
//  * Several fragments: one worker round per level, the same device functions in separate launches;
//    the outer copies' masks and B-wide sigma / t rows arrive through the dense mirror sync.
#include <cooperative_groups.h>

#include "apps_common.cuh"

namespace gl {
namespace {

namespace cg = cooperative_groups;

constexpr uint32_t kBcsUnvis = 0xFFFFFFFFu;
constexpr uint32_t kBcsChunk = 1024;   // rows up to this length: one warp; longer: chunks of this many entries
constexpr uint32_t kBcsMaxB = 32;
#define GL_BCS_CTAS 4

struct BcsGraph {
  const uint64_t* rp;
  const uint32_t* col;
  uint32_t n;                    // inner vertices (the rows)
  uint32_t B;                    // lane stride of the state
  const uint32_t* long_v;        // [nlong] the rows longer than kBcsChunk
  const uint32_t* long_base;     // [nlong + 1] their first chunk
  const uint32_t* chunk_row;     // [nchunk] the long row (index into long_v) of a chunk
  uint32_t nlong, nchunk;
  uint32_t* depth;               // [n * B]
  double* sigma;                 // [(n + outer) * B]; after the backward pass: delta
  double* t;                     // [(n + outer) * B]
  uint32_t* vis;                 // [n]
  double* part;                  // [nchunk * B]
};

struct BcsCount {
  unsigned long long found;      // (vertex, lane) pairs found / processed
  unsigned long long scanned;    // row entries read
};

GL_DEV uint32_t bcs_warp_id() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
GL_DEV uint32_t bcs_nwarps() { return (gridDim.x * blockDim.x) >> 5; }

// Lane-wise sum over the entries [j0, j1): lane b adds val[w * B + b] for each entry w whose mask
// has bit b of `want` set, in entry order.  Entries are fetched 32 at a time (column and mask), then
// walked one by one from registers.
GL_DEV double bcs_gather(const BcsGraph& g, const uint32_t* mask, const double* val, uint64_t j0, uint64_t j1,
                         uint32_t want) {
  const uint32_t lane = lane_id();
  double s = 0.0;
  for (uint64_t base = j0; base < j1; base += 32) {
    const uint64_t j = base + lane;
    uint32_t u = 0, m = 0;
    if (j < j1) {
      u = __ldg(g.col + j);
      m = __ldcg(mask + u) & want;
    }
    uint32_t any = __ballot_sync(0xFFFFFFFFu, m != 0);
    while (any) {   // only entries some lane takes, in entry order
      const uint32_t k = __ffs(any) - 1;
      any &= any - 1;
      const uint32_t mk = __shfl_sync(0xFFFFFFFFu, m, k);
      const uint32_t uk = __shfl_sync(0xFFFFFFFFu, u, k);
      if ((mk >> lane) & 1u) s += __ldcg(val + (uint64_t) uk * g.B + lane);
    }
  }
  return s;
}

// forward: the lanes of v still to be reached
GL_DEV uint32_t bcs_want_fwd(const BcsGraph& g, uint32_t v, uint32_t live) { return live & ~__ldcg(g.vis + v); }
// backward: the lanes of v at depth d
GL_DEV uint32_t bcs_want_back(const BcsGraph& g, uint32_t v, uint32_t d) {
  const uint32_t lane = lane_id();
  const bool at = lane < g.B && __ldcg(g.depth + (uint64_t) v * g.B + lane) == d;
  return __ballot_sync(0xFFFFFFFFu, at);
}

// forward level d + 1 for v from its lane sums: a lane that wants and found a level-d neighbour is reached
GL_DEV void bcs_finish_fwd(const BcsGraph& g, uint32_t v, uint32_t want, double s, uint32_t d, uint32_t* next,
                           unsigned long long& found) {
  const uint32_t lane = lane_id();
  const bool hit = ((want >> lane) & 1u) && s > 0.0;   // every reached sigma is >= 1
  const uint32_t nb = __ballot_sync(0xFFFFFFFFu, hit);
  if (hit) {
    g.depth[(uint64_t) v * g.B + lane] = d + 1;
    g.sigma[(uint64_t) v * g.B + lane] = d == 0 ? 1.0 : s;   // one path per depth-1 vertex
  }
  if (lane == 0) {
    if (nb) g.vis[v] = __ldcg(g.vis + v) | nb;
    next[v] = nb;
    found += __popc(nb);
  }
}

// backward level d for v: delta and t of the lanes at depth d; mask[v] = those lanes
GL_DEV void bcs_finish_back(const BcsGraph& g, uint32_t v, uint32_t me, double s, uint32_t* out_mask,
                            unsigned long long& found) {
  const uint32_t lane = lane_id();
  if ((me >> lane) & 1u) {
    const uint64_t i = (uint64_t) v * g.B + lane;
    const double sg = __ldcg(g.sigma + i);
    const double delta = __dmul_rn(s, sg);
    g.t[i] = __dmul_rn(1.0 / sg, __dadd_rn(1.0, delta));
    g.sigma[i] = delta;
  }
  if (lane == 0) {
    out_mask[v] = me;
    found += __popc(me);
  }
}

// Phase 1 of a level: every vertex with a row of up to kBcsChunk entries is gathered and finished by one
// warp; every chunk of a longer row leaves its B-wide partial in part.  fwd: level d -> d + 1 reading
// mask `in` (level d) and writing `out` (level d + 1); !fwd: backward level d reading `in` (level d + 1)
// and writing `out` (level d).
template <bool kFwd>
GL_DEV void bcs_rows(const BcsGraph& g, uint32_t d, uint32_t live, const uint32_t* in, uint32_t* out,
                     BcsCount* cnt) {
  unsigned long long found = 0, scanned = 0;
  const uint32_t nw = bcs_nwarps(), lane = lane_id();
  for (uint32_t item = bcs_warp_id(); item < g.n + g.nchunk; item += nw) {
    if (item < g.n) {
      const uint32_t v = item;
      const uint64_t r0 = __ldg(g.rp + v), r1 = __ldg(g.rp + v + 1);
      if (r1 - r0 > kBcsChunk) continue;   // chunked below
      const uint32_t want = kFwd ? bcs_want_fwd(g, v, live) : bcs_want_back(g, v, d);
      double s = 0.0;
      if (want && r1 > r0) {
        s = bcs_gather(g, in, kFwd ? g.sigma : g.t, r0, r1, want);
        scanned += r1 - r0;
      }
      if (kFwd) bcs_finish_fwd(g, v, want, s, d, out, found);
      else bcs_finish_back(g, v, want, s, out, found);
    } else {
      const uint32_t ck = item - g.n, row = __ldg(g.chunk_row + ck), v = __ldg(g.long_v + row);
      const uint32_t want = kFwd ? bcs_want_fwd(g, v, live) : bcs_want_back(g, v, d);
      if (!want) continue;   // the fold does not read the partials then
      const uint64_t c0 = __ldg(g.rp + v) + (uint64_t) (ck - __ldg(g.long_base + row)) * kBcsChunk;
      const uint64_t c1 = min((unsigned long long) (c0 + kBcsChunk), (unsigned long long) __ldg(g.rp + v + 1));
      const double s = bcs_gather(g, in, kFwd ? g.sigma : g.t, c0, c1, want);
      if (lane < g.B) g.part[(uint64_t) ck * g.B + lane] = s;
      scanned += c1 - c0;
    }
  }
  found = warp_sum(found);
  if (lane == 0) {
    if (found) atomicAdd(&cnt->found, found);
    if (scanned) atomicAdd(&cnt->scanned, scanned);
  }
}

// Phase 2: every long row adds its chunk partials in chunk order and is finished.
template <bool kFwd>
GL_DEV void bcs_long(const BcsGraph& g, uint32_t d, uint32_t live, uint32_t* out, BcsCount* cnt) {
  unsigned long long found = 0;
  const uint32_t nw = bcs_nwarps(), lane = lane_id();
  for (uint32_t row = bcs_warp_id(); row < g.nlong; row += nw) {
    const uint32_t v = __ldg(g.long_v + row);
    const uint32_t want = kFwd ? bcs_want_fwd(g, v, live) : bcs_want_back(g, v, d);
    double s = 0.0;
    if (want && lane < g.B)
      for (uint32_t ck = __ldg(g.long_base + row); ck < __ldg(g.long_base + row + 1); ++ck)
        s += __ldcg(g.part + (uint64_t) ck * g.B + lane);
    if (kFwd) bcs_finish_fwd(g, v, want, s, d, out, found);
    else bcs_finish_back(g, v, want, s, out, found);
  }
  if (lane == 0 && found) atomicAdd(&cnt->found, found);
}

// level 0 of a batch: lane b's source (an inner lid or kBcsUnvis); duplicates share a vertex
GL_DEV void bcs_seed(const BcsGraph& g, const uint32_t* src, uint32_t* mask0, unsigned long long* present) {
  unsigned long long p = 0;
  for (uint32_t b = 0; b < g.B; ++b) {
    const uint32_t s = src[b];
    if (s == kBcsUnvis) continue;
    g.depth[(uint64_t) s * g.B + b] = 0;
    g.sigma[(uint64_t) s * g.B + b] = 1.0;
    mask0[s] |= 1u << b;
    g.vis[s] |= 1u << b;
    ++p;
  }
  *present += p;
}

// bc[v] += delta of lanes 0..B-1 in lane order (depth 0: the source itself, which adds nothing)
GL_DEV void bcs_accumulate(const BcsGraph& g, double* bc, uint32_t gtid, uint32_t nthr) {
  for (uint32_t v = gtid; v < g.n; v += nthr) {
    double acc = bc[v];
    for (uint32_t b = 0; b < g.B; ++b) {
      const uint64_t i = (uint64_t) v * g.B + b;
      const uint32_t dd = __ldcg(g.depth + i);
      if (dd != 0 && dd != kBcsUnvis) acc += __ldcg(g.sigma + i);
    }
    bc[v] = acc;
  }
}

// ---------------------------------------------------------------------------
// One fragment: one cooperative launch per batch.
// ---------------------------------------------------------------------------
struct BcsBatchCtl {
  BcsCount c[3];                 // step t uses c[t % 3] (see k_bc_fused)
};

struct BcsBatchArgs {
  BcsGraph g;
  uint32_t live;                 // lanes with a source in the graph
  const uint32_t* src;           // [B]
  uint32_t* mask[2];             // [n]
  double* bc;
  BcsBatchCtl* ctl;
  unsigned long long* stat;      // [2]: reached (vertex, source) pairs, row entries read
};

__global__ void __launch_bounds__(kTB, GL_BCS_CTAS) k_bcs_batch(BcsBatchArgs a) {
  cg::grid_group grid = cg::this_grid();
  const BcsGraph& g = a.g;
  BcsBatchCtl* ctl = a.ctl;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nthr = gridDim.x * blockDim.x;
  uint32_t t = 0;
  unsigned long long reached = 0, scanned = 0;   // thread 0
  auto end_step = [&]() {
    grid.sync();
    if (gtid == 0) ctl->c[(t + 2) % 3] = BcsCount{0, 0};
    ++t;
  };
  if (gtid == 0) {
    ctl->c[0] = ctl->c[1] = ctl->c[2] = BcsCount{0, 0};
    bcs_seed(g, a.src, a.mask[0], &reached);
  }
  grid.sync();
  // forward: level d + 1 from level d until a level is empty
  uint32_t d = 0, cur = 0;
  for (;;) {
    BcsCount* C = &ctl->c[t % 3];
    bcs_rows<true>(g, d, a.live, a.mask[cur], a.mask[cur ^ 1], C);
    if (g.nlong) {
      grid.sync();
      bcs_long<true>(g, d, a.live, a.mask[cur ^ 1], C);
    }
    end_step();
    const volatile BcsCount* V = C;
    const unsigned long long found = V->found;
    if (gtid == 0) {
      reached += found;
      scanned += V->scanned;
    }
    cur ^= 1;   // mask[cur] now holds level d + 1 (all zero when found == 0)
    if (!found) break;
    ++d;
  }
  // backward: level d = L .. 1, reading the level-(d + 1) mask and writing level d's
  for (; d >= 1; --d) {
    BcsCount* C = &ctl->c[t % 3];
    bcs_rows<false>(g, d, a.live, a.mask[cur], a.mask[cur ^ 1], C);
    if (g.nlong) {
      grid.sync();
      bcs_long<false>(g, d, a.live, a.mask[cur ^ 1], C);
    }
    end_step();
    if (gtid == 0) scanned += ((const volatile BcsCount*) C)->scanned;
    cur ^= 1;
  }
  bcs_accumulate(g, a.bc, gtid, nthr);
  if (gtid == 0) {
    a.stat[0] = reached;
    a.stat[1] = scanned;
  }
}

// ---------------------------------------------------------------------------
// Several fragments: one level per worker round.
// ---------------------------------------------------------------------------
__global__ void k_bcs_seed(BcsGraph g, const uint32_t* src, uint32_t* mask0, unsigned long long* present) {
  bcs_seed(g, src, mask0, present);
}
template <bool kFwd>
__global__ void __launch_bounds__(kTB) k_bcs_rows(BcsGraph g, uint32_t d, uint32_t live, const uint32_t* in,
                                                  uint32_t* out, BcsCount* cnt) {
  bcs_rows<kFwd>(g, d, live, in, out, cnt);
}
template <bool kFwd>
__global__ void __launch_bounds__(kTB) k_bcs_long(BcsGraph g, uint32_t d, uint32_t live, uint32_t* out,
                                                  BcsCount* cnt) {
  bcs_long<kFwd>(g, d, live, out, cnt);
}
__global__ void k_bcs_accumulate(BcsGraph g, double* bc) {
  bcs_accumulate(g, bc, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

uint64_t fnv1a(const int64_t* p, uint64_t n) {
  uint64_t h = 1469598103934665603ull;
  for (uint64_t i = 0; i < n; ++i) {
    uint64_t x = (uint64_t) p[i];
    for (int k = 0; k < 8; ++k) {
      h ^= (x >> (8 * k)) & 0xFF;
      h *= 1099511628211ull;
    }
  }
  return h;
}

struct BcSourcesApp : gl_app {
  DevBuf<uint32_t> depth, vis, mask0, mask1, long_v, long_base, chunk_row, d_src;
  DevBuf<double> sigma, t, part, bc;
  DevBuf<BcsBatchCtl> d_ctl;
  DevBuf<BcsCount> d_cnt;
  DevBuf<unsigned long long> d_stat;   // one fragment: [2 * batches]; several: [1] sources present
  PinnedBuf<BcsCount> h_cnt;
  std::vector<unsigned long long> h_stat;
  cudaEvent_t ev_done = nullptr;
  BcsGraph g{};
  uint32_t B = 0, tvnum = 0;
  int fused_grid = 0;
  bool have_list = false;
  std::vector<uint32_t> lids;   // the list as this fragment's inner lids (kBcsUnvis: not here / not a vertex)
  uint64_t nbatch = 0, in_graph = 0;
  // several fragments
  uint64_t batch = 0;
  int dir = 0;                  // 0 forward, 1 backward
  uint32_t lvl = 0, cur = 0;    // the level being expanded (forward) or processed (backward)
  uint64_t reached = 0;         // this fragment's (vertex, source) pairs, sources included
  std::vector<uint8_t> in_group;   // per list entry: a vertex of some fragment of the group

  ~BcSourcesApp() override {
    if (ev_done) cudaEventDestroy(ev_done);
  }

  size_t ResultElemBytes() const override { return sizeof(double); }
  uint32_t* mask(uint32_t i) { return i ? mask1.get() : mask0.get(); }

  int Setup() override {
    if (fv.directed) {
      set_error("bc_sources needs an undirected fragment");
      return GL_ERR_ARG;
    }
    const int req = cfg.reserved[0];
    if (req < 0 || req > (int) kBcsMaxB) {
      set_error("bc_sources: batch width reserved[0] = %d is not in 0..32", req);
      return GL_ERR_ARG;
    }
    if (cfg.reserved[1] < 0) {
      set_error("bc_sources: reserved[1] = %d is negative", cfg.reserved[1]);
      return GL_ERR_ARG;
    }
    B = req ? (uint32_t) req : kBcsMaxB;
    tvnum = fv.ivnum + fv.ovnum;
    const uint32_t n = fv.ivnum;
    const size_t tv = std::max<uint32_t>(tvnum, 1), iv = std::max<uint32_t>(n, 1);
    cudaStream_t s = eng.stream;
    // long rows and their chunks (fixed for the fragment)
    std::vector<uint64_t> rp(n + 1);
    GL_CUDA(cudaMemcpy(rp.data(), fv.oe_rp, sizeof(uint64_t) * (n + 1), cudaMemcpyDeviceToHost));
    std::vector<uint32_t> lv, lb(1, 0), cr;
    for (uint32_t v = 0; v < n; ++v) {
      const uint64_t deg = rp[v + 1] - rp[v];
      if (deg <= kBcsChunk) continue;
      const uint32_t nc = (uint32_t) ((deg + kBcsChunk - 1) / kBcsChunk);
      for (uint32_t k = 0; k < nc; ++k) cr.push_back((uint32_t) lv.size());
      lv.push_back(v);
      lb.push_back(lb.back() + nc);
    }
    GL_CUDA(long_v.alloc(std::max<size_t>(lv.size(), 1)));
    GL_CUDA(long_base.alloc(lb.size()));
    GL_CUDA(chunk_row.alloc(std::max<size_t>(cr.size(), 1)));
    if (!lv.empty()) GL_CUDA(cudaMemcpy(long_v, lv.data(), sizeof(uint32_t) * lv.size(), cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(long_base, lb.data(), sizeof(uint32_t) * lb.size(), cudaMemcpyHostToDevice));
    if (!cr.empty()) GL_CUDA(cudaMemcpy(chunk_row, cr.data(), sizeof(uint32_t) * cr.size(), cudaMemcpyHostToDevice));
    // fit[0]: the widest row the mirror area holds for every peer's outer copies (several fragments);
    // fit[1]: the widest batch free HBM holds, 20 B bytes per vertex (sigma, t, depth) and 8 B per chunk,
    // when B is not requested (reserved[1] > 0 stands in for it: a test hook).  Both are decided once for
    // the group (min all-reduce): every rank must cut the list into the same batches.
    int64_t fit[2] = {(int64_t) B, (int64_t) B};
    if (!req) {
      if (cfg.reserved[1] > 0) {
        fit[1] = cfg.reserved[1];
      } else {
        size_t free_b = 0, total_b = 0;
        GL_CUDA(cudaMemGetInfo(&free_b, &total_b));
        const size_t reserve = free_b / 16 + (64ull << 20) + sizeof(double) * iv + 16 * tv;
        const size_t per_lane = 16 * tv + 4 * iv + 8 * std::max<size_t>(cr.size(), 1);
        fit[1] = free_b > reserve ? (int64_t) ((free_b - reserve) / per_lane) : 0;
      }
      fit[1] = std::min<int64_t>(fit[1], B);
    }
    uint32_t most = 0;
    if (fv.fnum > 1) {
      GL_TRY(mm.Init(comm, fv, 8));
      std::vector<uint32_t> gr(fv.fnum + 1);
      GL_CUDA(cudaMemcpy(gr.data(), fv.outer_range, sizeof(uint32_t) * (fv.fnum + 1), cudaMemcpyDeviceToHost));
      for (uint32_t f = 0; f < fv.fnum; ++f) most = std::max(most, gr[f + 1] - gr[f]);
      if (most) fit[0] = std::min<int64_t>(fit[0], (int64_t) (comm->mirror_bytes / (8 * (size_t) most)));
      GL_TRY(mm.AllReduceI64(fit, 2, 1));
    }
    if (fit[0] < 1) {
      set_error("bc_sources: mirror_bytes (%zu) cannot hold one 8-byte row per outer copy of a fragment group",
                comm->mirror_bytes);
      return GL_ERR_ARG;
    }
    if (fit[1] < 1) {
      set_error("bc_sources: free HBM cannot hold one source's state (20 bytes per vertex) on every fragment");
      return GL_ERR_NOMEM;
    }
    B = (uint32_t) std::min(fit[0], fit[1]);
    if (fv.fnum > 1) GL_TRY(mm.BuildMirrorPlan(s, fv));
    GL_CUDA(depth.alloc(iv * B));
    GL_CUDA(sigma.alloc(tv * B));
    GL_CUDA(t.alloc(tv * B));
    GL_CUDA(part.alloc(std::max<size_t>(cr.size(), 1) * B));
    GL_CUDA(vis.alloc(iv));
    GL_CUDA(mask0.alloc(tv));
    GL_CUDA(mask1.alloc(tv));
    GL_CUDA(bc.alloc(iv));
    GL_CUDA(d_ctl.alloc(1));
    GL_CUDA(d_cnt.alloc(1));
    GL_CUDA(h_cnt.alloc(1));
    g.rp = fv.oe_rp;
    g.col = fv.oe_col;
    g.n = n;
    g.B = B;
    g.long_v = long_v;
    g.long_base = long_base;
    g.chunk_row = chunk_row;
    g.nlong = (uint32_t) lv.size();
    g.nchunk = (uint32_t) cr.size();
    g.depth = depth;
    g.sigma = sigma;
    g.t = t;
    g.vis = vis;
    g.part = part;
    return GL_OK;
  }

  int SetSources(const int64_t* oids, uint64_t n) override {
    std::vector<uint32_t> l;
    if (fv.fnum > 1) {
      // every rank must pass the same list: max(x) == -max(-x) for the length and the hash
      const int64_t len = oids ? (int64_t) n : -1, h = oids ? (int64_t) (fnv1a(oids, n) >> 1) : -1;
      int64_t v[4] = {len, h, -len, -h};
      GL_TRY(mm.AllReduceI64(v, 4, 2));
      if (v[0] != -v[2] || v[1] != -v[3]) {
        set_error("gl_app_set_sources: the ranks of the fragment group passed different lists");
        return GL_ERR_ARG;
      }
    }
    if (!oids) {
      // every vertex of the group in gid order: fragment 0's inner vertices in lid order, then fragment 1's ..
      std::vector<int64_t> cnt(fv.fnum, 0);
      cnt[fv.fid] = fv.ivnum;
      GL_TRY(mm.AllReduceI64(cnt.data(), (int) fv.fnum, 0));
      for (uint32_t f = 0; f < fv.fnum; ++f)
        for (int64_t i = 0; i < cnt[f]; ++i) l.push_back(f == fv.fid ? (uint32_t) i : kBcsUnvis);
    } else {
      l.resize(n);
      for (uint64_t i = 0; i < n; ++i)
        if (gl_frag_oid2lid(frag, oids[i], &l[i]) != GL_OK) l[i] = kBcsUnvis;
    }
    // an entry no fragment holds keeps its lane out of every batch's live mask
    std::vector<int64_t> here(l.size());
    for (size_t i = 0; i < l.size(); ++i) here[i] = l[i] != kBcsUnvis;
    if (fv.fnum > 1 && oids && n) GL_TRY(mm.AllReduceI64(here.data(), (int) here.size(), 2));
    in_group.assign(l.size(), 1);
    if (oids)
      for (size_t i = 0; i < l.size(); ++i) in_group[i] = here[i] != 0;
    lids.swap(l);
    nbatch = (lids.size() + B - 1) / B;
    std::vector<uint32_t> padded(lids);
    padded.resize(std::max<uint64_t>(nbatch * B, 1), kBcsUnvis);
    GL_CUDA(d_src.alloc(padded.size()));
    GL_CUDA(cudaMemcpy(d_src, padded.data(), sizeof(uint32_t) * padded.size(), cudaMemcpyHostToDevice));
    GL_CUDA(d_stat.alloc(std::max<uint64_t>(2 * nbatch, 2)));
    in_graph = 0;
    for (uint32_t x : lids) in_graph += x != kBcsUnvis;
    have_list = true;
    return GL_OK;
  }

  uint32_t live_of(uint64_t b) const {
    uint32_t m = 0;
    for (uint32_t k = 0; k < B && b * B + k < lids.size(); ++k)
      if (in_group[b * B + k]) m |= 1u << k;
    return m;
  }

  int ClearBatch() {
    cudaStream_t s = eng.stream;
    GL_CUDA(cudaMemsetAsync(depth, 0xFF, sizeof(uint32_t) * std::max<uint32_t>(fv.ivnum, 1) * B, s));
    GL_CUDA(cudaMemsetAsync(vis, 0, sizeof(uint32_t) * std::max<uint32_t>(fv.ivnum, 1), s));
    GL_CUDA(cudaMemsetAsync(mask0, 0, sizeof(uint32_t) * std::max<uint32_t>(tvnum, 1), s));
    return GL_OK;
  }

  int Init() override {
    if (!have_list) {
      set_error("bc_sources: no source list: call gl_app_set_sources first");
      return GL_ERR_ARG;
    }
    GL_CUDA(cudaMemsetAsync(bc, 0, sizeof(double) * std::max<uint32_t>(fv.ivnum, 1), eng.stream));
    GL_CUDA(cudaMemsetAsync(d_stat, 0, sizeof(unsigned long long) * std::max<uint64_t>(2 * nbatch, 2), eng.stream));
    batch = 0;
    dir = 0;
    lvl = 0;
    cur = 0;
    reached = 0;
    return GL_OK;
  }

  int PEval() override {
    cudaStream_t s = eng.stream;
    if (fv.fnum > 1) {
      if (nbatch == 0) return GL_OK;
      GL_TRY(SeedMulti());
      mm.ForceContinue();
      return GL_OK;
    }
    if (!fused_grid) fused_grid = persistent_grid(k_bcs_batch, eng.sm_count);
    for (uint64_t b = 0; b < nbatch; ++b) {
      GL_TRY(ClearBatch());
      BcsBatchArgs a;
      a.g = g;
      a.live = live_of(b);
      a.src = d_src.get() + b * B;
      a.mask[0] = mask0;
      a.mask[1] = mask1;
      a.bc = bc;
      a.ctl = d_ctl;
      a.stat = d_stat.get() + 2 * b;
      void* args[] = {&a};
      GL_CUDA(cudaLaunchCooperativeKernel((void*) k_bcs_batch, dim3(fused_grid), dim3(kTB), args, 0, s));
      GL_COUNT_LAUNCH();
    }
    h_stat.assign(2 * nbatch, 0);
    if (nbatch)
      GL_CUDA(cudaMemcpyAsync(h_stat.data(), d_stat, sizeof(unsigned long long) * 2 * nbatch, cudaMemcpyDeviceToHost, s));
    if (!ev_done) GL_CUDA(cudaEventCreate(&ev_done));
    GL_CUDA(cudaEventRecord(ev_done, s));
    GL_CUDA(cudaStreamSynchronize(s));
    for (uint64_t b = 0; b < nbatch; ++b) {
      q_frontier += h_stat[2 * b];
      q_entries += h_stat[2 * b + 1];
    }
    query_end = ev_done;
    return GL_OK;
  }

  // several fragments: clear and seed batch `batch`, forward from level 0
  int SeedMulti() {
    cudaStream_t s = eng.stream;
    GL_TRY(ClearBatch());
    GL_LAUNCH(k_bcs_seed, 1, 1, s, g, d_src.get() + batch * B, mask0.get(), d_stat.get());
    dir = 0;
    lvl = 0;
    cur = 0;
    return GL_OK;
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    const uint32_t live = live_of(batch);
    const int grid = (int) std::min<uint64_t>(((uint64_t) fv.ivnum + g.nchunk + 7) / 8 + 1, (uint64_t) eng.sm_count * 8);
    GL_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(BcsCount), s));
    // the outer copies take the owners' level mask and sigma (forward) or t (backward) rows
    GL_TRY(mm.SyncValuesToGhosts(s, mask(cur), 4));
    GL_TRY(mm.SyncRowsToGhosts(s, dir == 0 ? sigma.get() : t.get(), (int) (8 * B)));
    if (dir == 0) {
      GL_LAUNCH(k_bcs_rows<true>, grid, kTB, s, g, lvl, live, mask(cur), mask(cur ^ 1), d_cnt.get());
      if (g.nlong) GL_LAUNCH(k_bcs_long<true>, grid, kTB, s, g, lvl, live, mask(cur ^ 1), d_cnt.get());
    } else {
      GL_LAUNCH(k_bcs_rows<false>, grid, kTB, s, g, lvl, live, mask(cur), mask(cur ^ 1), d_cnt.get());
      if (g.nlong) GL_LAUNCH(k_bcs_long<false>, grid, kTB, s, g, lvl, live, mask(cur ^ 1), d_cnt.get());
    }
    GL_CUDA(cudaMemcpyAsync(h_cnt, d_cnt, sizeof(BcsCount), cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    note_step(h_cnt->scanned, (uint32_t) std::min<unsigned long long>(h_cnt->found, UINT32_MAX), 2);
    cur ^= 1;
    if (dir == 0) {
      reached += h_cnt->found;
      int64_t found = (int64_t) h_cnt->found;
      GL_TRY(mm.AllReduceI64(&found, 1, 0));
      if (found) {
        ++lvl;
      } else if (lvl > 0) {
        dir = 1;   // lvl is the deepest level; mask(cur) is the empty level below it
      } else {
        GL_TRY(NextBatch());
        return GL_OK;
      }
      mm.ForceContinue();
      return GL_OK;
    }
    if (--lvl >= 1) {
      mm.ForceContinue();
      return GL_OK;
    }
    return NextBatch();
  }

  int NextBatch() {
    cudaStream_t s = eng.stream;
    if (fv.ivnum)
      GL_LAUNCH(k_bcs_accumulate, (int) std::min<uint32_t>((fv.ivnum + 255) / 256, eng.sm_count * 8), 256, s, g,
                bc.get());
    if (++batch < nbatch) {
      GL_TRY(SeedMulti());
      mm.ForceContinue();
    }
    return GL_OK;
  }

  void FillStats(gl_query_stats* st) override {
    if (fv.fnum > 1) {
      unsigned long long present = 0;
      if (cudaMemcpy(&present, d_stat.get(), sizeof(present), cudaMemcpyDeviceToHost) != cudaSuccess) return;
      st->frontier_vertices = reached + present;
      st->touched_vertices = reached;
      return;
    }
    st->supersteps = (int) nbatch;
    st->frontier_vertices = q_frontier;
    st->touched_vertices = q_frontier - in_graph;
    st->entries_scanned = q_entries;
    const int n = (int) std::min<uint64_t>(nbatch, GL_MAX_STEP_STATS);
    st->n_steps = n;
    for (int i = 0; i < GL_MAX_STEP_STATS; ++i) {
      st->step_ms[i] = 0.f;
      st->step_frontier[i] = i < n ? (uint32_t) std::min<unsigned long long>(h_stat[2 * i], UINT32_MAX) : 0;
      st->step_entries[i] = i < n ? h_stat[2 * i + 1] : 0;
      st->step_mode[i] = i < n ? 2 : 0;
    }
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_CUDA(cudaMemcpyAsync(host_out, bc, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_bc_sources() { return new BcSourcesApp; }

}  // namespace gl
