// app_lcc_directed.cu — local clustering coefficient of a directed graph by weighted oriented
// triangle counting.
//
// Semantics of examples/analytical_apps/lcc/lcc_directed.h:146-362 + lcc_directed_context.h:52-67
// (LCCDirected, run_app_opt.h:426-441):
//   N(v) = the distinct neighbours of v in oe(v) ∪ ie(v) (v itself when it has a self loop);
//   d(v) = |N(v)|; w(v,u) = CSR entries of u in oe(v) ∪ ie(v) = #(v->u) + #(u->v), symmetric;
//   tri(v) = sum of w(u,x) over unordered pairs {u, x} ⊆ N(v) \ {v}, u != x, u and x adjacent;
//   lcc(v) = tri / (d (d - 1)), 0 when d < 2.
// The reference orients every pair along (|oe| + |ie|, IdHasher(gid)); any strict total order gives the
// same tri because every weight is symmetric, and this app breaks degree ties by gid as app_lcc.cu does.
// Two deliberate differences (include/grape_b200.h): weights are exact (the reference keeps them in a
// uint8_t, so 256 parallel entries weigh 0) and counts are 64-bit (LCCDirected32 can wrap on hubs).
//
// PEval builds the oriented rows N+(v) = { u in N(v) : u ranked below v } with their weights:
//   1. deg(v) = |oe(v)| + |ie(v)|; outer copies take their owners' value (dense mirror sync);
//   2. oe(v) and ie(v) are both sorted by lid, so the union is walked in merge order (merge path, ties
//      to oe): a distinct neighbour belongs to its first occurrence, in oe if it is there, otherwise in
//      ie, and its weight is the length of its equal range in each row.  A count pass (d and |N+|), a
//      scan and a fill pass write the oriented rows; rows of up to kLccdWarpRow merged entries are walked
//      by a warp, longer ones (R-MAT in-rows of hubs) by a CTA;
//   3. several fragments: rows hold gids, sorted by gid (outer gids do not follow lid order), and every
//      fragment replicates its peers' rows and weights (PeerCsr).
// IncEval (TriangleApp in dag_common.cuh, shared with app_lcc.cu) stage 0: one warp per oriented edge
// (v,u) intersects N+(u) with the sorted N+(v); for every common x: tri[x] += w(v,u), tri[u] += w(v,x),
// tri[v] += w(u,x), in 64-bit atomics.  A triangle is counted once, by the owner of its highest-ranked
// vertex; counts that land on outer copies go to their owners as (lid, count) items, added in stage 1.
#include "dag_common.cuh"

namespace gl {
namespace {

constexpr uint64_t kLccdWarpRow = kTB;   // longer merged rows (|oe| + |ie|) are walked by a whole CTA

GL_DEV bool lccd_keep(uint32_t dv, uint32_t du, uint32_t gv, uint32_t gu) {
  return du < dv || (du == dv && gv > gu);
}

// entries equal to x from a[p] on (a sorted; 0 when a[p] != x): galloping, then binary search
GL_DEV uint64_t run_length(const uint32_t* a, uint64_t p, uint64_t n, uint32_t x) {
  if (p >= n || a[p] != x) return 0;
  uint64_t lo = p, step = 1, hi;
  for (;;) {
    hi = lo + step;
    if (hi >= n || a[hi] != x) break;
    lo = hi;
    step <<= 1;
  }
  if (hi > n) hi = n;
  ++lo;   // a[lo - 1] == x; the run ends in [lo, hi]
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] == x) lo = mid + 1; else hi = mid;
  }
  return lo - p;
}

// One row's two sorted halves, merged with ties to oe.
struct MergedRow {
  const uint32_t* O;
  const uint32_t* I;
  uint64_t na, nb;
};

// the merged entry at diagonal k; i0 = oe entries before diagonal k0 <= k (a chunk's start)
struct MergedAt {
  uint32_t x;
  uint64_t i, j;   // oe / ie entries before diagonal k
  bool from_o, first;
};
GL_DEV MergedAt merged_at(const MergedRow& r, uint64_t k, uint64_t k0, uint64_t i0) {
  uint64_t lo = k > r.nb ? k - r.nb : 0, hi = i0 + (k - k0);
  if (lo < i0) lo = i0;
  if (hi > r.na) hi = r.na;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (r.O[mid] <= r.I[k - mid - 1]) lo = mid + 1; else hi = mid;
  }
  MergedAt m;
  m.i = lo;
  m.j = k - lo;
  m.from_o = m.i < r.na && (m.j >= r.nb || r.O[m.i] <= r.I[m.j]);
  if (m.from_o) {
    m.x = r.O[m.i];
    m.first = m.i == 0 || r.O[m.i - 1] != m.x;
  } else {
    // every oe copy of x precedes it, so x is in oe iff O[i - 1] == x
    m.x = r.I[m.j];
    m.first = (m.j == 0 || r.I[m.j - 1] != m.x) && (m.i == 0 || r.O[m.i - 1] != m.x);
  }
  return m;
}

GL_DEV uint32_t merged_weight(const MergedRow& r, const MergedAt& m) {
  const uint64_t w = (m.from_o ? run_length(r.O, m.i, r.na, m.x) : 0) + run_length(r.I, m.j, r.nb, m.x);
  return (uint32_t) w;
}

struct LccdRows {
  const uint64_t *oe_rp, *ie_rp;
  const uint32_t *oe_col, *ie_col;
  const uint32_t* deg;   // [tvnum] |oe| + |ie| (outer copies: the owner's value)
  GidOf gid;
  uint32_t ivnum;
  // count pass
  uint64_t* cnt;         // [ivnum + 1] oriented entries per row (cnt[ivnum] stays 0)
  uint32_t* dd;          // [ivnum] deduplicated degree
  // fill pass
  const uint64_t* orp;
  uint32_t* okey;        // gid of the neighbour
  uint32_t* ow;          // weight (one fragment)
  uint64_t* oval;        // several fragments: weight << 32 | lid, sorted with okey afterwards
  GL_DEV MergedRow row(uint32_t v) const {
    const uint64_t ob = oe_rp[v], ib = ie_rp[v];
    return MergedRow{oe_col + ob, ie_col + ib, oe_rp[v + 1] - ob, ie_rp[v + 1] - ib};
  }
  GL_DEV void put(uint64_t at, const MergedRow& r, const MergedAt& m, uint32_t gu) const {
    const uint32_t w = merged_weight(r, m);
    okey[at] = gu;
    if (oval) oval[at] = ((uint64_t) w << 32) | m.x;
    else ow[at] = w;
  }
};

// rows of up to kLccdWarpRow merged entries: one warp per row
template <bool kFill>
__global__ void __launch_bounds__(kTB) k_lccd_rows_warp(LccdRows a) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < a.ivnum; v += warps) {
    const MergedRow r = a.row(v);
    const uint64_t n = r.na + r.nb;
    if (n > kLccdWarpRow) continue;
    const uint32_t dv = a.deg[v], gv = a.gid(v);
    uint64_t i0 = 0, o = kFill ? a.orp[v] : 0;
    uint32_t distinct = 0, kept = 0;
    for (uint64_t k0 = 0; k0 < n; k0 += 32) {
      const uint64_t k = k0 + lane_id();
      MergedAt m{};
      bool keep = false;
      uint32_t gu = 0;
      if (k < n) {
        m = merged_at(r, k, k0, i0);
        if (m.first) {
          gu = a.gid(m.x);
          keep = lccd_keep(dv, a.deg[m.x], gv, gu);
        }
      }
      i0 = __shfl_sync(0xffffffffu, m.i + (m.from_o ? 1 : 0), 31);   // used only when lane 31 had an entry
      if (kFill) {
        const uint32_t mask = __ballot_sync(0xffffffffu, keep);
        if (keep) a.put(o + __popc(mask & ((1u << lane_id()) - 1)), r, m, gu);
        o += __popc(mask);
      } else {
        distinct += m.first && k < n;
        kept += keep;
      }
    }
    if (!kFill) {
      distinct = warp_sum(distinct);
      kept = warp_sum(kept);
      if (lane_id() == 0) {
        a.cnt[v] = kept;
        a.dd[v] = distinct;
      }
    }
  }
}

// longer rows: a CTA per row.  Every CTA takes kTB consecutive rows at a time and walks the long ones.
template <bool kFill>
__global__ void __launch_bounds__(kTB) k_lccd_rows_cta(LccdRows a) {
  __shared__ uint32_t s_rows[kTB];
  __shared__ uint32_t s_scan[kTB / 32 + 1];
  __shared__ uint64_t s_i0[2];
  for (uint64_t base = (uint64_t) blockIdx.x * kTB; base < a.ivnum; base += (uint64_t) gridDim.x * kTB) {
    const uint64_t vv = base + threadIdx.x;
    bool is_long = false;
    if (vv < a.ivnum) {
      const uint32_t v = (uint32_t) vv;
      is_long = (a.oe_rp[v + 1] - a.oe_rp[v]) + (a.ie_rp[v + 1] - a.ie_rp[v]) > kLccdWarpRow;
    }
    uint32_t nlong = 0;
    const uint32_t at = block_excl_scan(is_long ? 1u : 0u, s_scan, &nlong);
    if (is_long) s_rows[at] = (uint32_t) vv;
    if (threadIdx.x == 0) s_i0[0] = 0;
    __syncthreads();
    for (uint32_t t = 0; t < nlong; ++t) {
      const uint32_t v = s_rows[t];
      const MergedRow r = a.row(v);
      const uint64_t n = r.na + r.nb;
      const uint32_t dv = a.deg[v], gv = a.gid(v);
      uint64_t o = kFill ? a.orp[v] : 0;
      uint32_t distinct = 0, kept = 0;
      int par = 0;
      for (uint64_t k0 = 0; k0 < n; k0 += kTB, par ^= 1) {
        const uint64_t k = k0 + threadIdx.x;
        const uint64_t i0 = s_i0[par];
        MergedAt m{};
        bool keep = false;
        uint32_t gu = 0;
        if (k < n) {
          m = merged_at(r, k, k0, i0);
          if (m.first) {
            gu = a.gid(m.x);
            keep = lccd_keep(dv, a.deg[m.x], gv, gu);
          }
          if (threadIdx.x == kTB - 1) s_i0[par ^ 1] = m.i + (m.from_o ? 1 : 0);
        }
        if (kFill) {
          uint32_t total = 0;
          const uint32_t pos = block_excl_scan(keep ? 1u : 0u, s_scan, &total);   // synchronises the CTA
          if (keep) a.put(o + pos, r, m, gu);
          o += total;
        } else {
          distinct += m.first && k < n;
          kept += keep;
          __syncthreads();
        }
      }
      if (!kFill) {
        uint32_t td = 0, tk = 0;
        block_excl_scan(distinct, s_scan, &td);
        block_excl_scan(kept, s_scan, &tk);
        if (threadIdx.x == 0) {
          a.cnt[v] = tk;
          a.dd[v] = td;
        }
      }
      if (threadIdx.x == 0) s_i0[0] = 0;
      __syncthreads();
    }
  }
}

__global__ void k_lccd_degree(const uint64_t* __restrict__ oe_rp, const uint64_t* __restrict__ ie_rp,
                              uint32_t ivnum, uint32_t* deg) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < ivnum) deg[v] = (uint32_t) ((oe_rp[v + 1] - oe_rp[v]) + (ie_rp[v + 1] - ie_rp[v]));
}

__global__ void k_lccd_split(const uint64_t* __restrict__ val, uint64_t om, uint32_t* olid, uint32_t* ow) {
  for (uint64_t p = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; p < om; p += (uint64_t) gridDim.x * blockDim.x) {
    const uint64_t x = val[p];
    olid[p] = (uint32_t) x;
    ow[p] = (uint32_t) (x >> 32);
  }
}

__global__ void k_lccd_orient_src(const uint64_t* __restrict__ orp, uint32_t ivnum, uint32_t* osrc) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps)
    for (uint64_t p = orp[v] + lane_id(); p < orp[v + 1]; p += 32) osrc[p] = v;
}

struct LccDirectedApp : TriangleApp<true> {
  DevBuf<uint32_t> dd;   // [ivnum] deduplicated degree

  int Setup() override {
    // the reference runs LCCDirected on kBothOutIn directed fragments only
    if (!fv.directed) {
      set_error("lcc_directed needs a directed fragment; GL_APP_LCC is the local clustering coefficient of an "
                "undirected one");
      return GL_ERR_ARG;
    }
    if (frag->ie_alias_oe) {
      set_error("lcc_directed needs the incoming adjacency (gl_frag_desc.ie / kBothOutIn)");
      return GL_ERR_ARG;
    }
    GL_CUDA(dd.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    return TriangleApp::Setup();
  }

  // PEval: degrees, then the oriented rows with their weights (lcc_directed.h:146-240)
  int PEval() override {
    cudaStream_t s = eng.stream;
    const GidOf gid{fv.ivnum, fv.fid, fv.fid_offset, fv.ovgid};
    if (fv.ivnum) GL_LAUNCH(k_lccd_degree, (fv.ivnum + 255) / 256, 256, s, fv.oe_rp, fv.ie_rp, fv.ivnum, deg.get());
    if (fv.fnum > 1) GL_TRY(mm.SyncValuesToGhosts(s, deg, 4));
    LccdRows a{fv.oe_rp, fv.ie_rp, fv.oe_col, fv.ie_col, deg, gid, fv.ivnum, cnt, dd, orp, nullptr, nullptr, nullptr};
    GL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(uint64_t) * ((size_t) fv.ivnum + 1), s));
    if (fv.ivnum) {
      GL_LAUNCH(k_lccd_rows_warp<false>, eng.sm_count * 8, kTB, s, a);
      GL_LAUNCH(k_lccd_rows_cta<false>, eng.sm_count * 4, kTB, s, a);
    }
    GL_TRY(scan_and_resize());
    if (fv.ivnum && om) {
      a.okey = okey;
      if (fv.fnum == 1) {
        // gid == lid: rows come out sorted, and okey doubles as the lid array
        a.ow = ow;
        GL_LAUNCH(k_lccd_rows_warp<true>, eng.sm_count * 8, kTB, s, a);
        GL_LAUNCH(k_lccd_rows_cta<true>, eng.sm_count * 4, kTB, s, a);
      } else {
        // outer gids do not follow lid order: sort every row by gid, carrying (weight, lid)
        DevBuf<uint64_t> val;
        GL_CUDA(val.alloc(om));
        a.oval = val;
        GL_LAUNCH(k_lccd_rows_warp<true>, eng.sm_count * 8, kTB, s, a);
        GL_LAUNCH(k_lccd_rows_cta<true>, eng.sm_count * 4, kTB, s, a);
        GL_TRY(sort_csr_rows(s, orp, fv.ivnum, om, &okey, &val));
        GL_LAUNCH(k_lccd_split, eng.sm_count * 8, 256, s, val, om, olid, ow);
      }
      GL_LAUNCH(k_lccd_orient_src, eng.sm_count * 8, 256, s, orp, fv.ivnum, osrc);
      GL_CUDA(cudaStreamSynchronize(s));
    }
    GL_TRY(peers.replicate(mm, s, fv, orp, okey, om, ow));
    mm.ForceContinue();
    return GL_OK;
  }

  int Result(void* host_out, size_t) override { return WriteResult(host_out, dd, 1.0); }
};

}  // namespace

gl_app* make_lcc_directed() { return new LccDirectedApp; }

}  // namespace gl
