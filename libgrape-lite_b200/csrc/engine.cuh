// engine.cuh — the vertex/edge-parallel engine (kernel skeletons).
//
// Replaces grape::cuda::ParallelEngine::ForEach{Outgoing,Incoming}Edge and its
// load-balancing device functions LBNONE/LBCM/LBWARP/LBCTA/LBSTRICT
// (grape/cuda/parallel/parallel_engine.h:621-979, 987-1434).  The skeletons
// are templates over an edge operator `Op` so that the library's fixed
// functions (apps.cu) and user device lambdas (compat headers) instantiate the
// SAME hand-written kernels.
//
// Design: a superstep never round-trips to the host to size its work.
//  * The frontier is a bitmap.  `k_frontier_scan` fuses "scan bitmap ->
//    compact -> degree prefix -> edge scan": a CTA draws tiles of 1024
//    vertices from a device ticket, expands the set bits into shared memory,
//    prefix-sums the row lengths and walks the tile's edges CTA-cooperatively
//    (the reference's `cm` mapping) — without the reference's separate O(V)
//    compaction pass, DeviceScan launches, cudaMallocAsync and stream sync
//    (parallel_engine.h:1396-1434).
//  * Rows longer than kHubDeg are not walked inside the tile (one CTA would
//    serialise a 10^5-entry R-MAT hub); they are cut into kHubChunk-entry
//    pieces on a device work list that `k_hub_scan` spreads over all SMs with
//    128-bit coalesced loads.
//  * Every kernel is a persistent grid of (SMs x resident CTAs) blocks.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace gl {

constexpr int kTB = 256;          // threads per CTA
constexpr int kTileV = 1024;      // vertices per tile (32 bitmap words)
constexpr uint32_t kHubDeg = 1024;    // rows longer than this go to the hub list
constexpr uint32_t kHubChunk = 1024;  // entries per hub work item

// Device control block of one engine (zeroed per superstep by k_ctrl_reset).
struct ScanCtrl {
  unsigned int tile_ticket;
  unsigned int hub_count;
  unsigned int hub_ticket;
  unsigned int aux_ticket;
  unsigned long long scanned;     // CSR entries read
  unsigned long long frontier;    // vertices expanded
  unsigned long long next_count;  // vertices newly activated (local)
  unsigned long long next_edges;  // sum of their degrees
  unsigned long long remote_count;  // outer vertices updated
  unsigned long long aux;         // op-specific (e.g. far-set size)
  unsigned long long touched;     // state writes
  unsigned long long pad;
};

struct HubItem {
  uint32_t v;
  uint32_t pad;
  uint64_t begin, end;
};

struct EdgeRange {  // which adjacency of the fragment to scan
  const uint64_t* rp;
  const uint32_t* col;
  const void* w;
};

// per-thread accumulators flushed once per kernel
struct ScanAcc {
  uint32_t next_count = 0;
  uint64_t next_edges = 0;
  uint32_t remote = 0;
  uint32_t aux = 0;
  uint32_t touched = 0;
};

#ifdef __CUDACC__

GL_DEV uint32_t warp_incl_scan(uint32_t x) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane_id() >= (uint32_t) o) x += y;
  }
  return x;
}

// exclusive scan over the CTA's kTB threads; returns exclusive prefix, writes
// the CTA total to *total.  s_warp: 8-word shared scratch.
GL_DEV uint32_t block_excl_scan(uint32_t x, uint32_t* s_warp, uint32_t* total) {
  uint32_t incl = warp_incl_scan(x);
  uint32_t wid = threadIdx.x >> 5;
  if (lane_id() == 31) s_warp[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    uint32_t v = lane_id() < (kTB / 32) ? s_warp[lane_id()] : 0;
    uint32_t vi = warp_incl_scan(v);
    if (lane_id() < (kTB / 32)) s_warp[lane_id()] = vi - v;
    if (lane_id() == (kTB / 32) - 1) s_warp[kTB / 32] = vi;
  }
  __syncthreads();
  uint32_t r = incl - x + s_warp[wid];
  *total = s_warp[kTB / 32];
  __syncthreads();
  return r;
}

template <typename T>
GL_DEV T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Ops that need the CSR position of the entry they are handed (the reference's
// GetOutgoingEdgeIndex(u, nbr) idiom: `&nbr - row begin`, device_fragment.h:398-421)
// declare `static constexpr bool kWantsPos = true` and implement
// edge_at(u, meta, v, w, pos, acc); everybody else keeps edge(u, meta, v, w, acc)
// and compiles to exactly the same code as before.
template <class Op, class = void>
struct op_wants_pos : std::false_type {};
template <class Op>
struct op_wants_pos<Op, std::void_t<decltype(Op::kWantsPos)>> : std::integral_constant<bool, Op::kWantsPos> {};
template <class Op, class M, class W>
GL_DEV void call_edge(const Op& op, uint32_t u, const M& m, uint32_t v, W w, uint64_t pos, ScanAcc& acc) {
  if constexpr (op_wants_pos<Op>::value) op.edge_at(u, m, v, w, pos, acc);
  else op.edge(u, m, v, w, acc);
}

GL_DEV void flush_acc(const ScanAcc& a, ScanCtrl* c) {
  uint32_t nc = warp_sum(a.next_count);
  unsigned long long ne = warp_sum((unsigned long long) a.next_edges);
  uint32_t rm = warp_sum(a.remote);
  uint32_t ax = warp_sum(a.aux);
  uint32_t tc = warp_sum(a.touched);
  if (lane_id() == 0) {
    if (nc) atomicAdd(&c->next_count, (unsigned long long) nc);
    if (ne) atomicAdd(&c->next_edges, ne);
    if (rm) atomicAdd(&c->remote_count, (unsigned long long) rm);
    if (ax) atomicAdd(&c->aux, (unsigned long long) ax);
    if (tc) atomicAdd(&c->touched, (unsigned long long) tc);
  }
}

template <typename W>
GL_DEV W load_w(const void* w, uint64_t pos) {
  return w ? ((const W*) w)[pos] : (W) 1;
}

// ---------------------------------------------------------------------------
// Frontier scan phase: fused bitmap -> tile list -> CTA-cooperative edge walk.
// Written as a __device__ phase so that the stand-alone kernel
// (k_frontier_scan) and the fused whole-query kernels (one cooperative launch
// per query, grid.sync between supersteps) share the same code.
// Op requirements:
//   using Meta = ...; using W = float|double;
//   static constexpr bool kWeighted;
//   Meta assign(uint32_t u) const;
//   void edge(uint32_t u, Meta m, uint32_t v, W w, ScanAcc& acc) const;
// ---------------------------------------------------------------------------
constexpr int kSuperTiles = 8;                    // tiles per ticket
constexpr int kSuperV = kTileV * kSuperTiles;     // 8192 vertices = 256 words
constexpr int kMaxTileHubs = 32;                  // long rows emitted cooperatively per tile

template <class Meta>
struct ScanSmem {
  uint32_t v[kTileV];
  uint64_t rp[kTileV];
  uint32_t pfx[kTileV + 1];
  Meta meta[kTileV];
  uint32_t words[kTB];
  uint32_t warp[kTB / 32 + 1];
  uint32_t nz[kSuperTiles];
  uint32_t ticket;
  uint32_t hubn, hubbase;       // long rows met in the current tile
  uint32_t hubidx[kMaxTileHubs];
};

// Draws the next super-tile (8192 bits) and stages its words in shared memory.
// `word_of(widx)` returns the candidate word.  Returns false when the work is
// exhausted; sm.nz[k] tells whether sub-tile k has any set bit.
// (Tickets of several super-tiles -- fetched together, one atomic per batch -- were measured on
//  the BFS tail levels: consecutive ones tripled them (expensive super-tiles come in runs in a
//  degree-ordered graph), strided ones were 2 us per level slower than this.)
template <class SM, class WordFn>
GL_DEV bool next_super_tile(SM& sm, unsigned int* ticket, uint32_t nverts,
                            WordFn word_of, uint32_t* super_out) {
  const uint32_t nsuper = (nverts + kSuperV - 1) / kSuperV;
  const uint32_t nwords = (nverts + 31) / 32;
  for (;;) {
    if (threadIdx.x == 0) sm.ticket = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t st = sm.ticket;
    if (st >= nsuper) return false;
    const uint32_t widx = st * (kSuperV / 32) + threadIdx.x;
    const uint32_t word = widx < nwords ? word_of(widx) : 0u;
    sm.words[threadIdx.x] = word;
    const bool any_w = __any_sync(0xffffffffu, word != 0);
    if (lane_id() == 0) sm.nz[threadIdx.x >> 5] = any_w;
    const int any = __syncthreads_or(word != 0);
    if (any) {
      *super_out = st;
      return true;
    }
  }
}

// The hub list is sized for a frontier, where a row appears once.  A queue may repeat an entry
// (ForEach over an array processes every entry), so a queue of copies of one long row can emit
// more work items than the list holds.  Ops that can be handed such a queue declare
// `static constexpr bool kHubOverflowInline = true`: the entries of the items past hub_cap are
// then walked where the row was met instead of being dropped.  Everybody else compiles to
// exactly the same code as before.
template <class Op, class = void>
struct op_hub_overflow_inline : std::false_type {};
template <class Op>
struct op_hub_overflow_inline<Op, std::void_t<decltype(Op::kHubOverflowInline)>>
    : std::integral_constant<bool, Op::kHubOverflowInline> {};

// first entry of row [b, e) that did not fit into the hub list (e if all of it did)
GL_DEV uint64_t hub_overflow_begin(uint64_t b, uint64_t e, uint32_t at, uint32_t pieces, uint32_t hub_cap) {
  if ((uint64_t) at + pieces <= hub_cap) return e;
  return b + (uint64_t) (at < hub_cap ? hub_cap - at : 0) * kHubChunk;
}

template <class Op>
GL_DEV void hub_push(uint32_t v, uint64_t b, uint64_t e, ScanCtrl* ctrl,
                     HubItem* hubs, uint32_t hub_cap, EdgeRange er, const Op& op, ScanAcc& acc) {
  const uint64_t dg = e - b;
  uint32_t pieces = (uint32_t) ((dg + kHubChunk - 1) / kHubChunk);
  uint32_t at = atomicAdd(&ctrl->hub_count, pieces);
  for (uint32_t p = 0; p < pieces; ++p) {
    if (at + p < hub_cap) {
      HubItem h;
      h.v = v;
      h.pad = 0;
      h.begin = b + (uint64_t) p * kHubChunk;
      h.end = (h.begin + kHubChunk < e) ? h.begin + kHubChunk : e;
      hubs[at + p] = h;
    }
  }
  if constexpr (op_hub_overflow_inline<Op>::value) {
    using W = typename Op::W;
    const uint64_t ob = hub_overflow_begin(b, e, at, pieces, hub_cap);
    if (ob < e) {  // this thread alone met the row: walk the rest serially
      const auto meta = op.assign(v);
      for (uint64_t p = ob; p < e; ++p) {
        W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
        call_edge(op, v, meta, er.col[p], w, p, acc);
      }
      atomicAdd(&ctrl->scanned, (unsigned long long) (e - ob));
    }
  }
}

// Walks the edges of the sm.v[0..nf) vertex list CTA-cooperatively.
template <class Op>
GL_DEV void walk_tile(ScanSmem<typename Op::Meta>& sm, uint32_t nf, EdgeRange er,
                      const Op& op, ScanCtrl* ctrl, HubItem* hubs, uint32_t hub_cap,
                      uint32_t hub_deg, ScanAcc& acc, uint64_t& scanned) {
  using W = typename Op::W;
  // row extents; thread t owns list items [4t, 4t+4)
  uint32_t dsum = 0;
  uint32_t degs[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t i = threadIdx.x * 4 + k;
    degs[k] = 0;
    if (i < nf) {
      uint32_t v = sm.v[i];
      uint64_t b = er.rp[v], e = er.rp[v + 1];
      uint64_t dg = e - b;
      sm.rp[i] = b;
      sm.meta[i] = op.assign(v);
      if (dg > hub_deg) {
        // long row: handed to the hub phase; its work items are written by
        // the whole CTA below (a single thread emitting 700 items of the
        // source hub costs tens of microseconds)
        uint32_t slot = atomicAdd(&sm.hubn, 1u);
        if (slot < (uint32_t) kMaxTileHubs) sm.hubidx[slot] = i;
        else hub_push<Op>(v, b, e, ctrl, hubs, hub_cap, er, op, acc);
        dg = 0;
      }
      degs[k] = (uint32_t) dg;
      dsum += degs[k];
    }
  }
  uint32_t total;
  uint32_t doff = block_excl_scan(dsum, sm.warp, &total);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t i = threadIdx.x * 4 + k;
    if (i < nf) {
      sm.pfx[i] = doff;
      doff += degs[k];
    }
  }
  if (threadIdx.x == 0) sm.pfx[nf] = total;
  __syncthreads();
  const uint32_t nh = sm.hubn < (uint32_t) kMaxTileHubs ? sm.hubn : (uint32_t) kMaxTileHubs;
  if (nh) {  // uniform
    for (uint32_t h = 0; h < nh; ++h) {
      const uint32_t i = sm.hubidx[h];
      const uint32_t v = sm.v[i];
      const uint64_t b = sm.rp[i], e = er.rp[v + 1];
      const uint32_t pieces = (uint32_t) ((e - b + kHubChunk - 1) / kHubChunk);
      if (threadIdx.x == 0) sm.hubbase = atomicAdd(&ctrl->hub_count, pieces);
      __syncthreads();
      const uint32_t at = sm.hubbase;
      for (uint32_t p = threadIdx.x; p < pieces; p += kTB) {
        if (at + p < hub_cap) {
          HubItem it;
          it.v = v;
          it.pad = 0;
          it.begin = b + (uint64_t) p * kHubChunk;
          it.end = (it.begin + kHubChunk < e) ? it.begin + kHubChunk : e;
          hubs[at + p] = it;
        }
      }
      if constexpr (op_hub_overflow_inline<Op>::value) {
        using W = typename Op::W;
        const uint64_t ob = hub_overflow_begin(b, e, at, pieces, hub_cap);
        if (ob < e) {  // uniform: the CTA walks the entries that did not fit
          const auto meta = sm.meta[i];
          for (uint64_t p = ob + threadIdx.x; p < e; p += kTB) {
            W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
            call_edge(op, v, meta, ld_stream_u32(er.col + p), w, p, acc);
          }
          if (threadIdx.x == 0) scanned += e - ob;
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) sm.hubn = 0;
  }
  for (uint32_t e0 = 0; e0 < total; e0 += kTB) {
    uint32_t e = e0 + threadIdx.x;
    if (e < total) {
      // largest j with pfx[j] <= e
      uint32_t lo = 0, hi = nf;
      while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (sm.pfx[mid] <= e) lo = mid; else hi = mid;
      }
      uint64_t pos = sm.rp[lo] + (e - sm.pfx[lo]);
      uint32_t v = ld_stream_u32(er.col + pos);
      W w = Op::kWeighted ? load_w<W>(er.w, pos) : (W) 1;
      call_edge(op, sm.v[lo], sm.meta[lo], v, w, pos, acc);
    }
  }
  if (threadIdx.x == 0) scanned += total;
  __syncthreads();
}

template <class Op>
GL_DEV void frontier_scan_phase(ScanSmem<typename Op::Meta>& sm,
                                const uint32_t* __restrict__ frontier,
                                uint32_t nverts, EdgeRange er, const Op& op,
                                ScanCtrl* ctrl, HubItem* hubs, uint32_t hub_cap,
                                uint32_t hub_deg, ScanAcc& acc) {
  uint64_t scanned = 0;
  uint32_t expanded = 0;
  uint32_t st;
  if (threadIdx.x == 0) sm.hubn = 0;
  __syncthreads();
  // bits at positions >= nverts (outer copies sharing the last word when nverts
  // is not a multiple of 32) are not frontier vertices of this scan
  const uint32_t last_w = nverts >> 5, last_mask = (1u << (nverts & 31)) - 1u;
  while (next_super_tile(sm, &ctrl->tile_ticket, nverts,
                         [&](uint32_t w) { return w == last_w ? (frontier[w] & last_mask) : frontier[w]; }, &st)) {
    for (int k = 0; k < kSuperTiles; ++k) {
      if (!sm.nz[k]) continue;  // uniform
      // expand the sub-tile's set bits: thread t owns bits [4t, 4t+4)
      uint32_t word = sm.words[k * 32 + (threadIdx.x >> 3)];
      uint32_t nib = (word >> ((threadIdx.x & 7) * 4)) & 0xFu;
      uint32_t nf;
      uint32_t off = block_excl_scan(__popc(nib), sm.warp, &nf);
      const uint32_t vbase = st * kSuperV + k * kTileV + threadIdx.x * 4;
      while (nib) {
        uint32_t b = __ffs(nib) - 1;
        nib &= nib - 1;
        sm.v[off++] = vbase + b;
      }
      __syncthreads();
      expanded += (threadIdx.x == 0) ? nf : 0;
      walk_tile<Op>(sm, nf, er, op, ctrl, hubs, hub_cap, hub_deg, acc, scanned);
    }
  }
  if (threadIdx.x == 0) {
    if (scanned) atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
    if (expanded) atomicAdd(&ctrl->frontier, (unsigned long long) expanded);
  }
}

// Ops whose per-entry work is a bit set in a bitmap can take a whole warp's entries at once
// (Op::kWarpEntries + Op::warp_edge): the hub phase then hands over 32 consecutive entries of the
// row per call, all lanes converged.
template <class Op, class = void>
struct has_warp_entries : std::false_type {};
template <class Op>
struct has_warp_entries<Op, std::void_t<decltype(Op::kWarpEntries)>> : std::true_type {};

// Hub phase: one work item = <= kHubChunk consecutive entries of one long row,
// read with 128-bit coalesced loads.
template <class Op>
GL_DEV void hub_scan_phase(uint32_t* s_item, EdgeRange er, const Op& op,
                           ScanCtrl* ctrl, const HubItem* hubs, uint32_t hub_cap,
                           ScanAcc& acc) {
  using W = typename Op::W;
  uint64_t scanned = 0;
  uint32_t n = ctrl->hub_count;
  if (n > hub_cap) n = hub_cap;
  for (;;) {
    if (threadIdx.x == 0) *s_item = atomicAdd(&ctrl->hub_ticket, 1u);
    __syncthreads();
    uint32_t it = *s_item;
    __syncthreads();
    if (it >= n) break;
    HubItem h = hubs[it];
    auto meta = op.assign(h.v);
    uint64_t b = h.begin, e = h.end;
    if constexpr (has_warp_entries<Op>::value) {
      // warp w of the CTA takes entries [b + 32 w, b + 32 w + 32), then strides by the CTA width
      for (uint64_t base = b + (threadIdx.x & ~31u); base < e; base += kTB) {
        const uint64_t p = base + lane_id();
        const bool valid = p < e;
        const uint32_t v = valid ? ld_stream_u32(er.col + p) : 0u;
        op.warp_edge(v, valid, acc);
      }
      if (threadIdx.x == 0) scanned += e - b;
      continue;
    }
    uint64_t ab = (b + 3) & ~3ull;
    if (ab > e) ab = e;
    uint64_t ae = ab + ((e - ab) & ~3ull);
    for (uint64_t p = b + threadIdx.x; p < ab; p += kTB) {
      uint32_t v = ld_stream_u32(er.col + p);
      W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
      call_edge(op, h.v, meta, v, w, p, acc);
    }
    for (uint64_t p = ab + 4ull * threadIdx.x; p < ae; p += 4ull * kTB) {
      uint4 c = ld_stream_u4((const uint4*) (er.col + p));
      W w0 = (W) 1, w1 = (W) 1, w2 = (W) 1, w3 = (W) 1;
      if (Op::kWeighted && er.w) {
        const W* wp = (const W*) er.w + p;
        w0 = wp[0]; w1 = wp[1]; w2 = wp[2]; w3 = wp[3];
      }
      call_edge(op, h.v, meta, c.x, w0, p, acc);
      call_edge(op, h.v, meta, c.y, w1, p + 1, acc);
      call_edge(op, h.v, meta, c.z, w2, p + 2, acc);
      call_edge(op, h.v, meta, c.w, w3, p + 3, acc);
    }
    for (uint64_t p = ae + threadIdx.x; p < e; p += kTB) {
      uint32_t v = ld_stream_u32(er.col + p);
      W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
      call_edge(op, h.v, meta, v, w, p, acc);
    }
    if (threadIdx.x == 0) scanned += e - b;
  }
  if (threadIdx.x == 0 && scanned)
    atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}


// Hub phase with the TMA engine staging the work items (north star: "TMA bulk
// staging of CSR column-index tiles into shared memory"): the next item's
// <= 1024 column indices (and f32 weights) stream into shared memory through
// cp.async.bulk + mbarrier (SASS UBLKCP) while the CTA walks the current one.
// Items start at arbitrary positions of a row: the copy starts at the enclosing
// 16-byte boundary (col / w allocations are padded past their last entry).
struct HubTmaSmem {
  uint32_t col[2][kHubChunk + 16];
  float w[2][kHubChunk + 16];
  uint64_t bar[2];
  uint32_t item[2];
};

template <class Op>
GL_DEV void hub_scan_phase_tma(HubTmaSmem& sm, EdgeRange er, const Op& op, ScanCtrl* ctrl, const HubItem* hubs,
                               uint32_t hub_cap, ScanAcc& acc) {
  using W = typename Op::W;
  static_assert(sizeof(W) == 4, "the staged weights are 4 bytes wide");
  uint64_t scanned = 0;
  uint32_t n = ctrl->hub_count;
  if (n > hub_cap) n = hub_cap;
  const bool with_w = Op::kWeighted && er.w != nullptr;
  auto issue = [&](int stage, const HubItem& h) {
    const uint64_t a = h.begin & ~3ull;
    const uint32_t len = (uint32_t) (((h.end - a) + 3) & ~3ull);
    const uint32_t bytes = len * 4u;
    mbar_expect_tx(&sm.bar[stage], with_w ? 2u * bytes : bytes);
    tma_load_1d(&sm.col[stage][0], er.col + a, bytes, &sm.bar[stage]);
    if (with_w) tma_load_1d(&sm.w[stage][0], (const float*) er.w + a, bytes, &sm.bar[stage]);
  };
  if (threadIdx.x == 0) {
    mbar_init(&sm.bar[0], 1);
    mbar_init(&sm.bar[1], 1);
    mbar_fence_init();
    const uint32_t first = atomicAdd(&ctrl->hub_ticket, 1u);
    sm.item[0] = first;
    if (first < n) issue(0, hubs[first]);
  }
  __syncthreads();
  for (uint32_t k = 0;; ++k) {
    const int stage = (int) (k & 1);
    const uint32_t cur = sm.item[stage];
    if (cur >= n) break;   // uniform: read after a CTA barrier
    if (threadIdx.x == 0) {
      const uint32_t nxt = atomicAdd(&ctrl->hub_ticket, 1u);
      sm.item[stage ^ 1] = nxt;
      if (nxt < n) issue(stage ^ 1, hubs[nxt]);   // slot stage^1 was drained before the last barrier
    }
    const HubItem h = hubs[cur];
    const auto meta = op.assign(h.v);
    const uint64_t a = h.begin & ~3ull;
    mbar_wait_parity(&sm.bar[stage], (k >> 1) & 1);
    const uint32_t lo = (uint32_t) (h.begin - a), hi = (uint32_t) (h.end - a);
    for (uint32_t i = lo + threadIdx.x; i < hi; i += kTB) {
      const uint32_t v = sm.col[stage][i];
      W w = (W) 1;
      if (with_w) w = (W) sm.w[stage][i];
      call_edge(op, h.v, meta, v, w, a + i, acc);
    }
    if (threadIdx.x == 0) scanned += h.end - h.begin;
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0 && scanned) atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}

template <class Op>
__global__ void __launch_bounds__(kTB)
k_frontier_scan(const uint32_t* __restrict__ frontier, uint32_t nverts,
                EdgeRange er, Op op, ScanCtrl* ctrl, HubItem* hubs,
                uint32_t hub_cap, uint32_t hub_deg) {
  __shared__ ScanSmem<typename Op::Meta> sm;
  ScanAcc acc;
  frontier_scan_phase<Op>(sm, frontier, nverts, er, op, ctrl, hubs, hub_cap, hub_deg, acc);
  flush_acc(acc, ctrl);
}

// ops with 4-byte weights (or none) can take the TMA-staged hub phase
template <class Op>
struct op_tma_ok : std::integral_constant<bool, sizeof(typename Op::W) == 4> {};

template <class Op>
__global__ void __launch_bounds__(kTB)
k_hub_scan(EdgeRange er, Op op, ScanCtrl* ctrl, const HubItem* hubs,
           uint32_t hub_cap) {
  __shared__ uint32_t s_item;
  ScanAcc acc;
  hub_scan_phase<Op>(&s_item, er, op, ctrl, hubs, hub_cap, acc);
  flush_acc(acc, ctrl);
}

template <class Op>
__global__ void __launch_bounds__(kTB)
k_hub_scan_tma(EdgeRange er, Op op, ScanCtrl* ctrl, const HubItem* hubs, uint32_t hub_cap) {
  __shared__ __align__(128) HubTmaSmem sm;
  ScanAcc acc;
  if constexpr (op_tma_ok<Op>::value) hub_scan_phase_tma<Op>(sm, er, op, ctrl, hubs, hub_cap, acc);
  flush_acc(acc, ctrl);
}

// Work sources (grape/cuda/utils/work_source.h): item i -> vertex id
struct ArraySrc {
  const uint32_t* q;
  GL_DEV uint32_t operator()(uint32_t i) const { return q[i]; }
};
struct RangeSrc {
  uint32_t start;
  GL_DEV uint32_t operator()(uint32_t i) const { return start + i; }
};

// ---------------------------------------------------------------------------
// Queue-driven variants (WorkSourceArray / WorkSourceRange): the LB modes.
// ---------------------------------------------------------------------------
// LB none: thread per vertex, serial row walk (LBNONE, :621-646)
template <class Op, class Src = ArraySrc>
__global__ void __launch_bounds__(kTB)
k_queue_scan_none(Src q, uint32_t n, EdgeRange er,
                  Op op, ScanCtrl* ctrl) {
  using W = typename Op::W;
  ScanAcc acc;
  uint64_t scanned = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += gridDim.x * blockDim.x) {
    uint32_t u = q(i);
    auto m = op.assign(u);
    uint64_t b = er.rp[u], e = er.rp[u + 1];
    for (uint64_t p = b; p < e; ++p) {
      W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
      call_edge(op, u, m, er.col[p], w, p, acc);
    }
    scanned += e - b;
  }
  flush_acc(acc, ctrl);
  unsigned long long s = warp_sum((unsigned long long) scanned);
  if (lane_id() == 0 && s) atomicAdd(&ctrl->scanned, s);
}

// LB wm: a warp takes 32 queue entries, scans their degrees and the lanes
// sweep the concatenated edges (LBWARP, :773-845)
template <class Op, class Src = ArraySrc>
__global__ void __launch_bounds__(kTB)
k_queue_scan_warp(Src q, uint32_t n, EdgeRange er,
                  Op op, ScanCtrl* ctrl) {
  using W = typename Op::W;
  using Meta = typename Op::Meta;
  ScanAcc acc;
  uint64_t scanned = 0;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  for (uint32_t base = wid * 32; base < n; base += warps * 32) {
    uint32_t i = base + lane_id();
    uint32_t u = 0;
    uint64_t b = 0;
    uint32_t dg = 0;
    Meta m = Meta();
    if (i < n) {
      u = q(i);
      b = er.rp[u];
      uint64_t d64 = er.rp[u + 1] - b;
      dg = d64 > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t) d64;
      m = op.assign(u);
    }
    uint32_t incl = warp_incl_scan(dg);
    uint32_t excl = incl - dg;
    uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    const uint32_t rounds = (total + 31) >> 5;
    for (uint32_t r = 0; r < rounds; ++r) {
      const uint32_t e = (r << 5) + lane_id();
      const bool active = e < total;
      // owner lane = largest l with excl_l <= e (excl is non-decreasing)
      uint32_t lo = 0, hi = 32;
#pragma unroll
      for (int it = 0; it < 5; ++it) {
        uint32_t mid = (lo + hi) >> 1;
        uint32_t ex = __shfl_sync(0xffffffffu, excl, mid);
        if (ex <= e) lo = mid; else hi = mid;
      }
      const uint32_t owner = lo;
      uint32_t ou = __shfl_sync(0xffffffffu, u, owner);
      uint32_t oex = __shfl_sync(0xffffffffu, excl, owner);
      uint32_t blo = __shfl_sync(0xffffffffu, (uint32_t) b, owner);
      uint32_t bhi = __shfl_sync(0xffffffffu, (uint32_t) (b >> 32), owner);
      Meta om = __shfl_sync(0xffffffffu, m, owner);
      if (active) {
        uint64_t p = (((uint64_t) bhi << 32) | blo) + (e - oex);
        W w = Op::kWeighted ? load_w<W>(er.w, p) : (W) 1;
        call_edge(op, ou, om, er.col[p], w, p, acc);
      }
    }
    scanned += dg;
  }
  flush_acc(acc, ctrl);
  unsigned long long s = warp_sum((unsigned long long) scanned);
  if (lane_id() == 0 && s) atomicAdd(&ctrl->scanned, s);
}

// Queue scan phase: a CTA takes kTileV queue entries per ticket and walks them
// with the same tile walk as the frontier scan; rows longer than hub_deg go to
// the hub list.  A __device__ phase so that the stand-alone kernel
// (k_queue_scan_cta) and fused whole-query kernels share it.
template <class Op, class Src = ArraySrc>
GL_DEV void queue_scan_phase(ScanSmem<typename Op::Meta>& sm, Src q, uint32_t n, EdgeRange er,
                             const Op& op, ScanCtrl* ctrl, HubItem* hubs, uint32_t hub_cap,
                             uint32_t hub_deg, ScanAcc& acc) {
  const uint32_t ntiles = (n + kTileV - 1) / kTileV;
  uint64_t scanned = 0;
  if (threadIdx.x == 0) sm.hubn = 0;
  __syncthreads();
  for (;;) {
    if (threadIdx.x == 0) sm.ticket = atomicAdd(&ctrl->tile_ticket, 1u);
    __syncthreads();
    const uint32_t tile = sm.ticket;
    if (tile >= ntiles) break;
    const uint32_t base = tile * kTileV;
    const uint32_t nf = (n - base) < (uint32_t) kTileV ? (n - base) : (uint32_t) kTileV;
    for (uint32_t i = threadIdx.x; i < nf; i += kTB) sm.v[i] = q(base + i);
    __syncthreads();
    walk_tile<Op>(sm, nf, er, op, ctrl, hubs, hub_cap, hub_deg, acc, scanned);
  }
  if (threadIdx.x == 0 && scanned)
    atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}

// LB cm / cta: the queue scan phase as a kernel (cm keeps every row in the
// tile: hub_deg = UINT32_MAX; cta defers long rows to k_hub_scan).
template <class Op, class Src = ArraySrc>
__global__ void __launch_bounds__(kTB)
k_queue_scan_cta(Src q, uint32_t n, EdgeRange er,
                 Op op, ScanCtrl* ctrl, HubItem* hubs, uint32_t hub_cap,
                 uint32_t hub_deg) {
  __shared__ ScanSmem<typename Op::Meta> sm;
  ScanAcc acc;
  queue_scan_phase<Op, Src>(sm, q, n, er, op, ctrl, hubs, hub_cap, hub_deg, acc);
  flush_acc(acc, ctrl);
}

// LB strict: exact edge balance.  pfx[i] = exclusive prefix of the queue's
// degrees (pfx[n] = total); CTA c owns entries [c*per, (c+1)*per)
// (LBSTRICT :881-979, without the host-side sorted_search / allocations).
template <class Op, class Src = ArraySrc>
__global__ void __launch_bounds__(kTB)
k_queue_scan_strict(Src q, uint32_t n,
                    const uint64_t* __restrict__ pfx, EdgeRange er, Op op,
                    ScanCtrl* ctrl) {
  using W = typename Op::W;
  ScanAcc acc;
  const uint64_t total = pfx[n];
  const uint64_t per = (total + gridDim.x - 1) / gridDim.x;
  const uint64_t lo_e = per * blockIdx.x;
  uint64_t hi_e = lo_e + per;
  if (hi_e > total) hi_e = total;
  for (uint64_t e = lo_e + threadIdx.x; e < hi_e; e += kTB) {
    // largest j with pfx[j] <= e
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (pfx[mid] <= e) lo = mid; else hi = mid;
    }
    uint32_t u = q(lo);
    uint64_t pos = er.rp[u] + (e - pfx[lo]);
    W w = Op::kWeighted ? load_w<W>(er.w, pos) : (W) 1;
    call_edge(op, u, op.assign(u), ld_stream_u32(er.col + pos), w, pos, acc);
  }
  flush_acc(acc, ctrl);
  if (threadIdx.x == 0 && hi_e > lo_e)
    atomicAdd(&ctrl->scanned, (unsigned long long) (hi_e - lo_e));
}

template <class Src = ArraySrc>
__global__ void k_queue_degrees(Src q, uint32_t n, const uint64_t* rp, uint64_t* deg) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint32_t u = q(i);
    deg[i] = rp[u + 1] - rp[u];
  }
  if (i == n) deg[i] = 0;
}

#endif  // __CUDACC__
}  // namespace gl
