// app_bfs.cu — direction-optimising level-synchronous BFS.
//
// Behaviour follows examples/analytical_apps/cuda/bfs/bfs.h:25-273 (PEval
// :86-133 seeds the source, IncEval :135-271 expands one level, push or pull)
// and the CPU app bfs/bfs.h:44-212.  Result: int64 depth per inner vertex,
// unreachable = INT64_MAX (bfs.h:31,40-45).  Levels are order-independent, so
// any push/pull schedule yields bit-identical output.
//
// Re-design
//  * No per-vertex depth array on the hot path.  Level d IS a bitmap
//    (lv[d], 2 MB at scale 24) plus one visited bitmap; both stay L2 resident.
//    The int64 depth array the reference exposes is materialised once, with
//    coalesced reads/writes, when the result is requested.  This removes the
//    reference's scattered 8-byte depth writes (bfs.h:195-196) and the 8 B x V
//    state initialisation from every query.
//  * Push levels run the engine's fused frontier scan (engine.cuh).
//  * Pull levels test, for every unvisited vertex, its highest-degree
//    neighbour first (hub_nbr[], built once in Setup like the reference's
//    PrepareToRunApp artefacts): one coalesced 4-byte load + one L2-resident
//    bitmap probe resolves most candidates without touching row pointers or
//    column indices; the rest fall back to the row scan of bfs.h:239-259.
//  * Single fragment: the whole query is ONE cooperative launch
//    (k_bfs_fused); grid.sync() replaces the reference's 4 host
//    synchronisations per round (bfs.h:169-170,189,263).  Multi-fragment runs
//    keep one launch group per superstep around the halo exchange.
#include <cooperative_groups.h>

#include <thread>

#include "host_pool.h"

#include "apps_common.cuh"

namespace cg = cooperative_groups;

#ifndef GL_BFS_FUSED_CTAS
#define GL_BFS_FUSED_CTAS 4
#endif

namespace gl {
namespace {

struct OpBfsPush {
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* vis;
  uint32_t* nxt;
  uint32_t* remote;
  const uint64_t* rp;
  uint32_t ivnum;
  // Frontier-edge statistic for the push -> pull switch (only read while the query is still in its
  // first push phase).  deg8 != null: one byte per vertex (1 + floor(log2(degree)), L2-resident 16 MB at
  // 2^24 vertices) instead of a random 16-byte row-pointer read per discovered vertex (134 MB array);
  // the estimate 1.5 * 2^(k-1) is within +-33 %, the switch thresholds are an order-of-magnitude rule.
  const uint8_t* deg8 = nullptr;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  static GL_DEV unsigned long long degree_of_class(uint32_t k) {
    return k == 0 ? 0ull : (k == 1 ? 1ull : (3ull << (k - 2)));
  }
  GL_DEV unsigned long long degree_of(uint32_t v) const {
    if (!deg8) return rp[v + 1] - rp[v];
    return degree_of_class(deg8[v]);
  }
  // statistics of a vertex this level visited first; `deg` = degree_of(v) when v is inner
  GL_DEV void note_fresh(uint32_t v, unsigned long long deg, ScanAcc& acc) const {
    acc.touched++;
    if (v < ivnum) {
      acc.next_count++;
      acc.next_edges += deg;
    } else {
      acc.remote++;
    }
  }
  // Hub rows, 32 consecutive entries per call (engine.cuh, has_warp_entries).  The rows of the
  // hub-first shadow graph are sorted, so neighbouring lanes mostly hit the same bitmap word: the
  // lanes of a run of equal words OR their bits together and the run's last lane issues ONE atomicOr
  // per bitmap instead of one per entry (the source hub of a scale-24 R-MAT graph has 7e5 entries
  // over 2e4 words).  Exactly the per-entry semantics: a bit counts for the first lane of the run
  // that carries it, and only if the word did not hold it before.
  // Two parts, so that a caller can have the bitmap reads of several calls in flight at once:
  // warp_edge_bit (load) and warp_edge_set (update).
  static constexpr bool kWarpEntries = true;
  GL_DEV void warp_edge(uint32_t v, bool valid, ScanAcc& acc) const {
    const uint32_t bit = warp_edge_bit(v, valid);
    if (!__any_sync(0xffffffffu, bit != 0)) return;
    if (warp_edge_set(v, bit)) note_fresh(v, v < ivnum ? degree_of(v) : 0ull, acc);
  }
  // v's bit unless the visited bitmap already holds it (plain, possibly stale read)
  GL_DEV uint32_t warp_edge_bit(uint32_t v, bool valid) const {
    return valid ? (1u << (v & 31)) & ~vis[v >> 5] : 0u;
  }
  // All lanes converged.  Sets the lanes' bits in vis / nxt (/ remote); true on the lane whose
  // entry visited v first.
  GL_DEV bool warp_edge_set(uint32_t v, uint32_t bit) const {
    const uint32_t lane = lane_id();
    const uint32_t w = v >> 5;
    // runs of lanes with the same word (invalid / already-visited lanes join their neighbours' runs
    // with an empty bit set, or form runs of their own that end without an atomic)
    const uint32_t wp = __shfl_up_sync(0xffffffffu, w, 1);
    const bool head = lane == 0 || wp != w;
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    const uint32_t seg = __popc(heads & (0xFFFFFFFFu >> (31 - lane)));
    uint32_t incl = bit;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      const uint32_t so = __shfl_up_sync(0xffffffffu, seg, o);
      if (lane >= (uint32_t) o && so == seg) incl |= t;
    }
    const uint32_t prev_incl = __shfl_up_sync(0xffffffffu, incl, 1);
    const uint32_t excl = head ? 0u : prev_incl;
    const uint32_t tails = (heads >> 1) | 0x80000000u;
    const bool tail = (tails >> lane) & 1u;
    uint32_t old = 0;
    if (tail && incl) {
      old = atomicOr(vis + w, incl);
      const uint32_t fresh = incl & ~old;
      if (fresh) {
        atomicOr(nxt + w, fresh);        // level bitmap of depth+1 (also for outer v)
        // outer copies (lid >= ivnum) are reported to their owners
        const uint32_t lo = w << 5;
        uint32_t outer = 0;
        if (lo >= ivnum) outer = 0xFFFFFFFFu;
        else if (lo + 32 > ivnum) outer = 0xFFFFFFFFu << (ivnum - lo);
        if (fresh & outer) atomicOr(remote + w, fresh & outer);
      }
    }
    const uint32_t mytail = lane + __ffs(tails >> lane) - 1;
    old = __shfl_sync(0xffffffffu, old, mytail);
    return (bit & ~old & ~excl) != 0;
  }
  GL_DEV void edge(uint32_t, Meta, uint32_t v, W, ScanAcc& acc) const {
    if (bit_test(vis, v)) return;        // plain (possibly stale) read first
    if (!bit_set_atomic(vis, v)) return; // somebody else won
    bit_set_atomic(nxt, v);              // level bitmap of depth+1 (also for outer v)
    acc.touched++;
    if (v < ivnum) {
      acc.next_count++;
      acc.next_edges += degree_of(v);
    } else {
      bit_set_atomic(remote, v);
      acc.remote++;
    }
  }
};

__global__ void k_bfs_deg8(const uint64_t* rp, uint32_t n, uint8_t* deg8) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long d = rp[i + 1] - rp[i];
  deg8[i] = d == 0 ? 0 : (uint8_t) (64 - __clzll((long long) d));   // 1 + floor(log2 d)
}

__global__ void k_bfs_nz(const uint64_t* rp, uint32_t n, uint32_t* nz) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool has = i < n && rp[i + 1] > rp[i];
  uint32_t w = __ballot_sync(0xffffffffu, has);
  if ((threadIdx.x & 31) == 0 && i < n) nz[i >> 5] = w;
}

__global__ void k_bfs_popc(const uint32_t* bm, uint32_t words, unsigned long long* out) {
  unsigned long long c = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) c += __popc(bm[i]);
  c = warp_sum(c);
  if (lane_id() == 0 && c) atomicAdd(out, c);
}

// rows with at least min_len entries
__global__ void k_bfs_count_rows(const uint64_t* rp, uint32_t n, uint64_t min_len, unsigned long long* out) {
  unsigned long long c = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += rp[i + 1] - rp[i] >= min_len;
  c = warp_sum(c);
  if (lane_id() == 0 && c) atomicAdd(out, c);
}

// lid -> gid of every CSR entry / of the hub-neighbour table (global-frontier pull, several fragments)
__global__ void k_bfs_gcol(const uint32_t* __restrict__ col, uint64_t m, uint32_t ivnum, uint32_t my_gid0,
                           const uint32_t* __restrict__ ovgid, uint32_t* gcol) {
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
    const uint32_t c = col[i];
    gcol[i] = c < ivnum ? (my_gid0 | c) : ovgid[c - ivnum];
  }
}
__global__ void k_bfs_gid_table(const uint32_t* __restrict__ lids, uint32_t n, uint32_t ivnum, uint32_t my_gid0,
                                const uint32_t* __restrict__ ovgid, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = lids[i];
  out[i] = c == kInfU32 ? kInfU32 : (c < ivnum ? (my_gid0 | c) : ovgid[c - ivnum]);
}

// several fragments, hub-first order: the gid of outer copy o in its owner's NEW lid space
__global__ void k_bfs_ovgid_new(const uint32_t* __restrict__ ovgid, const uint32_t* __restrict__ newlid, uint32_t ovnum,
                                uint32_t id_mask, uint32_t* out) {
  const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o < ovnum) out[o] = (ovgid[o] & ~id_mask) | (newlid[o] & id_mask);
}
// gid <-> row-sort key (lid = degree rank inside the owner fragment in the high bits, fid in the low
// bits): rows sorted by this key list the likeliest parents first, whichever fragment owns them
__global__ void k_bfs_gid_key(uint32_t* g, uint64_t m, int fid_offset, uint32_t id_mask, int to_key) {
  const int fid_bits = 32 - fid_offset;
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
    const uint32_t x = g[i];
    g[i] = to_key ? (((x & id_mask) << fid_bits) | (x >> fid_offset))
                  : (((x & ((1u << fid_bits) - 1u)) << fid_offset) | (x >> fid_bits));
  }
}
// Delegated hubs (several fragments, hub-first order): the kDlgPerFrag highest-ranked vertices of
// EVERY fragment are known to all GPUs by gid, and every GPU keeps, per hub, the list of its own
// inner vertices adjacent to it (the hub's row restricted to this fragment, read off the local
// rows: in a row sorted by the lid-major key the hub entries come first).  A BFS that starts at
// such a hub then runs level 0 on all GPUs at once, without a single message -- instead of one
// GPU walking a 10^6-entry row and shipping most of it to the others.
constexpr uint32_t kDlgPerFrag = 16;
// mode 0: count[h]++ ; mode 1: list[off[h] + cursor[h]++] = v
__global__ void k_bfs_dlg_scan(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ gcol, uint32_t ivnum,
                               int fid_offset, uint32_t id_mask, uint32_t* cnt, const uint64_t* __restrict__ off,
                               uint32_t* list, int mode) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= ivnum) return;
  const uint64_t b = rp[v], e = rp[v + 1];
  uint32_t prev = kInfU32;
  for (uint64_t p = b; p < e; ++p) {
    const uint32_t g = gcol[p];
    const uint32_t l = g & id_mask;
    if (l >= kDlgPerFrag) break;
    if (g == prev) continue;   // parallel edges
    prev = g;
    const uint32_t h = (g >> fid_offset) * kDlgPerFrag + l;
    const uint32_t at = atomicAdd(cnt + h, 1u);
    if (mode) list[off[h] + at] = v;
  }
}

__global__ void k_bfs_first_col(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint32_t n, uint32_t* out) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) out[v] = rp[v + 1] > rp[v] ? col[rp[v]] : kInfU32;
}

__global__ void k_bfs_deg32(const uint64_t* __restrict__ rp, uint32_t ivnum, uint32_t tvnum, uint32_t* deg) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tvnum) return;
  unsigned long long d = i < ivnum ? rp[i + 1] - rp[i] : 0;
  deg[i] = d > 0xFFFFFFFEull ? 0xFFFFFFFEu : (uint32_t) d;
}

__global__ void k_bfs_seed(uint32_t src, uint32_t* lv0, uint32_t* vis) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    lv0[src >> 5] |= 1u << (src & 31);
    vis[src >> 5] |= 1u << (src & 31);
  }
}

// hub_nbr[v] = the inner neighbour of v with the largest out-degree (ties ->
// first in the row); one warp per row.  Built once per app.
__global__ void __launch_bounds__(256)
k_bfs_hub_nbr(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint32_t ivnum, uint32_t* hub_nbr,
              const uint32_t* __restrict__ deg_all = nullptr) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const uint64_t b = rp[v], e = rp[v + 1];
    unsigned long long best = 0;
    for (uint64_t p = b + lane_id(); p < e; p += 32) {
      uint32_t u = col[p];
      // outer copies have no local row: their owner's degree when it was synced (deg_all), else they
      // rank below every inner neighbour
      unsigned long long dg = deg_all ? (unsigned long long) deg_all[u] + 1 : (u < ivnum ? rp[u + 1] - rp[u] + 1 : 1);
      if (dg > 0xFFFFFFFFull) dg = 0xFFFFFFFFull;
      uint64_t off = p - b;
      if (off > 0xFFFFFFFEull) off = 0xFFFFFFFEull;
      unsigned long long key = (dg << 32) | (0xFFFFFFFFu - (uint32_t) off);
      best = key > best ? key : best;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
      best = t > best ? t : best;
    }
    if (lane_id() == 0) hub_nbr[v] = (b < e) ? col[b + (0xFFFFFFFFu - (uint32_t) best)] : kInfU32;
  }
}

// ---------------------------------------------------------------------------
// Pull step over the inner vertices (bfs.h:239-259) as a phase shared by the
// stand-alone kernel and the fused whole-query kernel.
// ---------------------------------------------------------------------------
constexpr uint32_t kPullSerialCap = 8;   // row entries a single thread probes
constexpr uint32_t kListStage = 2048;    // tail-list entries a CTA gathers before one global append
struct PullSmem {
  uint32_t v[kTileV];
  uint32_t lng[kTileV];   // candidates whose row is longer than the cap
  uint32_t nlong;
  uint32_t found[kTileV / 32];
  uint32_t words[kTB];
  uint32_t cand[kTB];     // the ticket's candidate words, kept for the list append
  uint32_t warp[kTB / 32 + 1];
  uint32_t nz[kSuperTiles];
  uint32_t ticket;
  // list append: staged entries [0, min(nstage, stage_full)), flushed with one atomic per CTA
  uint32_t stage[kListStage];
  uint32_t nstage, stage_full, stage_base;
};

struct PullArgs {
  const uint64_t* rp;
  const uint32_t* col;
  const uint32_t* hub_nbr;
  uint32_t ivnum;
  const uint32_t* nz;
  // Several fragments, fused kernel: `col` / `hub_nbr` hold GIDs and the frontier is the
  // REPLICATED GLOBAL bitmap, kept as one segment per owner fragment (seg[f] = the bits of
  // fragment f's inner vertices; the owners store them into every peer over NVLink).  null:
  // `col` holds lids and the frontier is the local bitmap passed to the phase.
  const uint32_t* const* seg;
  int fid_offset;
  uint32_t id_mask;
  uint32_t hub_dummy;   // a valid id for the branch-free probes of non-candidates (lid 0 / my gid 0)
  uint32_t seg_off;     // word offset of this level's generation inside every segment slot
  int seg_cached;       // 1: these addresses were never read before in this launch -> L1 may cache them
  // Shipment of the NEXT frontier fused into the pull: a thread that finished its word stores it
  // straight into every fragment's next-generation segment (ship_send[p] = my slot at peer p,
  // ship_recv[ship_fid] = my own copy), so the NVLink stores drain while the pull is still running
  // instead of in a pass of their own after it.  null: no shipment.
  char* const* ship_send;
  const char* const* ship_recv;
  uint32_t ship_fid, ship_fnum, ship_off;
  // Single-fragment fused kernel only (bfs_pull_phase<false, true>).  hub_first = 1: the adjacency is
  // the hub-first shadow graph, so hub_nbr[v] is the first entry of v's sorted row (Setup fills it
  // from there), the lids [0, sweep_v) are the non-isolated vertices and the lids [0, multi_v) the
  // rows with two or more entries.  hub_first = 0: stage 2 scans whole rows and sweep_v = ivnum.
  uint32_t hub_first;
  uint32_t sweep_v, multi_v;
  // Tail candidate list (hub-first order; list_cap = 0: none): once few non-isolated vertices are
  // unvisited (BfsFusedArgs::list_gap), a pull level lists its unresolved candidates here; if they fit
  // list_cap, every later level pulls over that list instead of the bitmap (bfs_list_pull)
  uint32_t* list;
  uint32_t list_cap;
};

// A thread's share of a pull level's entries scanned and vertices expanded, when the caller adds them
// with the CTA's other counters (flush_acc_cta) instead of the phase adding them per warp.
struct PullCounts {
  unsigned long long scanned = 0;
  uint32_t frontier = 0;
};

// is vertex `id` in the frontier?  kGlobal is a compile-time switch: the single-fragment kernels
// keep the plain local-bitmap probe (a run-time branch here cost 8 % of the whole query)
template <bool kGlobal>
GL_DEV bool front_test(const PullArgs& a, const uint32_t* cur, uint32_t id) {
  if (kGlobal) {
    // A frontier bit is probed ~10^7 times per level: it must be an L1 hit.  L1 is not coherent
    // with the peers' stores, so every pull level of a launch reads a FRESH generation of the
    // segments (addresses no SM has loaded before in this launch); once the generations wrap
    // around (seg_cached = 0) the probes bypass L1.
    const uint32_t f = id >> a.fid_offset, l = id & a.id_mask;
    const uint32_t* p = a.seg[f] + a.seg_off + (l >> 5);
    const uint32_t w = a.seg_cached ? *p : __ldcg(p);
    return (w >> (l & 31)) & 1u;
  }
  return (cur[id >> 5] >> (id & 31)) & 1u;
}

// Stage-1 probes of one nibble of a candidate word: the candidates among its four vertices (bits of
// `nib`) whose hub neighbour (h) is in the frontier.  Branch-free: every probe is an unconditional load
// (index 0 / hub_dummy when the lane is not a candidate) so that the loads of a nibble are all in
// flight together instead of forming a chain of dependent branches.
template <bool kGlobal>
GL_DEV uint32_t pull_probe_nibble(const PullArgs& a, const uint32_t* __restrict__ cur, uint32_t nib, uint4 h) {
  const bool c0 = (nib & 1u) && h.x != kInfU32;
  const bool c1 = (nib & 2u) && h.y != kInfU32;
  const bool c2 = (nib & 4u) && h.z != kInfU32;
  const bool c3 = (nib & 8u) && h.w != kInfU32;
  const uint32_t dummy = kGlobal ? a.hub_dummy : 0u;
  const uint32_t i0 = c0 ? h.x : dummy, i1 = c1 ? h.y : dummy;
  const uint32_t i2 = c2 ? h.z : dummy, i3 = c3 ? h.w : dummy;
  const bool t0 = front_test<kGlobal>(a, cur, i0), t1 = front_test<kGlobal>(a, cur, i1);
  const bool t2 = front_test<kGlobal>(a, cur, i2), t3 = front_test<kGlobal>(a, cur, i3);
  uint32_t r = 0;
  r |= (c0 && t0) ? 1u : 0u;
  r |= (c1 && t1) ? 2u : 0u;
  r |= (c2 && t2) ? 4u : 0u;
  r |= (c3 && t3) ? 8u : 0u;
  return r;
}

// One super-tile = 8192 vertices = 256 words; thread t owns word t: it probes
// the hub neighbour of each of its (up to 32) candidates with eight
// independent 16-byte loads in flight (stage 1), hands the unresolved ones to
// a CTA-wide row scan (stage 2) and finally writes its visited / next-level
// word with plain stores (the word belongs to this thread during the pull).
// kTail (single-fragment fused kernel): the PullArgs hub_first fields apply,
// and make_list appends the candidates left unresolved to a.list, counted in
// ctrl->aux_ticket (the level that starts the tail, see bfs_list_pull), and
// the level's scanned / frontier counts are left in *cnt for the caller.
template <bool kGlobal, bool kTail = false>
GL_DEV bool bfs_pull_phase(PullSmem& sm, const PullArgs& a,
                           const uint32_t* __restrict__ cur, uint32_t* vis,
                           uint32_t* nxt, ScanCtrl* ctrl, ScanAcc& acc, bool make_list = false,
                           PullCounts* cnt = nullptr) {
  const uint32_t nwords = (a.ivnum + 31) / 32;
  const bool hub_first = kTail && a.hub_first;
  // hub-first order: entry 0 of a row is hub_nbr[v], which stage 1 has just tested
  const uint32_t skip = hub_first ? 1u : 0u;
  uint64_t scanned = 0;
  uint32_t cand = 0;
  uint32_t st;
  bool shipped = false;
  if (threadIdx.x == 0) {
    sm.nlong = 0;
    if (kTail) {
      sm.nstage = 0;
      sm.stage_full = kListStage;
    }
  }
  __syncthreads();
  while (next_super_tile(sm, &ctrl->tile_ticket, kTail ? a.sweep_v : a.ivnum,
                         [&](uint32_t w) { return a.nz[w] & ~vis[w]; }, &st)) {
    const uint32_t word = sm.words[threadIdx.x];
    const uint32_t wi = st * (kSuperV / 32) + threadIdx.x;
    const uint32_t vbase = wi * 32;
    sm.words[threadIdx.x] = 0;  // reused as the stage-2 result word
    if (kTail && make_list) sm.cand[threadIdx.x] = word;
    // ---- stage 1 ----
    uint32_t res = 0;
    if (kTail) {
      // The hub neighbours of a warp's 32 words are 4 KB in a row.  Lane l reads 16 bytes of them per
      // step, so that a warp load covers 4 lines: step j brings the 32 entries of lanes 4j..4j+3, and
      // lane l probes nibble l % 8 of lane 4j + l / 8.  (A thread reading its own 128 bytes made every
      // warp load touch 32 lines, eight times per line.)  The nibbles' results meet in the owning lane.
      if (__any_sync(0xffffffffu, word != 0)) {
        const uint32_t lane = lane_id();
        const uint4* wp = (const uint4*) (a.hub_nbr + (vbase - lane * 32)) + lane;
#pragma unroll 2
        for (int j = 0; j < 8; ++j) {
          const uint32_t nib = (__shfl_sync(0xffffffffu, word, 4 * j + (lane >> 3)) >> (4 * (lane & 7))) & 0xFu;
          uint4 h = make_uint4(kInfU32, kInfU32, kInfU32, kInfU32);
          if (nib) h = wp[32 * j];
          uint32_t r = pull_probe_nibble<kGlobal>(a, cur, nib, h) << (4 * (lane & 7));
          r |= __shfl_xor_sync(0xffffffffu, r, 1);
          r |= __shfl_xor_sync(0xffffffffu, r, 2);
          r |= __shfl_xor_sync(0xffffffffu, r, 4);
          r = __shfl_sync(0xffffffffu, r, (lane & 3) * 8);
          if ((lane >> 2) == (uint32_t) j) res = r;
        }
      }
      scanned += __popc(word);
    } else if (word) {
      // (the stand-alone and several-fragment pulls keep the per-thread read: not measured with the
      // warp-strided one, and the several-fragment kernels already spill at 64 registers)
      const uint4* hp = (const uint4*) (a.hub_nbr + vbase);
#pragma unroll 2
      for (int j = 0; j < 8; ++j) {
        const uint32_t nib = (word >> (4 * j)) & 0xFu;
        uint4 h = make_uint4(kInfU32, kInfU32, kInfU32, kInfU32);
        if (nib) h = hp[j];
        res |= pull_probe_nibble<kGlobal>(a, cur, nib, h) << (4 * j);
      }
      scanned += __popc(word);
    }
    // ---- stage 2: leftovers scan their row, kTileV candidates per pass ----
    uint32_t rest = word & ~res;
    if (hub_first) {
      // a row of one entry has nothing left to scan: only lids below multi_v enter stage 2
      rest &= vbase + 32 <= a.multi_v ? 0xFFFFFFFFu : (vbase >= a.multi_v ? 0u : (1u << (a.multi_v - vbase)) - 1u);
    }
    uint32_t total;
    uint32_t off = block_excl_scan(__popc(rest), sm.warp, &total);
    cand += (threadIdx.x == 0) ? total : 0;
    for (uint32_t base = 0; base < total; base += kTileV) {
      // stage the candidates whose rank falls in [base, base + kTileV)
      uint32_t r = rest, k = off;
      while (r) {
        uint32_t b = __ffs(r) - 1;
        r &= r - 1;
        if (k >= base && k < base + kTileV) sm.v[k - base] = vbase + b;
        ++k;
      }
      __syncthreads();
      const uint32_t nc = (total - base) < (uint32_t) kTileV ? (total - base) : (uint32_t) kTileV;
      // 2a: every thread probes at most kPullSerialCap entries of its (up to kTileV / kTB = 4) rows;
      // longer rows go to the warp-cooperative pass so that one unlucky thread cannot stall the
      // CTA behind a chain of dependent loads.  The four rows are walked in lock step: their
      // row-pointer reads, column reads and frontier probes are four independent chains in flight
      // (one after the other, a ticket of leftovers cost 4 x (2 + 2 probes) dependent latencies per
      // thread, and the level ended with CTAs waiting tens of microseconds for the last tickets).
      constexpr int kRows = kTileV / kTB;
      static_assert(kRows == 4, "stage 2a is written for four candidates per thread");
      // (the several-fragment probe keeps more state live: two rows at a time there, else spills)
      constexpr int kIL = kGlobal ? 2 : 4;
      const uint32_t dummy = kGlobal ? a.hub_dummy : 0u;
#pragma unroll 1
      for (int g = 0; g < kRows; g += kIL) {
        uint32_t vv[kIL], len[kIL];
        uint64_t bb[kIL];
#pragma unroll
        for (int k = 0; k < kIL; ++k) {
          const uint32_t i = threadIdx.x + (g + k) * kTB;
          vv[k] = i < nc ? sm.v[i] : kInfU32;
        }
#pragma unroll
        for (int k = 0; k < kIL; ++k) bb[k] = vv[k] != kInfU32 ? a.rp[vv[k]] + skip : 0ull;
        uint32_t act = 0, foundm = 0;
#pragma unroll
        for (int k = 0; k < kIL; ++k) {
          len[k] = vv[k] != kInfU32 ? (uint32_t) (a.rp[vv[k] + 1] - bb[k]) : 0u;
          if (len[k]) act |= 1u << k;
        }
        for (uint32_t p = 0; p < kPullSerialCap && act; ++p) {
          uint32_t ids[kIL];
#pragma unroll
          for (int k = 0; k < kIL; ++k) ids[k] = ((act >> k) & 1u) ? a.col[bb[k] + p] : dummy;
          bool t[kIL];
#pragma unroll
          for (int k = 0; k < kIL; ++k) t[k] = front_test<kGlobal>(a, cur, ids[k]);   // unconditional: all in flight
          scanned += __popc(act);
#pragma unroll
          for (int k = 0; k < kIL; ++k) {
            if ((act >> k) & 1u) {
              if (t[k]) {
                foundm |= 1u << k;
                act &= ~(1u << k);
              } else if (p + 1 >= len[k]) {
                act &= ~(1u << k);
              }
            }
          }
        }
#pragma unroll
        for (int k = 0; k < kIL; ++k) {
          if (vv[k] == kInfU32) continue;
          if ((foundm >> k) & 1u) atomicOr(&sm.words[(vv[k] >> 5) - st * (kSuperV / 32)], 1u << (vv[k] & 31));
          else if (len[k] > kPullSerialCap) sm.lng[atomicAdd(&sm.nlong, 1u)] = vv[k];
        }
      }
      __syncthreads();
      // 2b: one warp per long row, 32 entries per step
      const uint32_t nl = sm.nlong;
      for (uint32_t i = threadIdx.x >> 5; i < nl; i += kTB / 32) {
        const uint32_t v = sm.lng[i];
        const uint64_t b = a.rp[v] + skip;
        const uint32_t len = (uint32_t) (a.rp[v + 1] - b);
        const uint32_t* row = a.col + b;
        bool hit = false;
        uint32_t p = kPullSerialCap;
        for (; p < len; p += 32) {
          const uint32_t q = p + lane_id();
          const bool h = q < len && front_test<kGlobal>(a, cur, row[q]);
          if (__any_sync(0xffffffffu, h)) {
            hit = true;
            p += 32;
            break;
          }
        }
        if (lane_id() == 0) {
          scanned += (p < len ? p : len) - kPullSerialCap;
          if (hit) atomicOr(&sm.words[(v >> 5) - st * (kSuperV / 32)], 1u << (v & 31));
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) sm.nlong = 0;
    }
    if (total == 0) __syncthreads();  // sm.words zeroing vs. the next ticket
    const uint32_t found_w = res | sm.words[threadIdx.x];
    if (found_w && wi < nwords) {
      vis[wi] |= found_w;  // the word is owned by this thread during the pull
      nxt[wi] = found_w;
      if (kGlobal && a.ship_send) {
        for (uint32_t p = 0; p < a.ship_fnum; ++p) {
          uint32_t* dst = (p == a.ship_fid ? (uint32_t*) a.ship_recv[p] : (uint32_t*) a.ship_send[p]) + a.ship_off;
          dst[wi] = found_w;
        }
        shipped = a.ship_fnum > 1;
      }
    }
    acc.next_count += __popc(found_w);
    if (kTail && make_list) {
      // the candidates still unresolved become the tail list: staged in shared memory (a global
      // atomic per warp and ticket, all on one address, cost more than the level's whole pull);
      // a warp whose entries do not fit any more appends them to the list itself
      uint32_t surv = sm.cand[threadIdx.x] & ~found_w;
      const uint32_t ns = __popc(surv);
      const uint32_t incl = warp_incl_scan(ns);
      uint32_t at = 0;
      if (lane_id() == 31 && incl) {
        at = atomicAdd(&sm.nstage, incl);
        if (at + incl > kListStage) {
          atomicMin(&sm.stage_full, at);   // the staged entries stay a prefix
          at = kListStage + atomicAdd(&ctrl->aux_ticket, incl);
        }
      }
      at = __shfl_sync(0xffffffffu, at, 31) + incl - ns;
      for (; surv; surv &= surv - 1, ++at) {
        const uint32_t v = vbase + __ffs(surv) - 1;
        if (at < kListStage) sm.stage[at] = v;
        else if (at - kListStage < a.list_cap) a.list[at - kListStage] = v;
      }
    }
    __syncthreads();
  }
  if (kTail && make_list) {
    const uint32_t n = sm.nstage < sm.stage_full ? sm.nstage : sm.stage_full;
    if (threadIdx.x == 0 && n) sm.stage_base = atomicAdd(&ctrl->aux_ticket, n);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += kTB)
      if (sm.stage_base + i < a.list_cap) a.list[sm.stage_base + i] = sm.stage[i];
  }
  acc.touched = acc.next_count;
  if (kTail) {
    cnt->scanned = scanned;
    cnt->frontier = cand;
    return shipped;
  }
  unsigned long long s = warp_sum((unsigned long long) scanned);
  if (lane_id() == 0 && s) atomicAdd(&ctrl->scanned, s);
  if (threadIdx.x == 0 && cand) atomicAdd(&ctrl->frontier, (unsigned long long) cand);
  return shipped;
}

__global__ void __launch_bounds__(kTB, 4)
k_bfs_pull(PullArgs a, const uint32_t* __restrict__ cur, uint32_t* vis,
           uint32_t* nxt, ScanCtrl* ctrl) {
  __shared__ PullSmem sm;
  ScanAcc acc;
  bfs_pull_phase<false>(sm, a, cur, vis, nxt, ctrl, acc);
  flush_acc(acc, ctrl);
}

// Tail pull level (single fragment, hub-first order): the candidates are the
// list[0, n) that an earlier pull level left unresolved -- not a sweep of the
// whole bitmap.  One entry per thread, grid-stride, no tickets and no CTA
// barriers: hub probe, then the row from entry 1 (entry 0 is hub_nbr[v]);
// rows longer than 1 + kPullSerialCap are finished by their warp, 32 entries
// per step.  Words are shared between threads here, so hits set vis / nxt
// with atomicOr.  A resolved entry is overwritten with kInfU32 in place: the
// list is not compacted (no atomic round trip per level; in the tail few
// entries resolve per level, and a dead entry costs one coalesced load).
// The level's counts are left in `cnt` for flush_acc_cta.
GL_DEV void bfs_list_pull(const PullArgs& a, const uint32_t* __restrict__ cur, uint32_t* vis, uint32_t* nxt,
                          uint32_t n, ScanAcc& acc, PullCounts& cnt) {
  uint32_t* list = a.list;
  const uint32_t lane = lane_id();
  uint64_t scanned = 0;
  uint32_t cand = 0;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < n; base += gridDim.x * blockDim.x) {
    const uint32_t i = base + lane;
    const uint32_t v = i < n ? list[i] : kInfU32;
    bool hit = false;
    uint64_t b = 0;
    uint32_t len = 0;
    if (v != kInfU32) {
      const uint32_t h = a.hub_nbr[v];
      b = a.rp[v] + 1;
      const uint64_t e = a.rp[v + 1];
      hit = h != kInfU32 && front_test<false>(a, cur, h);
      len = e > b ? (uint32_t) (e - b) : 0u;
      const uint32_t serial = len < kPullSerialCap ? len : kPullSerialCap;
      ++cand;
      ++scanned;
      for (uint32_t p = 0; p < serial && !hit; ++p, ++scanned) hit = front_test<false>(a, cur, a.col[b + p]);
    }
    for (uint32_t lng = __ballot_sync(0xffffffffu, !hit && len > kPullSerialCap); lng; lng &= lng - 1) {
      const int src = __ffs(lng) - 1;
      const uint64_t lb = __shfl_sync(0xffffffffu, b, src);
      const uint32_t llen = __shfl_sync(0xffffffffu, len, src);
      bool found = false;
      uint32_t p = kPullSerialCap;
      for (; p < llen; p += 32) {
        const uint32_t q = p + lane;
        if (__any_sync(0xffffffffu, q < llen && front_test<false>(a, cur, a.col[lb + q]))) {
          found = true;
          p += 32;
          break;
        }
      }
      if (lane == (uint32_t) src) {
        hit = found;
        scanned += (p < llen ? p : llen) - kPullSerialCap;
      }
    }
    if (hit) {
      atomicOr(vis + (v >> 5), 1u << (v & 31));
      atomicOr(nxt + (v >> 5), 1u << (v & 31));
      list[i] = kInfU32;
      acc.next_count++;
    }
  }
  acc.touched = acc.next_count;
  cnt.scanned = scanned;
  cnt.frontier = cand;
}

// ---------------------------------------------------------------------------
// Fused whole-query BFS (single fragment): ONE cooperative launch runs every
// superstep.  Per-level device timestamps keep the ms/superstep report.
// ---------------------------------------------------------------------------
// level records a fused query keeps: with PEval's step 0 they fill the per-step arrays of gl_query_stats
constexpr int kMaxFusedStats = GL_MAX_STEP_STATS - 1;
struct BfsLevelStat {
  unsigned long long t_ns;
  unsigned long long scanned;
  uint32_t frontier;
  uint32_t mode;
};
struct BfsFusedCtl {
  ScanCtrl c[3];       // rotating per-level counters (level d uses c[d % 3])
  uint32_t levels;     // levels executed
  uint32_t has_src, src_lid;
  uint32_t overflow;   // ran out of level bitmaps
  uint32_t pad;
  unsigned long long touched;   // of the whole query, over every level and launch
  // entries scanned / vertices expanded by the levels past the level table below (it is finite)
  unsigned long long over_scanned, over_frontier;
  unsigned long long t_begin;
  // state a relaunch starts from: parked by the kernel when it stops because
  // the level-bitmap ring is full (the host spills the finished levels and
  // relaunches); several fragments: also the first launch's, from the seed kernel
  // (k_bfs_fused derives its first launch's state from its arguments)
  unsigned long long r_nf, r_mf, r_visited_edges, r_visited_cnt;
  uint32_t r_phase, r_pad;   // r_phase = ~0: derive from the seed
  unsigned long long p_nf, p_mf, p_visited_edges, p_visited_cnt;   // parked state (-> r_* by k_bfs_resume_prep)
  uint32_t p_phase, p_pad;
  // multi-fragment fused kernel: result of the last in-kernel collective and
  // how much of the communicator's sequence space the launch consumed
  long long xres[4];
  unsigned long long x_last_tag;
  uint32_t x_msg_rounds, x_mirror_syncs;
  unsigned long long x_items;   // items this GPU sent
  unsigned long long ph[32][6];  // GL_TRACE: phase timestamps of the first 32 levels (thread 0)
  unsigned long long xw[32][2];  // GL_TRACE: per level: peer wait / first grid.sync of its last xsync
  unsigned long long l_nf;               // several fragments: this fragment's part of the current frontier (statistics)
  unsigned long long r_visited_cnt_g;    // several fragments: vertices visited so far in the whole graph (resume state)
  // thread 0's first instruction of the fused multi-fragment kernel / last of either fused kernel (GL_KTIME)
  unsigned long long t_kstart, t_kend;
  unsigned long long xt[8];      // GL_TRACE: timestamps inside the most recent xsync (block 0, thread 0)
  uint32_t x_error, x_pad;   // 1 = a peer did not show up in time, 2 = landing slot overflow
  BfsLevelStat stat[kMaxFusedStats];
};

GL_DEV unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// When a pull phase keeps pulling although its frontier has become small (the tail of the query).
enum BfsTailRule : uint32_t {
  kNoTail,            // never: back to push
  kTailPerFrontier,   // while few candidates remain per frontier vertex (unvisited <= 64 n_f)
  kTailAbsolute,      // ... or few in absolute terms (unvisited <= V / 64)
};

// The push/pull schedule of every query path (both fused kernels and the stepwise host loop).
// push -> pull when the frontier's edges exceed 1/14 of the unvisited edges;
// pull -> push (for good) when the frontier shrinks below V/beta (Beamer et
// al.; the reference uses vertex ratios, bfs.h:171-180 — the schedule only
// affects speed, never the levels).  phase: 0 = initial push, 1 = pull,
// 2 = final push; k_bfs_fused adds kListPull = pull over the tail candidate
// list, kept until the query ends (never an input of bfs_next_phase).
// `tail` is a constant at every call site, so each caller compiles only its own rule.
constexpr uint32_t kListPull = 3;
__host__ __device__ __forceinline__ uint32_t bfs_next_phase(uint32_t phase, unsigned long long n_f, unsigned long long m_f,
                                                            unsigned long long m_u, unsigned long long vnum,
                                                            int direction_opt, uint32_t beta,
                                                            unsigned long long unvisited, BfsTailRule tail) {
  if (!direction_opt) return 0;
  if (phase == 0) return m_f > m_u / 14 ? 1u : 0u;
  if (phase == 1) {
    // A pull level costs ~ the unvisited non-isolated vertices, a push level
    // ~ the frontier's edges plus two grid barriers: keep pulling while the
    // frontier is large (Beamer) or, per `tail`, while few candidates remain;
    // go back to push for long sparse tails.
    // n_f >= floor(vnum / beta), without a division the compiler would hoist out of the level loop
    // and keep live (k_bfs_fused has no register to spare)
    if ((n_f + 1) * beta > vnum) return 1u;
    if (tail != kNoTail && unvisited <= 64ull * n_f) return 1u;
    if (tail == kTailAbsolute && unvisited <= vnum / 64) return 1u;
    return 2u;
  }
  return 2u;
}

// The state a launch of a fused kernel parks when the level ring is full: the host spills levels
// [0, max_lv-1) and relaunches from it (k_bfs_resume_prep).  A tail list does not survive the
// relaunch: its first level sweeps the bitmap again.
GL_DEV void bfs_park(BfsFusedCtl* ctl, unsigned long long n_f, unsigned long long m_f, unsigned long long visited_edges,
                     unsigned long long visited_cnt, uint32_t phase) {
  ctl->overflow = 1;
  ctl->p_nf = n_f;
  ctl->p_mf = m_f;
  ctl->p_visited_edges = visited_edges;
  ctl->p_visited_cnt = visited_cnt;
  ctl->p_phase = phase == kListPull ? 1u : phase;
}

// Thread 0's bookkeeping at the end of level `depth` of a fused kernel: the level's statistics
// (`frontier` vertices expanded, `mode` 1 = pull), the level count and the counters of the query;
// c[(depth+2)%3] was last read during this level and is cleared for level depth+1.
GL_DEV void bfs_level_end(BfsFusedCtl* ctl, uint32_t depth_base, uint32_t depth, unsigned long long frontier,
                          uint32_t mode) {
  const volatile ScanCtrl* VC = &ctl->c[depth % 3];
  const uint32_t adepth = depth_base + depth;
  if (adepth < (uint32_t) kMaxFusedStats) {
    BfsLevelStat ls;
    ls.t_ns = global_ns();
    ls.scanned = VC->scanned;
    ls.frontier = (uint32_t) (frontier > 0xFFFFFFFFull ? 0xFFFFFFFFull : frontier);
    ls.mode = mode;
    ctl->stat[adepth] = ls;
  } else {
    ctl->over_scanned += VC->scanned;
    ctl->over_frontier += frontier;
  }
  ctl->levels = adepth + 1;
  ctl->touched += VC->touched;
  ctl->c[(depth + 2) % 3] = ScanCtrl();
}

// first launch of a several-fragment query (k_bfs_fused_multi); k_bfs_fused seeds itself
__global__ void k_bfs_seed_fused(uint32_t src, int has_src, uint32_t* lv0, uint32_t* vis, const uint64_t* rp,
                                 BfsFusedCtl* ctl) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  ctl->c[0] = ScanCtrl();
  ctl->c[1] = ScanCtrl();
  ctl->c[2] = ScanCtrl();
  ctl->levels = 0;
  ctl->overflow = 0;
  ctl->touched = ctl->over_scanned = ctl->over_frontier = 0;
  unsigned long long deg = 0;
  if (has_src) {
    lv0[src >> 5] |= 1u << (src & 31);
    vis[src >> 5] |= 1u << (src & 31);
    deg = rp[src + 1] - rp[src];
  }
  ctl->has_src = has_src;
  ctl->src_lid = src;
  ctl->r_nf = has_src ? 1 : 0;
  ctl->r_mf = deg;
  ctl->r_visited_edges = deg;
  ctl->r_visited_cnt = has_src ? 1 : 0;
  ctl->r_visited_cnt_g = 1;
  ctl->r_phase = 0xFFFFFFFFu;
  ctl->x_error = 0;
  ctl->x_items = 0;
  ctl->x_msg_rounds = 0;
  ctl->x_mirror_syncs = 0;
  ctl->t_begin = global_ns();
}

// between two launches of a spilled query: fresh level counters
__global__ void k_bfs_resume_prep(BfsFusedCtl* ctl) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  ctl->c[0] = ScanCtrl();
  ctl->c[1] = ScanCtrl();
  ctl->c[2] = ScanCtrl();
  ctl->overflow = 0;
  ctl->r_nf = ctl->p_nf;
  ctl->r_mf = ctl->p_mf;
  ctl->r_visited_edges = ctl->p_visited_edges;
  ctl->r_visited_cnt = ctl->p_visited_cnt;
  ctl->r_phase = ctl->p_phase;
}

// the first of ring levels [0, nlevels) whose bitmap holds bit i; nlevels when none does
// (coalesced: the threads of a warp share words)
GL_DEV uint32_t bfs_first_level(const uint32_t* lv, uint32_t words, uint32_t nlevels, uint32_t i) {
  const uint32_t w = i >> 5, m = 1u << (i & 31);
  uint32_t l = 0;
  while (l < nlevels && !(lv[(size_t) l * words + w] & m)) ++l;
  return l;
}

// Spill: depth of every vertex found in ring levels [0, nlevels) goes to the
// int32 side array (absolute depth = base + ring index).
__global__ void k_bfs_spill(const uint32_t* lv, uint32_t words, uint32_t nlevels, uint32_t n,
                            uint32_t base, int32_t* spill) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t l = bfs_first_level(lv, words, nlevels, i);
  if (l < nlevels) spill[i] = (int32_t) (base + l);
}

struct BfsFusedArgs {
  PullArgs pa;
  EdgeRange er;
  uint32_t* lv;      // level bitmaps: lv + d*words
  uint32_t words;
  uint32_t max_lv;   // number of level bitmaps available
  uint32_t depth_base;  // absolute depth of ring level 0 (> 0 after a spill)
  uint32_t* vis;
  int direction_opt;
  uint32_t beta;     // pull -> push when n_f < V / beta ...
  unsigned long long nz_total;  // ... and many non-isolated vertices are still unvisited
  BfsFusedCtl* ctl;
  HubItem* hubs;
  uint32_t hub_cap, hub_deg;
  int hub_tma;       // hub phase staged through the TMA engine (GL_HUB_TMA=0: plain loads)
  const uint8_t* deg8;   // byte-sized degree classes for the frontier-edge statistic (OpBfsPush)
  uint32_t push_v;       // push levels sweep the frontier over lids [0, push_v)
  unsigned long long m_total;   // CSR entries of the graph (the push -> pull rule)
  uint32_t list_gap;             // pull levels try the tail list once at most this many vertices are unvisited
  uint32_t src;                  // the source's lid (k_bfs_fused, first launch)
  int has_src;
};

// Level 0 of a query that starts at a source, pushed: the frontier is the source alone, so the
// level is its row, split statically over every warp of the grid -- contiguous runs of 32-entry
// groups aligned to 128 bytes, at most kSrcGroups per warp and pass.  No work list, no ticket and no
// CTA barrier per item.  A warp issues all its column loads, then all its visited-bitmap reads, then the degree
// classes of the entries not yet visited (speculatively: deg8 depends on v only), and only then the
// bit updates group by group, so that the loads' latencies overlap instead of forming one chain per
// group.  The source counts as visited (thread 0 sets its bit concurrently): its own entries -- self
// loops -- never count.
constexpr uint32_t kSrcGroups = 8;
GL_DEV void bfs_source_row_push(const EdgeRange& er, const OpBfsPush& op, uint32_t src, ScanCtrl* C, ScanAcc& acc) {
  const uint64_t b = er.rp[src], e = er.rp[src + 1];
  const uint32_t* row = er.col + (b & ~31ull);   // the row from the start of its first group
  const uint64_t span = e - (b & ~31ull);
  const uint32_t ng = (uint32_t) ((span + 31) >> 5);   // the row's 32-entry groups (4-byte entries: < 2^32)
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t per = min((ng + warps - 1) / warps, kSrcGroups);
  const uint32_t lane = lane_id();
  for (uint32_t g = wid * per; g < ng; g += warps * per) {
    // the slice's entries are [lo, hi) from the start of its first group
    const uint32_t lo = g == 0 ? (uint32_t) b & 31u : 0u;
    const uint32_t hi = (uint32_t) min(span - ((uint64_t) g << 5), (uint64_t) per * 32);
    const uint32_t* q = row + ((uint64_t) g << 5) + lane;
    // (the per-entry state is packed: bit j of `unvis` / byte j of `cls` belong to v[j])
    uint32_t v[kSrcGroups];
#pragma unroll
    for (uint32_t j = 0; j < kSrcGroups; ++j) {
      const uint32_t o = 32 * j + lane;
      v[j] = (o >= lo && o < hi) ? ld_stream_u32(q + 32 * j) : src;   // src: no entry
    }
    uint32_t unvis = 0;
#pragma unroll
    for (uint32_t j = 0; j < kSrcGroups; ++j) unvis |= op.warp_edge_bit(v[j], v[j] != src) ? 1u << j : 0u;
    uint64_t cls = 0;
#pragma unroll
    for (uint32_t j = 0; j < kSrcGroups; ++j)
      if (((unvis >> j) & 1u) && op.deg8 && v[j] < op.ivnum) cls |= (uint64_t) op.deg8[v[j]] << (8 * j);
    // group by group: the entry at hand is always v[0] (the array shifts, so it stays in registers)
#pragma unroll 1
    for (uint32_t j = 0; j < per; ++j) {
      const uint32_t bit = (unvis & 1u) << (v[0] & 31);
      if (__any_sync(0xffffffffu, bit != 0) && op.warp_edge_set(v[0], bit))
        op.note_fresh(v[0], op.deg8 ? OpBfsPush::degree_of_class((uint32_t) cls & 0xFFu) : op.degree_of(v[0]), acc);
      unvis >>= 1;
      cls >>= 8;
#pragma unroll
      for (uint32_t k = 0; k + 1 < kSrcGroups; ++k) v[k] = v[k + 1];
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    C->scanned = e - b;
    C->frontier = 1;
  }
}

// flush_acc for a phase after which every warp of the grid holds counts (bfs_source_row_push, the
// pull levels of k_bfs_fused): the CTA sums them first and adds them with one atomic per counter:
// with an atomic per warp and counter (flush_acc), level 0 took 7 us longer on an H100 at 700 W.
// `pc` carries a pull level's scanned / frontier counts.  Leaves `acc` empty.
struct AccSmem {
  unsigned long long v[7][kTB / 32];
};
GL_DEV void flush_acc_cta(ScanAcc& acc, ScanCtrl* c, AccSmem& sm, const PullCounts& pc = PullCounts()) {
  static_assert(offsetof(ScanCtrl, touched) - offsetof(ScanCtrl, scanned) == 6 * sizeof(unsigned long long),
                "scanned, frontier, next_count, next_edges, remote_count, aux, touched are consecutive");
  const uint32_t wid = threadIdx.x >> 5;
  const unsigned long long x[7] = {pc.scanned, pc.frontier, acc.next_count, acc.next_edges, acc.remote, acc.aux,
                                   acc.touched};
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const unsigned long long s = warp_sum(x[k]);
    if (lane_id() == 0) sm.v[k][wid] = s;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    unsigned long long s = 0;
#pragma unroll
    for (int w = 0; w < kTB / 32; ++w) s += sm.v[threadIdx.x][w];
    if (s) atomicAdd(&c->scanned + threadIdx.x, s);
  }
  acc = ScanAcc();
}

// Level d reads lv[d] and writes lv[d+1] (pre-zeroed).  Every thread derives
// the push/pull decision from the same counters, so nothing is published
// between levels: one grid.sync per pull level, two per push level (tile
// phase | hub phase) except a first launch's level 0 (bfs_source_row_push).
// The control block starts zeroed (BfsApp::Init; k_bfs_resume_prep before a
// relaunch).
__global__ void __launch_bounds__(kTB, GL_BFS_FUSED_CTAS) k_bfs_fused(BfsFusedArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ __align__(128) union {
    ScanSmem<uint32_t> scan;
    PullSmem pull;
    HubTmaSmem hub;
    AccSmem acc;
  } sm;
  __shared__ uint32_t s_item;
  BfsFusedCtl* ctl = a.ctl;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  // running totals, replicated in every thread (the frontier's edges m_f are not kept: only the
  // phase rule reads them, right after a level, and a park reads them back from the counters)
  unsigned long long n_f, visited_edges, visited_cnt;
  const unsigned long long m_total = a.m_total;   // a kernel parameter: no register held across the levels
  uint32_t phase;
  if (a.depth_base == 0) {
    // first launch: the query starts here, with the source as the frontier of level 0
    const unsigned long long deg = a.has_src ? a.er.rp[a.src + 1] - a.er.rp[a.src] : 0ull;
    n_f = visited_cnt = a.has_src ? 1ull : 0ull;
    visited_edges = deg;
    phase = bfs_next_phase(0, n_f, deg, m_total - visited_edges, a.pa.ivnum, a.direction_opt, a.beta, a.nz_total,
                           kTailPerFrontier);
    if (gtid == 0) {
      ctl->t_begin = global_ns();
      if (a.has_src) {
        const uint32_t bit = 1u << (a.src & 31);
        a.lv[a.src >> 5] |= bit;
        atomicOr(a.vis + (a.src >> 5), bit);   // other warps may set bits of the same word
      }
    }
    // a pull level 0 reads both bitmaps (and owns visited words)
    if (phase != 0) grid.sync();
  } else {
    n_f = ctl->r_nf;
    visited_edges = ctl->r_visited_edges;
    visited_cnt = ctl->r_visited_cnt;
    phase = ctl->r_phase;
  }
  for (uint32_t depth = 0; n_f != 0; ++depth) {
    if (depth + 1 >= a.max_lv) {
      if (gtid == 0) {
        // m_f: the last level's next_edges (its counters are cleared one level later), else the launch's
        // start value (a first launch's level 0: the source's degree = visited_edges)
        const unsigned long long m_f = depth ? ((const volatile ScanCtrl*) &ctl->c[(depth + 2) % 3])->next_edges
                                             : (a.depth_base ? ctl->r_mf : visited_edges);
        bfs_park(ctl, n_f, m_f, visited_edges, visited_cnt, phase);
      }
      break;
    }
    ScanCtrl* C = &ctl->c[depth % 3];
    const uint32_t* cur = a.lv + (size_t) depth * a.words;
    uint32_t* nxt = a.lv + (size_t) (depth + 1) * a.words;
    ScanAcc acc;
    // A pull level lists its unresolved candidates once at most list_gap (> list_cap) non-isolated
    // vertices are unvisited: most of them are usually found by that level, and a list that comes out
    // longer than list_cap is simply not used (the next level sweeps the bitmap and tries again; the
    // attempt costs shared-memory appends).  The list's length travels from level to level in
    // C->aux_ticket.
    if (phase == kListPull) {
      const uint32_t n = ((const volatile ScanCtrl*) &ctl->c[(depth + 2) % 3])->aux_ticket;
      if (gtid == 0) C->aux_ticket = n;
      PullCounts pc;
      bfs_list_pull(a.pa, cur, a.vis, nxt, n, acc, pc);
      flush_acc_cta(acc, C, sm.acc, pc);
    } else if (phase == 1) {
      PullCounts pc;
      bfs_pull_phase<false, true>(sm.pull, a.pa, cur, a.vis, nxt, C, acc,
                                  a.pa.list_cap && a.nz_total <= visited_cnt + a.list_gap, &pc);
      // (sm.acc overlaps only the head of sm.pull.v, which the phase does not read after its last ticket)
      flush_acc_cta(acc, C, sm.acc, pc);
    } else {
      OpBfsPush op{a.vis, nxt, nullptr, a.er.rp, a.pa.ivnum, a.deg8};
      if (depth == 0 && a.depth_base == 0) {
        bfs_source_row_push(a.er, op, a.src, C, acc);
        flush_acc_cta(acc, C, sm.acc);
      } else {
        frontier_scan_phase<OpBfsPush>(sm.scan, cur, a.push_v, a.er, op, C, a.hubs, a.hub_cap, a.hub_deg, acc);
        grid.sync();
        if (a.hub_tma) hub_scan_phase_tma<OpBfsPush>(sm.hub, a.er, op, C, a.hubs, a.hub_cap, acc);
        else hub_scan_phase<OpBfsPush>(&s_item, a.er, op, C, a.hubs, a.hub_cap, acc);
        flush_acc(acc, C);
      }
    }
    grid.sync();
    const volatile ScanCtrl* VC = C;
    const unsigned long long next_count = VC->next_count;
    const unsigned long long next_edges = VC->next_edges;
    const bool listed = (phase == kListPull || (phase == 1 && a.pa.list_cap && a.nz_total <= visited_cnt + a.list_gap)) &&
                        VC->aux_ticket <= a.pa.list_cap;
    if (gtid == 0) bfs_level_end(ctl, a.depth_base, depth, n_f, (phase == 1 || phase == kListPull) ? 1u : 0u);
    n_f = next_count;
    visited_edges += next_edges;
    visited_cnt += next_count;
    // while a list is in use the level costs O(list) and one grid.sync: keep pulling (depths are the
    // same in either direction)
    phase = listed ? kListPull
                   : bfs_next_phase(phase, n_f, next_edges,
                                    m_total > visited_edges ? m_total - visited_edges : 0,
                                    a.pa.ivnum, a.direction_opt, a.beta,
                                    a.nz_total > visited_cnt ? a.nz_total - visited_cnt : 0, kTailPerFrontier);
  }
  if (gtid == 0) ctl->t_kend = global_ns();
}


// ---------------------------------------------------------------------------
// Fused whole-query BFS over SEVERAL fragments: one cooperative launch per GPU
// runs every level; the GPUs meet in device-side collectives over the NVLink-
// mapped landing areas (comm.h) — no host round trip, no kernel launch and no
// NCCL call between levels.
//   push level: scan | grid.sync | hub scan | grid.sync | pack outer hits into
//               the owners' landing slots | xsync (publishes item counts, sums
//               the frontier statistics) | apply received items
//   pull level: owners pack their frontier bits into the holders' mirror slots
//               | xsync | holders OR them into their outer copies | pull |
//               xsync (statistics)
// Every decision is derived from the all-reduced statistics, so all GPUs take
// the same branches and issue the same sequence of collectives.
// ---------------------------------------------------------------------------
struct BfsPayload {
  GL_DEV ItemU32 operator()(uint32_t, uint32_t lid) const { return ItemU32{lid}; }
};

struct XComm {
  uint32_t fid, fnum;
  int fid_offset;
  uint32_t id_mask;
  uint32_t capacity;                       // items per landing slot
  PeerSlot* const* slot_at_peer[2];        // [tag parity][fnum]: my slot in peer p's header
  const PeerSlot* local_slots;             // my header, parity 0 (parity 1 at + GL_MAX_FNUM)
  unsigned long long tag0;                 // first sequence number this launch may use
  char* const* send_slot[2];               // [msg parity][fnum]
  const char* const* recv_slot[2];
  uint32_t* const* peer_count[2];          // my count cell in peer p's header
  const uint32_t* local_counts;            // my header counts[2][GL_MAX_FNUM]
  uint32_t* send_count;                    // [fnum] local reservation counters
  uint32_t msg_round0, mirror_seq0;
  const uint32_t* mirror_lids;
  const uint64_t* mirror_off;
  MirrorBitsPlan plan;                     // word-parallel pack (plan.mask == null: lid-list pack)
  char* const* msend[2];
  const char* const* mrecv[2];
  const uint32_t* ghost_range;
  // replicated global frontier (pull levels): the mirror slots of one parity, seen as one
  // bitmap segment per owner fragment; seg_words = words of the largest fragment's segment
  int global_front;
  uint32_t seg_words, my_words;
  uint32_t seg_stride, seg_gens;   // words between two generations inside a slot; generations per parity
  int cta_fence;                   // 1: per-CTA fence.sys before a collective (see xsync)
};

struct XSmem {
  long long v[4][GL_MAX_FNUM];
  unsigned int total;
};

constexpr unsigned long long kXsyncTimeoutNs = 5000000000ull;

// Grid-wide + cross-GPU barrier and sum.  C != null: contribution =
// (next_count, items published, next_edges) of that control block; otherwise
// (e0, e1, 0).  publish_par >= 0: block 0 first publishes this round's item
// counts into the peers' headers.  Returns false when the launch must abort.
GL_DEV unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
GL_DEV void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// In-kernel collectives do not use PeerSlot::tag: each of the three 8-byte
// payload words carries a 16-bit stamp (0x4000 | tag mod 2^14) above a 48-bit
// value, so a contribution is three independent atomic 8-byte peer stores with
// no fence between payload and flag.  (The stamp can never equal the top bits
// of a raw value written by the host-launched k_peer_allreduce: 0 or 0xFFFF.)
GL_DEV unsigned long long x_stamp(unsigned long long tag) { return (0x4000ull | (tag & 0x3FFFull)) << 48; }

GL_DEV bool xsync(cg::grid_group& grid, const XComm& x, XSmem& xs, unsigned long long tag,
                  int publish_par, const ScanCtrl* C, long long e0, long long e1,
                  BfsFusedCtl* ctl, long long out[3], bool peer_stores = true, long long e2 = 0) {
  // The grid's peer stores (items, frontier words) must be visible system-wide before the stamps.
  // x.cta_fence = 0 (default): they happen-before block 0's fence.sys below through grid.sync()
  // (bar.sync + fence.gpu + barrier atomics: release/acquire at gpu scope), and fences are cumulative
  // in the PTX memory model -- ONE fence.sys per stamped word instead of one per CTA (fence.sys does
  // not scale: one per thread cost ~15 us per collective, one per storing CTA ~7-12 us).
  // x.cta_fence = 1 (GL_XSYNC_CTA_FENCE=1): every CTA that stored to a peer fences for itself first.
  if (x.cta_fence && __syncthreads_or(peer_stores ? 1 : 0)) {
    if (threadIdx.x == 0) __threadfence_system();
  }
  const bool tr = blockIdx.x == 0 && threadIdx.x == 0;
  if (tr) ctl->xt[0] = global_ns();
  grid.sync();
  if (tr) ctl->xt[1] = global_ns();
  if (blockIdx.x == 0) {
    const uint32_t p = threadIdx.x;
    if (p == 0) xs.total = 0;
    __syncthreads();
    if (publish_par >= 0 && p < x.fnum) {
      const uint32_t c = *(volatile uint32_t*) (x.send_count + p);
      if (p != x.fid) {
        *x.peer_count[publish_par][p] = c;   // NVLink peer store (ordered before the stamp by the fence below)
        atomicAdd(&xs.total, c);
        if (c > x.capacity) ctl->x_error = 2;
      }
      x.send_count[p] = 0;
    }
    __syncthreads();
    if (p < x.fnum) {
      unsigned long long i0 = (unsigned long long) e0, i1 = (unsigned long long) e1, i2 = (unsigned long long) e2;
      if (C) {
        const volatile ScanCtrl* VC = C;
        i0 = VC->next_count;
        i1 = xs.total;
        i2 = VC->next_edges;
      }
      const unsigned long long st = x_stamp(tag), vm = 0xFFFFFFFFFFFFull;
      PeerSlot* dst = x.slot_at_peer[tag & 1][p];
      __threadfence_system();   // the grid's peer stores and my count cell before my stamp
      st_relaxed_sys_u64((unsigned long long*) &dst->i0, st | (i0 & vm));
      st_relaxed_sys_u64((unsigned long long*) &dst->i1, st | (i1 & vm));
      st_relaxed_sys_u64((unsigned long long*) &dst->i2, st | (i2 & vm));
      const PeerSlot* src = x.local_slots + (tag & 1) * GL_MAX_FNUM + p;
      const unsigned long long t0 = global_ns();
      if (tr) ctl->xt[2] = t0;
      bool ok = true;
      unsigned long long r0, r1, r2;
      for (;;) {
        r0 = ld_acquire_sys_u64((const unsigned long long*) &src->i0);
        r1 = ld_acquire_sys_u64((const unsigned long long*) &src->i1);
        r2 = ld_acquire_sys_u64((const unsigned long long*) &src->i2);
        if ((r0 & ~vm) == st && (r1 & ~vm) == st && (r2 & ~vm) == st) break;
        __nanosleep(20);
        if (global_ns() - t0 > kXsyncTimeoutNs) {
          ok = false;
          break;
        }
      }
      if (!ok) ctl->x_error = 1;
      if (tr) ctl->xt[3] = global_ns();
      xs.v[0][p] = (long long) (r0 & vm);
      xs.v[1][p] = (long long) (r1 & vm);
      xs.v[2][p] = (long long) (r2 & vm);
    }
    __syncthreads();
    if (p == 0) {
      long long a = 0, b = 0, c = 0;
      for (uint32_t q = 0; q < x.fnum; ++q) {
        a += xs.v[0][q];
        b += xs.v[1][q];
        c += xs.v[2][q];
      }
      ctl->xres[0] = a;
      ctl->xres[1] = b;
      ctl->xres[2] = c;
      ctl->x_last_tag = tag;
      if (publish_par >= 0) ctl->x_items += xs.total;
      __threadfence();
    }
  }
  grid.sync();
  if (tr) ctl->xt[4] = global_ns();
  const volatile BfsFusedCtl* V = ctl;
  out[0] = V->xres[0];
  out[1] = V->xres[1];
  out[2] = V->xres[2];
  return V->x_error == 0;
}

// owner -> holders: the bits of `bitmap` at my mirrored inner vertices, then
// (after the barrier) OR the words received from every owner into my outer copies
GL_DEV bool mirror_pack(const XComm& x, uint32_t par, const uint32_t* bitmap) {
  const uint64_t nthreads = (uint64_t) gridDim.x * blockDim.x;
  const uint64_t gtid = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (x.plan.mask) return mirror_pack_bits_phase(x.plan, bitmap, x.msend[par], gtid, nthreads);
  for (uint32_t g = 0; g < x.fnum; ++g) {
    const uint64_t b = x.mirror_off[g], n = x.mirror_off[g + 1] - b;
    if (!n) continue;
    uint32_t* out = (uint32_t*) x.msend[par][g];
    const uint64_t npad = (n + 31) & ~31ull;
    for (uint64_t k = gtid; k < npad; k += nthreads) {
      bool bit = false;
      if (k < n) bit = bit_test(bitmap, x.mirror_lids[b + k]);
      const uint32_t w = __ballot_sync(0xffffffffu, bit);
      if (lane_id() == 0) out[k >> 5] = w;
    }
  }
  return true;
}
GL_DEV void mirror_unpack(const XComm& x, uint32_t par, uint32_t* bitmap) {
  const uint64_t nthreads = (uint64_t) gridDim.x * blockDim.x;
  const uint64_t gtid = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t f = 0; f < x.fnum; ++f) {
    const uint32_t base = x.ghost_range[f], n = x.ghost_range[f + 1] - base;
    if (!n || f == x.fid) continue;
    const uint32_t nw = (n + 31) >> 5;
    const uint32_t* in = (const uint32_t*) x.mrecv[par][f];
    for (uint64_t j = gtid; j < nw; j += nthreads) {
      const uint32_t w = __ldcg(in + j);   // written by the peer: bypass L1
      if (!w) continue;
      const uint32_t pos = base + ((uint32_t) j << 5), sh = pos & 31;
      atomicOr(bitmap + (pos >> 5), w << sh);
      if (sh) atomicOr(bitmap + (pos >> 5) + 1, w >> (32 - sh));
    }
  }
}
// Owner -> everybody: store the non-zero words of my frontier segment into the (parity, me)
// mirror slot of every fragment, my own included (the slots are kept zero between uses).
GL_DEV bool front_ship(const XComm& x, uint32_t par, uint32_t off, const uint32_t* bitmap) {
  const uint64_t nthreads = (uint64_t) gridDim.x * blockDim.x;
  const uint64_t gtid = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  bool wrote = false;
  for (uint64_t w = gtid; w < x.my_words; w += nthreads) {
    const uint32_t v = bitmap[w];
    if (!v) continue;
    for (uint32_t p = 0; p < x.fnum; ++p) {
      uint32_t* dst = (p == x.fid ? (uint32_t*) x.mrecv[par][p] : (uint32_t*) x.msend[par][p]) + off;
      dst[w] = v;
    }
    wrote = x.fnum > 1;
  }
  return wrote;
}
// the segments of parity `par` were consumed: back to zero for their next use.  16-byte loads, four
// segments' loads in flight per thread (one word per iteration made this a chain of ~30 dependent
// L2 latencies per level at eight fragments).
GL_DEV void front_zero(const XComm& x, uint32_t par, uint32_t off) {
  const uint64_t nthreads = (uint64_t) gridDim.x * blockDim.x;
  const uint64_t gtid = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n4 = x.seg_stride >> 2;   // a generation is seg_stride words (multiple of 64), zero-padded
  for (uint64_t i = gtid; i < n4; i += nthreads) {
    for (uint32_t f0 = 0; f0 < x.fnum; f0 += 4) {
      uint4 v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        v[k] = make_uint4(0u, 0u, 0u, 0u);
        if (f0 + k < x.fnum) v[k] = __ldcg((const uint4*) ((const uint32_t*) x.mrecv[par][f0 + k] + off) + i);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (v[k].x | v[k].y | v[k].z | v[k].w)
          ((uint4*) ((uint32_t*) x.mrecv[par][f0 + k] + off))[i] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

GL_DEV bool mirror_sync_bits(cg::grid_group& grid, const XComm& x, XSmem& xs, unsigned long long tag,
                             uint32_t par, uint32_t* bitmap, BfsFusedCtl* ctl) {
  const bool wrote = mirror_pack(x, par, bitmap);
  long long dummy[3];
  if (!xsync(grid, x, xs, tag, -1, nullptr, 0, 0, ctl, dummy, wrote)) return false;
  mirror_unpack(x, par, bitmap);
  grid.sync();
  return true;
}

struct BfsMultiArgs {
  BfsFusedArgs f;
  uint32_t* remote;
  uint32_t ovnum;
  const uint32_t* ovgid;
  unsigned long long g_m_total, g_vnum, g_nz_total;
  const uint32_t* dlg_list;   // delegated hubs (null: none)
  const uint64_t* dlg_off;
  XComm x;
};

// kGF: replicated global frontier (round 2) / per-holder bit-compressed slices (round 1) -- two
// instantiations, so that neither carries the other scheme's registers
template <bool kGF>
__global__ void __launch_bounds__(kTB, GL_BFS_FUSED_CTAS) k_bfs_fused_multi(BfsMultiArgs A) {
  cg::grid_group grid = cg::this_grid();
  __shared__ __align__(128) union {
    ScanSmem<uint32_t> scan;
    PullSmem pull;
    XSmem xs;
    PackSmem pack;
    HubTmaSmem hub;
  } sm;
  __shared__ uint32_t s_item;
  const BfsFusedArgs& a = A.f;
  const XComm& x = A.x;
  BfsFusedCtl* ctl = a.ctl;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t nthreads = (uint64_t) gridDim.x * blockDim.x;
  unsigned long long tag = x.tag0;
  uint32_t msg_round = x.msg_round0, mseq = x.mirror_seq0;
  unsigned long long n_f, m_f, visited_edges;
  unsigned long long visited_cnt = ctl->r_visited_cnt_g;   // whole graph (an upper bound: re-reported outer hits count twice)
  uint32_t phase = ctl->r_phase;
  bool premirrored = false;
  uint32_t hub_src = 0;    // first launch of a query whose source is delegated hub (hub_src - 1)
  uint32_t gen = 0;        // frontier generations shipped by this launch (global-frontier scheme)
  uint32_t cur_off = 0;    // word offset of the generation holding the current level's frontier
  int cur_cached = 1;
  long long S[3];
  if (gtid == 0) {
    ctl->x_last_tag = x.tag0 - 1;   // (same thread later records every collective)
    ctl->t_kstart = global_ns();
  }
  if (phase == 0xFFFFFFFFu) {
    // first launch of the query: the source's owner contributes (1, deg)
    // ... and, when the source is one of the delegated hubs, its index + 1 (everybody else adds 0)
    long long e2 = 0;
    if (A.dlg_list && ctl->has_src && ctl->src_lid < kDlgPerFrag) e2 = (long long) (x.fid * kDlgPerFrag + ctl->src_lid) + 1;
    if (!xsync(grid, x, sm.xs, tag++, -1, nullptr, (long long) ctl->r_nf, (long long) ctl->r_mf, ctl, S, true, e2)) return;
    hub_src = (uint32_t) S[2];
    n_f = (unsigned long long) S[0];
    m_f = (unsigned long long) S[1];
    visited_edges = m_f;
    visited_cnt = n_f;
    if (gtid == 0) ctl->l_nf = ctl->r_nf;   // this fragment's part of the current frontier (statistics)
    phase = 0;
  } else {
    n_f = ctl->r_nf;
    m_f = ctl->r_mf;
    visited_edges = ctl->r_visited_edges;
    if (gtid == 0) ctl->l_nf = n_f / x.fnum;   // resumed after a ring spill: the share is not carried over
  }
  for (uint32_t depth = 0; n_f != 0; ++depth) {
    if (depth + 1 >= a.max_lv) {
      if (gtid == 0) {
        bfs_park(ctl, n_f, m_f, visited_edges, 0, phase);
        ctl->r_visited_cnt_g = visited_cnt;
      }
      break;
    }
    // direction on WHOLE-GRAPH statistics (identical on every GPU).  Only the global-frontier scheme,
    // whose pull levels exchange no per-vertex messages, keeps pulling in the tail (a push level after
    // the pulls re-reports every outer neighbour of its frontier), also while fewer than V/64 candidates
    // remain: such a pull costs less than a push level's pack + message round + apply.
    const unsigned long long m_u = A.g_m_total > visited_edges ? A.g_m_total - visited_edges : 0;
    const unsigned long long unvis = A.g_nz_total > visited_cnt ? A.g_nz_total - visited_cnt : 0;
    const uint32_t nphase = bfs_next_phase(phase, n_f, m_f, m_u, A.g_vnum, a.direction_opt, a.beta, unvis,
                                           kGF ? kTailAbsolute : kNoTail);
    ScanCtrl* C = &ctl->c[depth % 3];
    uint32_t* cur = a.lv + (size_t) depth * a.words;
    uint32_t* nxt = a.lv + (size_t) (depth + 1) * a.words;
    ScanAcc acc;
    const uint32_t tl = a.depth_base + depth;
#define GL_MARK(k) do { if (gtid == 0 && tl < 32) ctl->ph[tl][k] = global_ns(); } while (0)
    GL_MARK(0);
    if (hub_src && depth == 0) {
      // level 0 from a delegated hub: every GPU marks its own neighbours of the source out of its
      // local list; nothing to pack, ship or apply
      OpBfsPush op{a.vis, nxt, A.remote, a.er.rp, a.pa.ivnum, a.deg8};
      const uint64_t b = A.dlg_off[hub_src - 1], e = A.dlg_off[hub_src];
      for (uint64_t i = b + gtid; i < e; i += nthreads) {
        const uint32_t v = A.dlg_list[i];
        if (bit_set_atomic(a.vis, v)) {
          bit_set_atomic(nxt, v);
          acc.touched++;
          acc.next_count++;
          acc.next_edges += op.degree_of(v);
        }
      }
      if (gtid == 0) {
        atomicAdd(&C->scanned, (unsigned long long) (e - b));
        if (ctl->has_src) atomicAdd(&C->frontier, 1ull);
      }
      flush_acc(acc, C);
      GL_MARK(1);
      bool wrote = false;
      if (kGF) {
        // a hub's neighbourhood is almost always followed by a pull level: its frontier words ride with
        // this level's statistics collective (a push level next zeroes the unused shipment, as after a pull)
        grid.sync();   // the words of nxt are final
        ++mseq;
        cur_off = ((gen >> 1) % x.seg_gens) * x.seg_stride;
        cur_cached = (gen >> 1) < x.seg_gens;
        ++gen;
        wrote = front_ship(x, mseq & 1, cur_off, nxt);
        premirrored = true;
      }
      GL_MARK(2);
      GL_MARK(3);
      if (!xsync(grid, x, sm.xs, tag++, -1, C, 0, 0, ctl, S, wrote)) return;
      GL_MARK(4);
      GL_MARK(5);
    } else if (nphase != 1) {
      if (premirrored && kGF) {
        front_zero(x, mseq & 1, cur_off);   // the speculative shipment of this frontier stays unused
        grid.sync();
      }
      premirrored = false;   // (a speculative shipment of this frontier stays unused)
      if (phase == 1 && !kGF) {
        // leaving the pull phase: outer copies learn which vertices their
        // owners visited meanwhile, so they are not reported again
        // (global-frontier scheme: skipped -- a holder may report an already visited vertex once
        //  more, the owner's visited test drops it; the tail frontiers are tiny)
        ++mseq;
        if (!mirror_sync_bits(grid, x, sm.xs, tag++, mseq & 1, a.vis, ctl)) return;
      }
      OpBfsPush op{a.vis, nxt, A.remote, a.er.rp, a.pa.ivnum, a.deg8};
      GL_MARK(1);
      frontier_scan_phase<OpBfsPush>(sm.scan, cur, a.pa.ivnum, a.er, op, C, a.hubs, a.hub_cap, a.hub_deg, acc);
      grid.sync();
      if (a.hub_tma) hub_scan_phase_tma<OpBfsPush>(sm.hub, a.er, op, C, a.hubs, a.hub_cap, acc);
      else hub_scan_phase<OpBfsPush>(&s_item, a.er, op, C, a.hubs, a.hub_cap, acc);
      flush_acc(acc, C);
      grid.sync();
      GL_MARK(2);
      // report newly reached outer copies to their owners (k_pack_outer)
      const uint32_t par = msg_round & 1;
      bool wrote_items = false;
      {
        MsgView mv;
        mv.fid = x.fid;
        mv.fnum = x.fnum;
        mv.fid_offset = x.fid_offset;
        mv.id_mask = x.id_mask;
        mv.item_bytes = 4;
        mv.capacity = x.capacity;
        mv.send_slot = x.send_slot[par];
        mv.send_count = x.send_count;
        mv.recv_slot = nullptr;
        mv.recv_count = nullptr;
        wrote_items = pack_outer_phase<ItemU32, BfsPayload>(sm.pack, A.remote, a.pa.ivnum, A.ovnum, A.ovgid, mv,
                                                            BfsPayload(), true);
      }
      GL_MARK(3);
      if (!xsync(grid, x, sm.xs, tag++, (int) par, C, 0, 0, ctl, S, wrote_items)) return;
      GL_MARK(4);
      if (S[1] > 0) {
        // apply what the other fragments found (ParallelProcess, bfs.h:158-166)
        for (uint32_t src = 0; src < x.fnum; ++src) {
          if (src == x.fid) continue;
          const uint32_t n = __ldcg(x.local_counts + par * GL_MAX_FNUM + src);
          const uint32_t* items = (const uint32_t*) x.recv_slot[par][src];
          for (uint64_t i = gtid; i < n; i += nthreads) {
            const uint32_t v = __ldcg(items + i);
            if (bit_set_atomic(a.vis, v)) bit_set_atomic(nxt, v);
          }
        }
        grid.sync();
      }
      GL_MARK(5);
      ++msg_round;
    } else {
      if (kGF) {
        if (!premirrored) {
          // the frontier came out of a push level: replicate my segment of it now
          ++mseq;
          cur_off = ((gen >> 1) % x.seg_gens) * x.seg_stride;
          cur_cached = (gen >> 1) < x.seg_gens;
          ++gen;
          const bool wrote0 = front_ship(x, mseq & 1, cur_off, cur);
          long long dummy[3];
          if (!xsync(grid, x, sm.xs, tag++, -1, nullptr, 0, 0, ctl, dummy, wrote0)) return;
        }
        GL_MARK(1);
        PullArgs pa = a.pa;
        pa.seg = (const uint32_t* const*) x.mrecv[mseq & 1];   // every owner's segment of this level's frontier
        pa.seg_off = cur_off;
        pa.seg_cached = cur_cached;
        // the next level's frontier is shipped word by word out of the pull itself (into the next
        // generation of the other parity) and becomes visible with the statistics collective
        const uint32_t nxt_off = ((gen >> 1) % x.seg_gens) * x.seg_stride;
        const int nxt_cached = (gen >> 1) < x.seg_gens;
        pa.ship_send = x.msend[(mseq + 1) & 1];
        pa.ship_recv = x.mrecv[(mseq + 1) & 1];
        pa.ship_fid = x.fid;
        pa.ship_fnum = x.fnum;
        pa.ship_off = nxt_off;
        const bool wrote = bfs_pull_phase<true>(sm.pull, pa, cur, a.vis, nxt, C, acc);
        flush_acc(acc, C);
        GL_MARK(2);
        if (!xsync(grid, x, sm.xs, tag++, -1, C, 0, 0, ctl, S, wrote)) return;
        // every CTA of this GPU is past the pull (xsync's barriers): the consumed generation goes back
        // to zero for a later query / a wrapped generation; nobody reads it before a later barrier
        front_zero(x, mseq & 1, cur_off);
        ++mseq;
        cur_off = nxt_off;
        cur_cached = nxt_cached;
        ++gen;
        premirrored = true;
        GL_MARK(4);
      } else {
      if (!premirrored) {
        ++mseq;
        if (!mirror_sync_bits(grid, x, sm.xs, tag++, mseq & 1, cur, ctl)) return;
      } else {
        // the previous pull level already shipped this frontier with its statistics
        mirror_unpack(x, mseq & 1, cur);
        grid.sync();
      }
      GL_MARK(1);
      bfs_pull_phase<false>(sm.pull, a.pa, cur, a.vis, nxt, C, acc);
      flush_acc(acc, C);
      grid.sync();
      GL_MARK(2);
      // A pull level is usually followed by another one: ship the new frontier's
      // bits to the holders NOW, so the statistics collective is also the mirror
      // barrier of the next level (one cross-GPU exchange per pull level, not two)
      ++mseq;
      const bool wrote = mirror_pack(x, mseq & 1, nxt);
      if (!xsync(grid, x, sm.xs, tag++, -1, C, 0, 0, ctl, S, wrote)) return;
      premirrored = true;
      GL_MARK(4);
      }
    }
#undef GL_MARK
    phase = nphase;
    if (gtid == 0) {
      if (tl < 32) {
        ctl->xw[tl][0] = ctl->xt[3] - ctl->xt[2];
        ctl->xw[tl][1] = ctl->xt[1] - ctl->xt[0];
      }
      // the statistics record THIS fragment's share of the level's frontier (n_f is the whole graph's):
      // a push level's is what its scan expanded; a pull level's is what the fragment found itself in
      // the previous level (vertices that arrived as messages in a push level before it are not counted)
      bfs_level_end(ctl, a.depth_base, depth, phase == 1 ? ctl->l_nf : ((const volatile ScanCtrl*) C)->frontier,
                    phase == 1 ? 1u : 0u);
      ctl->l_nf = ((const volatile ScanCtrl*) C)->next_count;
      ctl->x_msg_rounds = msg_round - x.msg_round0;
      ctl->x_mirror_syncs = mseq - x.mirror_seq0;
    }
    n_f = (unsigned long long) (S[0] + S[1]);
    m_f = (unsigned long long) S[2];
    visited_edges += m_f;
    visited_cnt += n_f;
  }
  if (gtid == 0) ctl->t_kend = global_ns();
}

struct BfsApply {
  uint32_t* cur;
  uint32_t* vis;
  const uint64_t* rp;
  GL_DEV void operator()(const ItemU32& it, ScanAcc& acc) const {
    uint32_t v = it.lid;
    if (bit_set_atomic(vis, v)) {  // bfs.h:158-166 (curr_depth < depth[v])
      bit_set_atomic(cur, v);
      acc.aux++;
      acc.next_edges += rp[v + 1] - rp[v];
    }
  }
};

// depth[v] = first level whose bitmap holds v
// (perm != null: the bitmaps are indexed by the hub-first rank of the vertex)
// (spill != null: levels older than `base` were moved to the side array)
__global__ void k_depth_from_levels(const uint32_t* lv, uint32_t words,
                                    uint32_t nlevels, uint32_t n, const uint32_t* perm,
                                    uint32_t base, const int32_t* spill, int64_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t pi = perm ? perm[i] : i;
  if (spill && spill[pi] >= 0) {
    out[i] = spill[pi];
    return;
  }
  const uint32_t l = bfs_first_level(lv, words, nlevels, pi);
  out[i] = l < nlevels ? (int64_t) base + l : INT64_MAX;
}

// depth as ONE byte per vertex (0xFF = unreached): 8x fewer bytes across PCIe
// than the reference's int64 depth array; gl_app_result widens on the host
__global__ void k_depth_u8_from_levels(const uint32_t* lv, uint32_t words, uint32_t nlevels, uint32_t n,
                                       const uint32_t* perm, uint8_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t l = bfs_first_level(lv, words, nlevels, perm ? perm[i] : i);
  out[i] = (uint8_t) (l < nlevels ? l : 0xFFu);
}

struct BfsApp : gl_app {
  DevBuf<uint32_t> lv, vis, remote, hub_nbr;
  DevBuf<int64_t> out64;
  // the adjacency BFS runs on: the fragment's own CSR, or (single fragment) a
  // hub-first relabelled shadow copy — see hub_order.cu
  const uint64_t* g_rp = nullptr;
  const uint32_t* g_col = nullptr;
  const uint32_t* g_nz = nullptr;
  // adjacency the pull step scans (== g_* unless the fragment is directed)
  const uint64_t* p_rp = nullptr;
  const uint32_t* p_col = nullptr;
  DevBuf<uint32_t> nz_in;   // directed: inner vertices with in-degree > 0
  // several fragments, fused kernel: gid-space copies for the replicated global frontier
  DevBuf<uint32_t> gcol, hub_nbr_g;
  DevBuf<uint32_t> dlg_list;   // delegated hubs: my inner neighbours of hub h = dlg_list[dlg_off[h] .. dlg_off[h + 1])
  DevBuf<uint64_t> dlg_off;
  DevBuf<uint32_t> ovgid_p;   // hub-first order over several fragments: the outer copies' gids in the owners' new lid space
  bool hub_multi = false;
  uint32_t seg_words = 0, seg_stride = 0, seg_gens = 1;
  bool global_front = false;
  DevBuf<uint32_t> perm, order, nz_p, col_p;
  DevBuf<uint64_t> rp_p;
  // one fragment in hub-first order: rows of two or more entries are lids [0, multi_v); the fused
  // kernel's tail candidate list (kTailList entries)
  static constexpr uint32_t kTailList = 1u << 16;
  static constexpr uint32_t kListTry = 16;   // the list is tried from kListTry x kTailList unvisited vertices on
  uint32_t multi_v = 0;
  DevBuf<uint32_t> tail_list;
  uint32_t src_ = 0;
  int has_src_ = 0;
  unsigned long long nz_total = 0, visited_cnt = 0;
  size_t words = 0;
  uint32_t tvnum = 0;
  uint32_t max_lv = 0;
  uint32_t used_lv = 0;     // level bitmaps dirtied by the previous query
  uint32_t curr_depth = 0;
  // frontier statistics driving the push/pull switch (stepwise path)
  uint64_t n_f = 0, m_f = 0, visited_edges = 0;
  uint64_t g_m_total = 0, g_vnum = 0, g_nz_total = 0;   // whole-graph totals (all fragments)
  uint32_t phase = 0;
  DevBuf<BfsFusedCtl> d_ctl;
  PinnedBuf<BfsFusedCtl> h_ctl;
  int fused_grid = 0;

  ~BfsApp() override {
    if (ev_done) cudaEventDestroy(ev_done);
    for (auto e : ev8)
      if (e) cudaEventDestroy(e);
  }
  size_t ResultElemBytes() const override { return sizeof(int64_t); }

  uint32_t* level_bm(uint32_t d) { return lv + (size_t) d * words; }
  // pull -> push when the frontier shrinks below V / beta (bfs_next_phase), on every query path
  uint32_t beta() const { return cfg.reserved[2] > 0 ? (uint32_t) cfg.reserved[2] : 24u; }

  // The pull step walks the INCOMING adjacency (bfs.h:225-238): `ie` when the
  // fragment is directed, the (aliased) `oe` when it is not.  A directed
  // fragment that was created without an ie CSR (gl_frag_create, kOnlyOut)
  // can only push; levels are identical either way.
  bool can_pull() const { return cfg.direction_opt && (!fv.directed || !frag->ie_alias_oe); }

  // Hub-first shadow graph (hub_order.cu): BFS runs on a copy of the adjacency with the inner vertices
  // relabelled by descending degree, and the source moves to its new lid.
  int BuildHubFirst() {
    GL_TRY(build_hub_order(eng.stream, fv.oe_rp, fv.ivnum, &perm, &order));
    GL_TRY(build_permuted_csr(eng.stream, fv.oe_rp, fv.oe_col, frag->oe.entries, fv.ivnum, order, perm, &rp_p, &col_p));
    GL_CUDA(nz_p.alloc(words));
    GL_CUDA(cudaMemsetAsync(nz_p, 0, sizeof(uint32_t) * words, eng.stream));
    if (fv.ivnum) GL_LAUNCH(k_bfs_nz, (fv.ivnum + 255) / 256, 256, eng.stream, rp_p, fv.ivnum, nz_p);
    g_rp = rp_p;
    g_col = col_p;
    g_nz = nz_p;
    if (has_src_) GL_CUDA(cudaMemcpy(&src_, perm + src_, 4, cudaMemcpyDeviceToHost));
    return GL_OK;
  }

  // Several fragments, replicated global frontier: gid-space copies of the pull adjacency (gcol) and of
  // the hub-neighbour table (hub_nbr_g); `ovgid` = the gids of the outer copies.  sorted: the rows are
  // re-sorted by rank key and hub_nbr_g is read off their first column (hub-first order); otherwise
  // hub_nbr_g maps hub_nbr.
  int BuildGidPull(const uint32_t* ovgid, bool sorted) {
    const uint64_t m = fv.directed ? frag->ie.entries : frag->oe.entries;
    const uint32_t gid0 = fv.fid << fv.fid_offset;
    GL_CUDA(gcol.alloc(m + 16));
    GL_CUDA(hub_nbr_g.alloc((size_t) fv.ivnum + kSuperV));
    GL_CUDA(cudaMemsetAsync(hub_nbr_g, 0xFF, sizeof(uint32_t) * ((size_t) fv.ivnum + kSuperV), eng.stream));
    if (m) GL_LAUNCH(k_bfs_gcol, eng.sm_count * 8, 256, eng.stream, p_col, m, fv.ivnum, gid0, ovgid, gcol);
    if (sorted && m) {
      GL_LAUNCH(k_bfs_gid_key, eng.sm_count * 8, 256, eng.stream, gcol, m, fv.fid_offset, fv.id_mask, 1);
      GL_TRY(sort_csr_rows(eng.stream, p_rp, fv.ivnum, m, &gcol));
      GL_LAUNCH(k_bfs_gid_key, eng.sm_count * 8, 256, eng.stream, gcol, m, fv.fid_offset, fv.id_mask, 0);
    }
    if (!fv.ivnum) return GL_OK;
    // the first entry of a sorted row is its highest-ranked neighbour: the stage-1 probe of the pull
    if (sorted) GL_LAUNCH(k_bfs_first_col, (fv.ivnum + 255) / 256, 256, eng.stream, p_rp, gcol, fv.ivnum, hub_nbr_g);
    else GL_LAUNCH(k_bfs_gid_table, (fv.ivnum + 255) / 256, 256, eng.stream, hub_nbr, fv.ivnum, fv.ivnum, gid0, ovgid, hub_nbr_g);
    return GL_OK;
  }

  // Decide the vertex order first (one fragment: on local facts; several: on the collective totals),
  // then build the adjacency, its tables and the statistics once, on that order.
  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    words = (bm_words(tvnum) + 4) & ~(size_t) 3;
    // one bitmap per BFS level: up to 1 GiB of them, at most 4096
    size_t budget = (size_t) 1 << 30;
    max_lv = (uint32_t) std::max<size_t>(16, std::min<size_t>(4096, budget / (words * 4)));
    if (cfg.reserved[3] >= 4) max_lv = (uint32_t) cfg.reserved[3];   // test hook: tiny ring => spills
    GL_CUDA(lv.alloc(words * max_lv));
    GL_CUDA(cudaMemsetAsync(lv, 0, sizeof(uint32_t) * words * max_lv, eng.stream));
    GL_CUDA(vis.alloc(words));
    GL_CUDA(remote.alloc(words));
    GL_CUDA(hub_nbr.alloc((size_t) fv.ivnum + kSuperV));
    GL_CUDA(cudaMemsetAsync(hub_nbr, 0xFF, sizeof(uint32_t) * ((size_t) fv.ivnum + kSuperV), eng.stream));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    GL_CUDA(d_ctl.alloc(1));
    GL_CUDA(h_ctl.alloc(1));
    memset(h_ctl, 0, sizeof(BfsFusedCtl));
    g_rp = fv.oe_rp;
    g_col = fv.oe_col;
    g_nz = frag->nonzero_deg;
    // the source is fixed per app (AppConfig): resolve it once
    has_src_ = gl_frag_oid2lid(frag, cfg.source_oid, &src_) == GL_OK ? 1 : 0;
    used_lv = 0;
    // message = bare lid (bfs.h:50-51: sizeof(vid_t) per outer vertex)
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32)));
    g_m_total = frag->oe.entries;
    g_vnum = fv.ivnum;
    // hub-first shadow graph (one fragment, undirected, large enough to matter)
    bool hub_first = fv.fnum == 1 && can_pull() && !fv.directed &&
                     ((fv.ivnum >= (1u << 16) && cfg.reserved[1] == 0) || cfg.reserved[1] == 2);
    if (fv.fnum > 1) {
      GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
      long long a = (long long) frag->oe.entries, b = (long long) fv.ivnum;
      double c = 0;
      GL_TRY(mm.PeerAllReduce(eng.stream, &a, &b, &c, 0));
      g_m_total = (uint64_t) a;
      g_vnum = (uint64_t) b;
      // every GPU must spill its level ring at the same depth
      long long lo = (long long) max_lv, dummy = 0;
      GL_TRY(mm.PeerAllReduce(eng.stream, &lo, &dummy, &c, 1));
      max_lv = (uint32_t) lo;
      // Replicated global frontier for the pull levels of the fused kernel (cfg.reserved[7] = 1: the
      // round-1 scheme, per-holder bit-compressed shipments): gid copies of the pull adjacency and of
      // the hub-neighbour table; the mirror slots of one parity hold one frontier segment per owner.
      long long mw = (long long) bm_words(fv.ivnum), unused = 0;
      GL_TRY(mm.PeerAllReduce(eng.stream, &mw, &unused, &c, 2));
      seg_words = (uint32_t) mw;
      // a mirror slot (8 B per inner vertex) holds many 1-bit-per-vertex segments: one GENERATION per pull
      // level, so that a level's frontier bits sit at addresses no SM has cached yet (front_test)
      seg_stride = (seg_words + 63) & ~63u;
      seg_gens = (uint32_t) std::min<size_t>(32, seg_stride ? comm->mirror_bytes / ((size_t) seg_stride * 4) : 0);
      global_front = can_pull() && cfg.reserved[7] == 0 && seg_gens >= 2;
      // Hub-first order inside every fragment (as on one GPU): inner lids become degree ranks, so the
      // hot frontier / visited words are the first words of every segment, and the pull rows list the
      // highest-ranked neighbours first.  Decided on facts every rank shares (the steps below are
      // collective).  cfg.reserved[1] = 1 keeps the fragment's own order, 2 forces the hub-first
      // one also on small graphs (tests).
      hub_multi = global_front && fused() && !fv.directed &&
                  ((cfg.reserved[1] == 0 && g_vnum >= (1u << 16)) || cfg.reserved[1] == 2 || cfg.reserved[1] == 3);
      hub_first = hub_multi;
    }
    if (hub_first) GL_TRY(BuildHubFirst());
    p_rp = g_rp;
    p_col = g_col;
    if (fv.directed && can_pull()) {
      p_rp = fv.ie_rp;
      p_col = fv.ie_col;
      GL_CUDA(nz_in.alloc(words));
      GL_CUDA(cudaMemsetAsync(nz_in, 0, sizeof(uint32_t) * words, eng.stream));
      if (fv.ivnum) GL_LAUNCH(k_bfs_nz, (fv.ivnum + 255) / 256, 256, eng.stream, p_rp, fv.ivnum, nz_in);
      g_nz = nz_in;   // pull candidates / "still reachable" statistics: in-degree > 0
    }
    if (fv.ivnum && cfg.direction_opt) {
      GL_CUDA(deg8.alloc(fv.ivnum));
      GL_LAUNCH(k_bfs_deg8, (fv.ivnum + 255) / 256, 256, eng.stream, g_rp, fv.ivnum, deg8);
    }
    if (fv.fnum == 1 && fv.ivnum && can_pull()) {
      // hub-first order: the first entry of a sorted row is its highest-degree neighbour, and the pull
      // relies on hub_nbr[v] being that entry (stage 2 starts after it)
      if (perm) GL_LAUNCH(k_bfs_first_col, (fv.ivnum + 255) / 256, 256, eng.stream, p_rp, p_col, fv.ivnum, hub_nbr);
      else GL_LAUNCH(k_bfs_hub_nbr, eng.sm_count * 8, 256, eng.stream, p_rp, p_col, fv.ivnum, hub_nbr);
    }
    {
      DevBuf<unsigned long long> d_cnt;
      GL_CUDA(d_cnt.alloc(2));
      GL_CUDA(cudaMemsetAsync(d_cnt, 0, 16, eng.stream));
      GL_LAUNCH(k_bfs_popc, eng.sm_count * 4, 256, eng.stream, g_nz, (uint32_t) bm_words(fv.ivnum), d_cnt);
      GL_CUDA(cudaMemcpyAsync(&nz_total, d_cnt, 8, cudaMemcpyDeviceToHost, eng.stream));
      unsigned long long m2 = 0;
      if (fv.fnum == 1 && perm) {
        // descending degree: the rows of two or more entries are a prefix of the lids
        GL_LAUNCH(k_bfs_count_rows, eng.sm_count * 4, 256, eng.stream, p_rp, fv.ivnum, (uint64_t) 2, d_cnt + 1);
        GL_CUDA(cudaMemcpyAsync(&m2, d_cnt + 1, 8, cudaMemcpyDeviceToHost, eng.stream));
        GL_CUDA(tail_list.alloc(kTailList));
      }
      GL_CUDA(cudaStreamSynchronize(eng.stream));
      multi_v = (uint32_t) m2;
    }
    if (fv.fnum == 1) return GL_OK;
    {
      long long z = (long long) nz_total, z2 = 0;
      double c = 0;
      GL_TRY(mm.PeerAllReduce(eng.stream, &z, &z2, &c, 0));
      g_nz_total = (uint64_t) z;
    }
    if (hub_multi) {
      // owners' new lids reach the outer copies through one dense mirror sync
      DevBuf<uint32_t> newlid;
      GL_CUDA(newlid.alloc(std::max<size_t>(tvnum, 1)));
      GL_CUDA(cudaMemsetAsync(newlid, 0, sizeof(uint32_t) * std::max<size_t>(tvnum, 1), eng.stream));
      if (fv.ivnum) GL_CUDA(cudaMemcpyAsync(newlid, perm, sizeof(uint32_t) * fv.ivnum, cudaMemcpyDeviceToDevice, eng.stream));
      GL_TRY(mm.SyncValuesToGhosts(eng.stream, newlid, 4));
      GL_CUDA(ovgid_p.alloc(std::max<uint32_t>(fv.ovnum, 1)));
      if (fv.ovnum)
        GL_LAUNCH(k_bfs_ovgid_new, (fv.ovnum + 255) / 256, 256, eng.stream, fv.ovgid, newlid + fv.ivnum, fv.ovnum, fv.id_mask, ovgid_p);
      GL_TRY(BuildGidPull(ovgid_p, true));
      if (cfg.reserved[1] != 3) {   // ([1] = 3: hub-first order without the delegated hubs, A/B)
        const uint32_t K = fv.fnum * kDlgPerFrag;
        DevBuf<uint32_t> cnt;
        GL_CUDA(cnt.alloc(K));
        GL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * K, eng.stream));
        if (fv.ivnum)
          GL_LAUNCH(k_bfs_dlg_scan, (fv.ivnum + 255) / 256, 256, eng.stream, p_rp, gcol, fv.ivnum, fv.fid_offset, fv.id_mask, cnt,
                    nullptr, nullptr, 0);
        std::vector<uint32_t> h_cnt(K);
        GL_CUDA(cudaMemcpyAsync(h_cnt.data(), cnt, sizeof(uint32_t) * K, cudaMemcpyDeviceToHost, eng.stream));
        GL_CUDA(cudaStreamSynchronize(eng.stream));
        std::vector<uint64_t> h_off(K + 1, 0);
        for (uint32_t h = 0; h < K; ++h) h_off[h + 1] = h_off[h] + h_cnt[h];
        GL_CUDA(dlg_off.alloc(K + 1));
        GL_CUDA(cudaMemcpyAsync(dlg_off, h_off.data(), sizeof(uint64_t) * (K + 1), cudaMemcpyHostToDevice, eng.stream));
        GL_CUDA(dlg_list.alloc(h_off[K] + 16));
        GL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * K, eng.stream));
        if (fv.ivnum)
          GL_LAUNCH(k_bfs_dlg_scan, (fv.ivnum + 255) / 256, 256, eng.stream, p_rp, gcol, fv.ivnum, fv.fid_offset, fv.id_mask, cnt,
                    dlg_off, dlg_list, 1);
        GL_TRY(sort_csr_rows(eng.stream, dlg_off, K, h_off[K], &dlg_list));   // ascending lid: neighbouring bits, neighbouring words
        GL_CUDA(cudaStreamSynchronize(eng.stream));
      }
      GL_CUDA(cudaStreamSynchronize(eng.stream));
    } else if (can_pull() && tvnum) {
      // the hub-neighbour prefilter should pick the true highest-degree neighbour, also when it is an
      // outer copy: owners' degrees reach the ghosts through one dense mirror sync (collective)
      DevBuf<uint32_t> deg32;
      GL_CUDA(deg32.alloc(tvnum));
      GL_LAUNCH(k_bfs_deg32, (tvnum + 255) / 256, 256, eng.stream, fv.oe_rp, fv.ivnum, tvnum, deg32);
      GL_TRY(mm.SyncValuesToGhosts(eng.stream, deg32, 4));
      if (fv.ivnum) GL_LAUNCH(k_bfs_hub_nbr, eng.sm_count * 8, 256, eng.stream, p_rp, p_col, fv.ivnum, hub_nbr, deg32);
      GL_CUDA(cudaStreamSynchronize(eng.stream));
    } else if (can_pull()) {
      GL_TRY(mm.SyncValuesToGhosts(eng.stream, nullptr, 4));   // keep the collective sequence identical on every rank
    }
    if (global_front && !hub_multi) {
      GL_TRY(BuildGidPull(fv.ovgid, false));
      GL_CUDA(cudaStreamSynchronize(eng.stream));
    }
    return GL_OK;
  }

  int Init() override {
    cudaStream_t s = eng.stream;
    uint32_t dirty = spilled ? max_lv : std::min<uint32_t>(max_lv, used_lv + 2);
    GL_CUDA(cudaMemsetAsync(lv, 0, sizeof(uint32_t) * words * dirty, s));
    if (spilled) GL_CUDA(cudaMemsetAsync(spill, 0xFF, sizeof(int32_t) * std::max<uint32_t>(fv.ivnum, 1), s));
    spilled = false;
    depth_base = 0;
    GL_CUDA(cudaMemsetAsync(vis, 0, sizeof(uint32_t) * words, s));
    GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
    // the fused kernels' level counters and query totals start from zero
    GL_CUDA(cudaMemsetAsync(d_ctl, 0, sizeof(BfsFusedCtl), s));
    if (global_front && comm->mirror_dirty) {
      // the frontier segments (the first seg_words words of every mirror slot) must be zero when the
      // query starts; the fused kernel leaves them zero, other users of the mirror area do not.
      // Collective by construction: every rank sees the same history of mirror-area users.
      GL_TRY(mm.PeerBarrier(s));
      for (int par = 0; par < 2; ++par)
        for (uint32_t f = 0; f < fv.fnum; ++f)
          GL_CUDA(cudaMemsetAsync(comm->local_base + comm->mirror_off(par, f), 0, (size_t) seg_stride * 4 * seg_gens, s));
      GL_CUDA(cudaStreamSynchronize(s));
      GL_TRY(mm.PeerBarrier(s));
      comm->mirror_dirty = false;
    }
    curr_depth = 0;
    used_lv = 0;
    n_f = m_f = visited_edges = 0;
    visited_cnt = 1;
    phase = 0;
    rounds_noted = false;
    pending_stats = false;
    return GL_OK;
  }

  // The level-bitmap ring is full (ring level max_lv-1 holds the unprocessed
  // frontier): move the depths of ring levels [0, max_lv-1) to the int32 side
  // array, restart the ring with the frontier at level 0.  BFS depth is then
  // only bounded by int32 like the reference's depth array (bfs.h:31).
  DevBuf<int32_t> spill;
  bool spilled = false;
  uint32_t depth_base = 0;
  int SpillRing() {
    cudaStream_t s = eng.stream;
    if (!spill) {
      GL_CUDA(spill.alloc(std::max<uint32_t>(fv.ivnum, 1)));
      GL_CUDA(cudaMemsetAsync(spill, 0xFF, sizeof(int32_t) * std::max<uint32_t>(fv.ivnum, 1), s));
    }
    if (fv.ivnum)
      GL_LAUNCH(k_bfs_spill, (fv.ivnum + 255) / 256, 256, s, lv, (uint32_t) words, max_lv - 1, fv.ivnum, depth_base, spill);
    GL_CUDA(cudaMemcpyAsync(lv, level_bm(max_lv - 1), sizeof(uint32_t) * words, cudaMemcpyDeviceToDevice, s));
    GL_CUDA(cudaMemsetAsync(level_bm(1), 0, sizeof(uint32_t) * words * (max_lv - 1), s));
    depth_base += max_lv - 1;
    spilled = true;
    return GL_OK;
  }

  PullArgs pull_args() const {
    return PullArgs{p_rp, p_col, hub_nbr, fv.ivnum, g_nz, nullptr, 0, 0, 0};
  }

  bool fused() const {
    return cfg.fuse_supersteps && (fv.fnum == 1 || (mm.use_peer_barrier && comm && comm->opened));
  }

  // Fused path: the whole query is one cooperative launch (PEval seeds and
  // launches; no IncEval round is needed afterwards).
  int RunFused() {
    cudaStream_t s = eng.stream;
    uint32_t src = 0;
    int has_src = has_src_;
    src = src_;   // already translated to the hub-first rank in Setup
    const bool multi = fv.fnum > 1;
    if (multi) GL_LAUNCH(k_bfs_seed_fused, 1, 32, s, src, has_src, level_bm(0), vis, g_rp, d_ctl);
    BfsFusedArgs a;
    a.pa = pull_args();
    a.er = EdgeRange{g_rp, g_col, nullptr};
    a.lv = lv;
    a.words = (uint32_t) words;
    a.max_lv = max_lv;
    a.vis = vis;
    a.direction_opt = can_pull() ? 1 : 0;
    a.beta = beta();
    a.nz_total = nz_total;
    a.m_total = g_m_total;
    a.ctl = d_ctl;
    a.hubs = eng.hubs;
    a.hub_cap = eng.hub_cap;
    a.hub_deg = eng.hub_deg;
    a.deg8 = deg8;
    // inside the fused kernel the TMA-staged hub phase is opt-in (GL_HUB_TMA=2); the stand-alone
    // k_hub_scan_tma is the default elsewhere
    a.hub_tma = (getenv("GL_HUB_TMA") && atoi(getenv("GL_HUB_TMA")) == 2) ? 1 : 0;
    a.src = src;
    a.has_src = has_src;
    // one fragment in hub-first order: the vertices with edges are lids [0, nz_total), so the sweeps
    // stop there (a push level also covers an isolated source)
    const bool hub_first = perm && !multi;
    a.pa.hub_first = hub_first ? 1u : 0u;
    a.pa.sweep_v = hub_first ? (uint32_t) nz_total : fv.ivnum;
    a.pa.multi_v = hub_first ? multi_v : 0u;
    a.push_v = hub_first ? std::min<uint32_t>(fv.ivnum, std::max<uint32_t>((uint32_t) nz_total, src + 1)) : fv.ivnum;
    a.pa.list = hub_first ? tail_list.get() : nullptr;
    a.pa.list_cap = hub_first ? kTailList : 0u;
    a.list_gap = kListTry * kTailList;
    if (!fused_grid)
      fused_grid = multi ? (global_front ? persistent_grid(k_bfs_fused_multi<true>, eng.sm_count)
                                         : persistent_grid(k_bfs_fused_multi<false>, eng.sm_count))
                         : persistent_grid(k_bfs_fused, eng.sm_count);
    BfsMultiArgs ma;
    if (multi) {
      ma.remote = remote;
      ma.ovnum = fv.ovnum;
      ma.ovgid = hub_multi ? ovgid_p : fv.ovgid;
      ma.g_m_total = g_m_total;
      ma.g_vnum = g_vnum;
      ma.g_nz_total = g_nz_total;
      ma.dlg_list = dlg_list;
      ma.dlg_off = dlg_off;
      XComm& x = ma.x;
      x.fid = fv.fid;
      x.fnum = fv.fnum;
      x.fid_offset = fv.fid_offset;
      x.id_mask = fv.id_mask;
      x.capacity = (uint32_t) std::min<size_t>(comm->landing_bytes / sizeof(ItemU32), 0xFFFFFFFFu);
      x.local_slots = (const PeerSlot*) (comm->local_base + GL_COMM_SLOT_OFF);
      x.local_counts = (const uint32_t*) comm->local_base;
      x.send_count = mm.d_send_count;
      x.mirror_lids = mm.d_mirror_lids;
      x.mirror_off = mm.d_mirror_off;
      x.plan = mm.bits_plan();
      if (!mm.mirror_sorted) x.plan.mask = nullptr;
      x.ghost_range = mm.d_ghost_range;
      x.global_front = global_front ? 1 : 0;
      x.seg_words = seg_words;
      x.my_words = (uint32_t) bm_words(fv.ivnum);
      x.seg_stride = seg_stride;
      x.seg_gens = seg_gens;
      x.cta_fence = (getenv("GL_XSYNC_CTA_FENCE") && atoi(getenv("GL_XSYNC_CTA_FENCE"))) ? 1 : 0;
      if (global_front) {
        a.pa.col = gcol;
        a.pa.hub_nbr = hub_nbr_g;
        a.pa.fid_offset = fv.fid_offset;
        a.pa.id_mask = fv.id_mask;
        a.pa.hub_dummy = fv.fid << fv.fid_offset;
      }
      for (int par = 0; par < 2; ++par) {
        x.slot_at_peer[par] = mm.d_peer_slot[par];
        x.send_slot[par] = mm.d_send_slot[par];
        x.recv_slot[par] = mm.d_recv_slot[par];
        x.peer_count[par] = mm.d_peer_count[par];
        x.msend[par] = mm.d_msend[par];
        x.mrecv[par] = mm.d_mrecv[par];
      }
    }
    for (;;) {
      a.depth_base = depth_base;
      if (multi) {
        ma.f = a;
        ma.x.tag0 = comm->seq_base + 1;
        ma.x.msg_round0 = (uint32_t) mm.round;
        ma.x.mirror_seq0 = (uint32_t) mm.mirror_seq;
        void* args[] = {&ma};
        GL_CUDA(cudaLaunchCooperativeKernel(global_front ? (void*) k_bfs_fused_multi<true> : (void*) k_bfs_fused_multi<false>,
                                            dim3(fused_grid), dim3(kTB), args, 0, s));
      } else {
        void* args[] = {&a};
        GL_CUDA(cudaLaunchCooperativeKernel((void*) k_bfs_fused, dim3(fused_grid), dim3(kTB), args, 0, s));
      }
      GL_COUNT_LAUNCH();
      GL_CUDA(cudaMemcpyAsync(h_ctl, d_ctl, sizeof(BfsFusedCtl), cudaMemcpyDeviceToHost, s));
      if (!ev_done) GL_CUDA(cudaEventCreate(&ev_done));
      GL_CUDA(cudaEventRecord(ev_done, s));   // the query's last device operation (overwritten by a relaunch after a spill)
      GL_CUDA(cudaStreamSynchronize(s));
      if (multi) {
        comm->seq_base = h_ctl->x_last_tag;
        mm.round += (int) h_ctl->x_msg_rounds;
        mm.mirror_seq += h_ctl->x_mirror_syncs;
        if (h_ctl->x_error) {
          set_error(h_ctl->x_error == 2 ? "fused BFS: landing slot overflow"
                                        : "fused BFS: a peer GPU did not reach the in-kernel barrier in time");
          return GL_ERR_COMM;
        }
      }
      if (!h_ctl->overflow) break;
      // deeper than the ring: spill and resume (high-diameter graphs)
      // A launch that parks right after a pull level leaves that level's shipment unconsumed in its
      // frontier generation.  Within THIS query the stale bits are harmless (every neighbour of an
      // already expanded frontier vertex is visited), but they must not survive into another query
      // on this communicator: the next Init re-zeroes the segments (collective; all ranks spill at
      // the same depth, so all of them set the flag).
      if (multi && global_front) comm->mirror_dirty = true;
      GL_TRY(SpillRing());
      GL_LAUNCH(k_bfs_resume_prep, 1, 32, s, d_ctl);
    }
    if (multi) mm.bytes_sent += h_ctl->x_items * sizeof(ItemU32);
    if (multi && getenv("GL_KTIME"))   // (not under GL_TRACE: its per-launch synchronisation distorts the gaps)
      fprintf(stderr, "[gl-ktime] f%u seed end -> first instruction %.1f us, kernel %.1f us, levels %u\n", fv.fid,
              (double) (h_ctl->t_kstart - h_ctl->t_begin) * 1e-3, (double) (h_ctl->t_kend - h_ctl->t_kstart) * 1e-3, h_ctl->levels);
    if (!multi && getenv("GL_KTIME") && h_ctl->levels && h_ctl->levels <= (uint32_t) kMaxFusedStats) {
      // one fragment: t_begin is the kernel's first instruction; what the query's events add around
      // the kernel is the launch and the epilogue (control block copy, end event)
      float ev_ms = 0.f;
      GL_CUDA(cudaEventElapsedTime(&ev_ms, rec.ev[0], ev_done));
      const unsigned long long t_last = h_ctl->stat[h_ctl->levels - 1].t_ns;
      fprintf(stderr, "[gl-ktime] first instruction -> last level %.1f us, last level -> kernel end %.1f us, "
              "events - kernel %.1f us, levels %u\n", (double) (t_last - h_ctl->t_begin) * 1e-3,
              (double) (h_ctl->t_kend - t_last) * 1e-3, ev_ms * 1e3 - (double) (h_ctl->t_kend - h_ctl->t_begin) * 1e-3,
              h_ctl->levels);
    }
    if (multi && trace_on()) {
      for (uint32_t l = 0; l < h_ctl->levels && l < 32; ++l) {
        const unsigned long long* t = h_ctl->ph[l];
        char line[256];
        int o = snprintf(line, sizeof(line), "[gl-trace] f%u level %2u mode %u:", fv.fid, l, h_ctl->stat[l].mode);
        for (int k = 1; k < 6; ++k)
          o += snprintf(line + o, sizeof(line) - o, " %7.1f", t[k] > t[0] ? (double) (t[k] - t[0]) * 1e-3 : -1.0);
        snprintf(line + o, sizeof(line) - o, " us | peer-wait %.1f gs1 %.1f\n", h_ctl->xw[l][0] * 1e-3, h_ctl->xw[l][1] * 1e-3);
        fputs(line, stderr);
      }
      fprintf(stderr, "[gl-trace] last xsync: gs1 %.1f  pre %.1f  wait %.1f  gs2 %.1f us\n",
              (h_ctl->xt[1] - h_ctl->xt[0]) * 1e-3, (h_ctl->xt[2] - h_ctl->xt[1]) * 1e-3,
              (h_ctl->xt[3] - h_ctl->xt[2]) * 1e-3, (h_ctl->xt[4] - h_ctl->xt[3]) * 1e-3);
    }
    used_lv = h_ctl->levels - depth_base + 1;
    q_touched += h_ctl->touched;
    for (uint32_t i = 0; i < h_ctl->levels && i < (uint32_t) kMaxFusedStats; ++i)
      note_step(h_ctl->stat[i].scanned, h_ctl->stat[i].frontier, (int) h_ctl->stat[i].mode);
    // a query deeper than the level table still reports all of its work
    q_entries += h_ctl->over_scanned;
    q_frontier += h_ctl->over_frontier;
    // every GPU left the kernel on the same all-reduced "frontier is empty": no round vote needed
    mm.decided_terminate = true;
    query_end = ev_done;
    return GL_OK;
  }

  // per-level device timestamps -> ms/superstep of the fused run
  void FillStats(gl_query_stats* st) override {
    if (!fused() || !h_ctl) return;
    st->supersteps = (int) h_ctl->levels + 1;
    int n = (int) std::min<uint32_t>(h_ctl->levels, (uint32_t) kMaxFusedStats) + 1;
    st->n_steps = n;
    unsigned long long prev = h_ctl->t_begin;
    // PEval (seed) is part of the launch prologue.  One fragment: t_begin is the fused kernel's first
    // instruction, so level 0 does not include the launch; several: the seed kernel's end.
    st->step_ms[0] = 0.f;
    for (int i = 1; i < n; ++i) {
      const BfsLevelStat& ls = h_ctl->stat[i - 1];
      st->step_ms[i] = (float) ((double) (ls.t_ns - prev) * 1e-6);
      st->step_entries[i] = ls.scanned;
      st->step_frontier[i] = ls.frontier;
      st->step_mode[i] = (uint8_t) ls.mode;
      prev = ls.t_ns;
    }
  }

  int PEval() override {
    if (fused()) return RunFused();
    uint32_t src;
    if (has_src_) {
      src = src_;
      GL_LAUNCH(k_bfs_seed, 1, 32, eng.stream, src, level_bm(0), vis);
      uint64_t rp2[2];
      GL_CUDA(cudaMemcpyAsync(rp2, g_rp + src, sizeof(rp2), cudaMemcpyDeviceToHost, eng.stream));
      GL_CUDA(cudaStreamSynchronize(eng.stream));
      n_f = 1;
      m_f = rp2[1] - rp2[0];
    }
    if (fv.fnum > 1) {
      mm.stat_in[0] = (long long) n_f;
      mm.stat_in[1] = (long long) m_f;
      pending_stats = true;
    } else {
      visited_edges = m_f;
    }
    used_lv = 1;
    mm.ForceContinue();
    return GL_OK;
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    if (curr_depth - depth_base + 1 >= max_lv) GL_TRY(SpillRing());
    uint32_t* cur = level_bm(curr_depth - depth_base);
    uint32_t* nxt = level_bm(curr_depth - depth_base + 1);
    GL_TRY(eng.reset_ctrl());
    const bool multi = fv.fnum > 1;
    if (multi) {
      // ParallelProcess (bfs.h:158-166): received vertices join the current level
      MsgView mv = mm.view();
      BfsApply ap{cur, vis, g_rp};
      GL_LAUNCH((k_unpack<ItemU32, BfsApply>), eng.sm_count * 4, kTB, s, mv, ap, eng.ctrl);
      GL_TRY(eng.reset_ctrl());
      GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
    }
    // Direction choice on WHOLE-GRAPH statistics (identical on every fragment,
    // because the pull step is collective: it starts with a mirror sync).
    // n_f / m_f / visited_edges are global sums carried by the round vote.
    // (the tail rule needs the unvisited count, which only one fragment keeps)
    const uint32_t prev_phase = phase;
    const uint64_t m_u = g_m_total > visited_edges ? g_m_total - visited_edges : 0;
    const uint64_t unvis = nz_total > visited_cnt ? nz_total - visited_cnt : 0;
    phase = bfs_next_phase(phase, n_f, m_f, m_u, g_vnum, can_pull() ? 1 : 0, beta(), unvis,
                           multi ? kNoTail : kTailPerFrontier);
    const bool use_pull = phase == 1;
    EdgeRange er{g_rp, g_col, nullptr};
    if (!use_pull) {
      // leaving the pull phase: outer copies learn which vertices their owners
      // visited meanwhile, so the push phase does not re-report them
      if (multi && prev_phase == 1) GL_TRY(mm.SyncBitsToGhosts(s, vis));
      OpBfsPush op{vis, nxt, remote, g_rp, fv.ivnum};
      GL_TRY(run_frontier_scan(eng, cur, fv.ivnum, er, op));
      if (multi) {
        MsgView mv = mm.view();
        GL_LAUNCH((k_pack_outer<ItemU32, BfsPayload>), eng.sm_count * 4, kTB, s, remote,
                  fv.ivnum, fv.ovnum, fv.ovgid, mv, BfsPayload(), 0, nullptr);
      }
    } else {
      // pull: refresh the frontier bits of the outer copies from their owners
      // (dense mirror sync over NVLink), then every unvisited inner vertex
      // scans its whole row locally: no per-vertex messages in this phase
      if (multi) GL_TRY(mm.SyncBitsToGhosts(s, cur));
      static thread_local int gp = 0;
      if (!gp) gp = persistent_grid(k_bfs_pull, eng.sm_count);
      GL_LAUNCH(k_bfs_pull, gp, kTB, s, pull_args(), cur, vis, nxt, eng.ctrl);
    }
    step_pull = use_pull;
    if (multi) {
      // the round vote reads the device counters and mirrors them to the host:
      // one host synchronisation per superstep (inside FinishARound)
      mm.vote_ctrl = eng.ctrl;
      mm.vote_h_ctrl = eng.h_ctrl;
      pending_stats = true;
    } else {
      GL_TRY(eng.fetch_ctrl());
      const ScanCtrl& c = *eng.h_ctrl;
      note_step(c.scanned, (uint32_t) std::min<uint64_t>(n_f, 0xFFFFFFFFu), use_pull ? 1 : 0);
      q_touched += c.touched;
      if (c.next_count > 0) mm.ForceContinue();
      n_f = c.next_count;
      m_f = c.next_edges;
      visited_edges += c.next_edges;
      visited_cnt += c.next_count;
    }
    ++curr_depth;
    used_lv = curr_depth - depth_base + 1;
    return GL_OK;
  }

  // called by the worker after FinishARound
  void AfterRound() override {
    if (!pending_stats) return;
    pending_stats = false;
    if (rounds_noted) {
      const ScanCtrl& c = *eng.h_ctrl;   // mirrored by the vote kernel
      // this fragment's share of a push level is what its scan expanded; a pull step has no such
      // count and reports the whole graph's level
      note_step(c.scanned, (uint32_t) std::min<uint64_t>(step_pull ? n_f : c.frontier, 0xFFFFFFFFu), step_pull ? 1 : 0);
      q_touched += c.touched;
    }
    rounds_noted = true;
    n_f = (uint64_t) mm.stat_out[0];
    m_f = (uint64_t) mm.stat_out[1];
    visited_edges += m_f;
  }
  bool pending_stats = false;
  bool step_pull = false;
  bool rounds_noted = false;   // PEval's vote carries no engine counters

  // compact result path: u8 depths, chunked D2H into pinned staging, widened to
  // the reference's int64 (bfs_context.h:31 depth_type) by host threads while the
  // next chunk is still crossing PCIe
  cudaEvent_t ev_done = nullptr;
  DevBuf<uint8_t> deg8, d_out8;
  PinnedBuf<uint8_t> h_out8;
  cudaEvent_t ev8[8] = {};
  int ResultCompact(int64_t* host_out, uint32_t nl) {
    cudaStream_t s = eng.stream;
    const uint32_t n = fv.ivnum;
    if (!d_out8) {
      GL_CUDA(d_out8.alloc(n));
      GL_CUDA(h_out8.alloc(n));
      for (auto& e : ev8) GL_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    GL_LAUNCH(k_depth_u8_from_levels, (n + 255) / 256, 256, s, lv, (uint32_t) words, nl, n, perm, d_out8);
    const uint32_t nchunks = n >= (1u << 20) ? 8 : 1;
    const uint32_t per = ((n + nchunks - 1) / nchunks + 63) & ~63u;
    for (uint32_t c = 0; c < nchunks; ++c) {
      const uint32_t b = std::min(n, c * per), e = std::min(n, b + per);
      if (e > b) GL_CUDA(cudaMemcpyAsync(h_out8 + b, d_out8 + b, e - b, cudaMemcpyDeviceToHost, s));
      GL_CUDA(cudaEventRecord(ev8[c], s));
    }
    // host threads widen chunk c while chunk c+1 is still crossing PCIe (host_pool.h)
    uint32_t bounds[9];
    for (uint32_t c = 0; c <= nchunks; ++c) bounds[c] = std::min(n, c * per);
    cudaError_t err = cudaSuccess;
    WidenPool::instance().widen_u8_to_i64(h_out8, host_out, bounds, nchunks, [&](uint32_t c) {
      cudaError_t e1 = cudaEventSynchronize(ev8[c]);
      if (e1 != cudaSuccess) err = e1;
    });
    _mm_sfence();
    GL_CUDA(err);
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    uint32_t nl = std::min<uint32_t>(max_lv, used_lv + 1);
    // The byte-wide result pays when this process has the host to itself (1.6-2.3 ms vs 2.9 ms); with
    // several rank processes on one host the widening threads of all ranks compete for the same memory
    // system and the plain int64 copy was measured to be as fast and far more stable (N = 2: 3.2 ms
    // vs 2.8-6.7 ms) -- GL_RESULT_COMPACT=1/0 overrides the choice.
    static const bool compact_ok = [] {
      if (const char* e = getenv("GL_RESULT_COMPACT")) return atoi(e) != 0;
      const char* lw = getenv("LOCAL_WORLD_SIZE");
      return !(lw && atoi(lw) > 1);
    }();
    if (compact_ok && !spilled && depth_base == 0 && nl <= 254 && cfg.reserved[6] == 0)
      return ResultCompact((int64_t*) host_out, nl);
    GL_LAUNCH(k_depth_from_levels, (fv.ivnum + 255) / 256, 256, eng.stream, lv, (uint32_t) words, nl, fv.ivnum, perm,
              depth_base, spilled ? spill.get() : nullptr, out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(int64_t) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_bfs() { return new BfsApp; }

}  // namespace gl
