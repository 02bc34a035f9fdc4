// apps_common.cuh — launch helpers and small kernels shared by the apps.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdlib>

#include "app_base.h"

namespace gl {

// persistent-grid size for a kernel: SMs x resident CTAs (queried once)
template <typename K>
int persistent_grid(K kernel, int sm_count, int threads = kTB) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  return per_sm * sm_count;
}

// GL_TRACE=1 in the environment: synchronise after every launch and print its
// wall time (debugging aid; never enabled in measurements)
inline bool trace_on() {
  static int on = -1;
  if (on < 0) on = getenv("GL_TRACE") ? 1 : 0;
  return on == 1;
}
#define GL_LAUNCH(kernel, grid, block, stream, ...)                                   \
  do {                                                                                \
    if (::gl::trace_on()) {                                                           \
      cudaStreamSynchronize(stream);                                                  \
      auto t0__ = std::chrono::steady_clock::now();                                   \
      kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__);                          \
      cudaStreamSynchronize(stream);                                                  \
      fprintf(stderr, "[gl-trace] %-60s %8.1f us\n", #kernel,                         \
              std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0__).count()); \
    } else {                                                                          \
      kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__);                          \
    }                                                                                 \
    GL_COUNT_LAUNCH();                                                                \
    GL_CUDA(cudaGetLastError());                                                      \
  } while (0)

// Runs one frontier-driven edge scan (tile kernel + hub kernel) on `er`.
template <class Op>
int run_frontier_scan(Engine& eng, const uint32_t* frontier, uint32_t nverts,
                      EdgeRange er, const Op& op) {
  static thread_local int g1 = 0, g2 = 0;
  if (!g1) g1 = persistent_grid(k_frontier_scan<Op>, eng.sm_count);
  if (!g2) g2 = persistent_grid(k_hub_scan<Op>, eng.sm_count);
  uint32_t ntiles = (nverts + kTileV - 1) / kTileV;
  int grid1 = (int) std::min<uint32_t>((uint32_t) g1, std::max<uint32_t>(ntiles, 1));
  GL_LAUNCH(k_frontier_scan<Op>, grid1, kTB, eng.stream, frontier, nverts, er,
            op, eng.ctrl, eng.hubs, eng.hub_cap, eng.hub_deg);
  // GL_HUB_TMA=0 selects the plain-load hub phase (A/B)
  static const bool tma = op_tma_ok<Op>::value && !(getenv("GL_HUB_TMA") && atoi(getenv("GL_HUB_TMA")) == 0);
  if (tma) {
    static thread_local int g3 = 0;
    if (!g3) g3 = persistent_grid(k_hub_scan_tma<Op>, eng.sm_count);
    GL_LAUNCH(k_hub_scan_tma<Op>, g3, kTB, eng.stream, er, op, eng.ctrl, eng.hubs, eng.hub_cap);
  } else {
    GL_LAUNCH(k_hub_scan<Op>, g2, kTB, eng.stream, er, op, eng.ctrl, eng.hubs, eng.hub_cap);
  }
  return GL_OK;
}

#ifdef __CUDACC__
// owner fragment of an outer vertex from its gid
GL_DEV uint32_t gid_fid(uint32_t gid, int fid_offset) { return gid >> fid_offset; }

// Generic producer: for every set bit v in `remote` over the outer range
// [ivnum, tvnum) send Item{lid_at_owner, payload(v)} to the owner.
// Replaces the "ForEach over outer vertices + SyncStateOnOuterVertexWarpOpt"
// idiom (e.g. cuda/sssp/sssp.h:295-304).
//
// A CTA takes 256 words (8192 outer copies) per step.  Outer copies are grouped
// by owner, so a word almost always belongs to ONE owner: every thread adds its
// word's popcount to a shared per-owner counter, ONE thread per owner reserves
// the CTA's share of the landing slot with a single global atomic, and the
// threads then write their items behind that base.  (Reserving per warp hit the
// same global counter ~10^5 times per round: 118 us for 370 K items.)  The few
// words that straddle an owner boundary reserve per item.
struct PackSmem {
  uint32_t cnt[GL_MAX_FNUM];
  uint32_t base[GL_MAX_FNUM];
};

// Returns whether THIS thread stored anything into a peer's landing slot.
template <typename Item, class Payload>
GL_DEV bool pack_outer_phase(PackSmem& ps, uint32_t* remote, uint32_t ivnum, uint32_t ovnum,
                             const uint32_t* __restrict__ ovgid, const MsgView& mv, const Payload& pay,
                             bool clear_bits) {
  const uint32_t w_lo = ivnum >> 5;
  const uint32_t w_hi = (ivnum + ovnum + 31) >> 5;          // exclusive
  const uint32_t nwords = w_hi > w_lo ? w_hi - w_lo : 0;
  const uint32_t nchunks = (nwords + blockDim.x - 1) / blockDim.x;
  bool wrote = false;
  for (uint32_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    if (threadIdx.x < mv.fnum) ps.cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t wi = w_lo + chunk * blockDim.x + threadIdx.x;
    uint32_t word = wi < w_hi ? remote[wi] : 0u;
    if (word && clear_bits) remote[wi] = 0;
    // bits outside [ivnum, ivnum + ovnum) belong to inner vertices / padding
    if (word) {
      const uint32_t v0 = wi << 5;
      if (v0 < ivnum) word &= ~((1u << (ivnum - v0)) - 1u);
      const uint32_t end = ivnum + ovnum;
      if (v0 + 32 > end) word &= (end > v0) ? ((end - v0 >= 32) ? 0xFFFFFFFFu : ((1u << (end - v0)) - 1u)) : 0u;
    }
    uint32_t dst = 0, off = 0;
    bool single = false;
    wrote |= word != 0;
    if (word) {
      const uint32_t vf = (wi << 5) + (__ffs(word) - 1), vl = (wi << 5) + (31 - __clz(word));
      const uint32_t d0 = ovgid[vf - ivnum] >> mv.fid_offset, d1 = ovgid[vl - ivnum] >> mv.fid_offset;
      if (d0 == d1) {
        single = true;
        dst = d0;
        off = atomicAdd(&ps.cnt[d0], (uint32_t) __popc(word));
      } else {
        // owner boundary inside the word (at most fnum-1 such words per fragment)
        uint32_t r = word;
        while (r) {
          const uint32_t v = (wi << 5) + (__ffs(r) - 1);
          r &= r - 1;
          const uint32_t gid = ovgid[v - ivnum];
          const uint32_t d = gid >> mv.fid_offset;
          const uint32_t pos = atomicAdd(mv.send_count + d, 1u);
          if (pos < mv.capacity) ((Item*) mv.send_slot[d])[pos] = pay(v, gid & mv.id_mask);
        }
      }
    }
    __syncthreads();
    if (threadIdx.x < mv.fnum && ps.cnt[threadIdx.x])
      ps.base[threadIdx.x] = atomicAdd(mv.send_count + threadIdx.x, ps.cnt[threadIdx.x]);
    __syncthreads();
    if (single) {
      uint32_t pos = ps.base[dst] + off;
      Item* out = (Item*) mv.send_slot[dst];
      uint32_t r = word;
      while (r) {
        const uint32_t v = (wi << 5) + (__ffs(r) - 1);
        r &= r - 1;
        if (pos < mv.capacity) out[pos] = pay(v, ovgid[v - ivnum] & mv.id_mask);
        ++pos;
      }
    }
    __syncthreads();   // ps.cnt / ps.base are reused by the next chunk
  }
  return wrote;
}

template <typename Item, class Payload>
__global__ void __launch_bounds__(kTB)
k_pack_outer(const uint32_t* __restrict__ remote, uint32_t ivnum, uint32_t ovnum,
             const uint32_t* __restrict__ ovgid, MsgView mv, Payload pay,
             int clear_bits, uint32_t* remote_rw) {
  __shared__ PackSmem ps;
  pack_outer_phase<Item, Payload>(ps, clear_bits ? remote_rw : const_cast<uint32_t*>(remote), ivnum, ovnum,
                                  ovgid, mv, pay, clear_bits != 0);
}

// Generic consumer: apply every received item (ParallelProcess,
// gpu_message_manager.h:362-393 + message_kernels.h:28-127).
template <typename Item, class Apply>
__global__ void __launch_bounds__(kTB)
k_unpack(MsgView mv, Apply apply, ScanCtrl* ctrl) {
  ScanAcc acc;
  for (uint32_t src = 0; src < mv.fnum; ++src) {
    if (src == mv.fid) continue;
    uint32_t n = mv.recv_count[src];
    if (n > mv.capacity) n = mv.capacity;   // an overflowing producer dropped the rest (FinishARound reports it)
    const Item* items = (const Item*) mv.recv_slot[src];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += gridDim.x * blockDim.x)
      apply(items[i], acc);
  }
  flush_acc(acc, ctrl);
}

// lid -> gid of the fragment's vertices (inner: fid << fid_offset | lid; outer: ovgid)
struct GidOf {
  uint32_t ivnum, fid;
  int fid_offset;
  const uint32_t* ovgid;
  GL_DEV uint32_t operator()(uint32_t x) const {
    return x < ivnum ? ((fid << fid_offset) | x) : ovgid[x - ivnum];
  }
};

// deg[v] = CSR row length of the inner vertex v (a template so that every app's unit may hold it)
template <typename T>
__global__ void k_row_length(const uint64_t* __restrict__ rp, uint32_t ivnum, T* deg) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < ivnum) deg[v] = (T) (rp[v + 1] - rp[v]);
}
#endif

// gid-valued label -> oid (WCC / CDLP outputs).  Without a vertex map the
// mapping is exact only for this library's contiguous-block partition.
struct LabelMap {
  int fid_offset;
  uint32_t id_mask, fnum;
  uint64_t chunk;
  const int64_t* inner_oids;
  int64_t oid_base;
  const int64_t* vm_l2o;    // device vertex map (gl_vm_*), or null
  const uint64_t* vm_off;
#ifdef __CUDACC__
  GL_DEV int64_t oid(uint32_t g) const {
    const uint32_t f = g >> fid_offset, l = g & id_mask;
    if (vm_l2o) return vm_l2o[vm_off[f] + l];
    if (fnum == 1) return inner_oids ? inner_oids[l] : oid_base + (int64_t) l;
    if (chunk && !inner_oids) return (int64_t) ((uint64_t) f * chunk + l);   // oid == global index
    return (int64_t) g;   // explicit oids, several fragments, no vertex map attached: raw gid
  }
#endif
};

LabelMap label_map(const gl_app& a);   // worker.cu

struct ItemU32 {
  uint32_t lid;
};
struct ItemU32U32 {
  uint32_t lid, val;
};
struct ItemU32F32 {
  uint32_t lid;
  float val;
};
struct ItemU32F64 {
  uint32_t lid, pad;
  double val;
};
struct ItemU32I64 {
  uint32_t lid, pad;
  int64_t val;
};

inline size_t bm_words(uint64_t bits) { return (size_t) ((bits + 31) / 32); }

}  // namespace gl
