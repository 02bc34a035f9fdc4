// app_core.cu — core decomposition and k-core on an undirected graph.
//
// Behaviour follows examples/analytical_apps/core_decomposition/core_decomposition.h
// and kcore/kcore.h (CPU apps, LoadStrategy::kOnlyOut).  A vertex's count starts
// at its row length (CSR entries: a multi-edge counts once per copy, a self loop
// twice).
//  * Core decomposition: at level L every unpeeled vertex whose count is <= L is
//    peeled with core L, and the entries of its row lower the counts of their
//    unpeeled endpoints, until no count crosses L; then the next level.  Isolated
//    vertices get core 0.  Result: int64 core number per inner vertex.
//  * k-core: the same peel, once, at L = k - 1, but every entry of a peeled row
//    is counted down (already peeled endpoints and the row's own self loops too).
//    Result: int64 final count = entries whose other endpoint survives the peel;
//    the k-core is the set of vertices with count >= k.
// Both results are integers fixed by the graph: bit-exact for any fragment count.
//
// One decrement batch: the c lanes of a warp whose entries point at the same u
// are combined (__match_any_sync), old = atomicSub(&cnt[u], c), and u is peeled
// when old > L && old - c <= L -- true for exactly one batch.
//
//  * One fragment: the whole query is ONE cooperative launch (k_core_fused).
//    Levels jump straight to max(L + 1, min count of the remaining vertices) (a
//    grid min) instead of stepping through every integer up to the largest core
//    (~2000 on R-MAT-22, of which ~260 are non-empty), and the sub-rounds of a
//    level (hundreds of them on R-MAT, most with < 1024 vertices) are separated
//    by grid.sync() instead of host round trips.  The remaining vertices are
//    kept in a list that is compacted whenever it has shrunk by half.
//  * Several fragments: one sub-round per superstep through the worker loop.
//    Counts owed to outer copies travel to their owners as (lid, count) items;
//    when no fragment has a frontier or a message in flight, an all-reduce (min)
//    picks the next level (core_decomposition.h:166-205 votes with Sum).
#include <cooperative_groups.h>

#include "apps_common.cuh"

namespace gl {
namespace {

namespace cg = cooperative_groups;

constexpr uint32_t kCoreUnset = 0xFFFFFFFFu;
#define GL_CORE_FUSED_CTAS 4

GL_DEV unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
GL_DEV bool bit_test_cg(const uint32_t* bm, uint32_t v) { return (__ldcg(bm + (v >> 5)) >> (v & 31)) & 1u; }

// append v to q among the currently active lanes (one atomic per warp)
GL_DEV void append_active(uint32_t* q, unsigned int* n, uint32_t v) {
  const uint32_t m = __activemask();
  const uint32_t leader = __ffs(m) - 1;
  uint32_t base = 0;
  if (lane_id() == leader) base = atomicAdd(n, (unsigned int) __popc(m));
  base = __shfl_sync(m, base, leader);
  q[base + __popc(m & ((1u << lane_id()) - 1))] = v;
}

// State at the start of a query for inner vertex v: count = row length; an
// isolated vertex has core 0 and is peeled.  Returns the row length.
template <bool kCore>
GL_DEV int core_init_vertex(uint32_t v, const uint64_t* rp, int32_t* cnt, uint32_t* core, uint32_t* peeled) {
  const int d = (int) (rp[v + 1] - rp[v]);
  cnt[v] = d;
  if (kCore) {
    core[v] = d == 0 ? 0u : kCoreUnset;
    if (d == 0) bit_set_atomic(peeled, v);
  }
  return d;
}

// The peel's edge operator.  kQueue: crossings are appended to a queue (one
// fragment); otherwise they set a bit of the next frontier, and entries to
// outer copies accumulate in ocnt for their owners.
template <bool kCore, bool kQueue>
struct OpPeel {
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  int32_t* cnt;
  uint32_t* core;
  uint32_t* peeled;
  uint32_t* out;        // kQueue: the next queue; else: the next frontier bitmap
  unsigned int* out_n;  // kQueue: its length
  uint32_t* ocnt;       // several fragments: entries owed to outer vertex ivnum + i
  uint32_t* remote;     // several fragments: outer vertices with a count to ship
  uint32_t ivnum;
  int L;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  GL_DEV void edge(uint32_t, Meta, uint32_t v, W, ScanAcc& acc) const {
    // core decomposition ignores peeled endpoints (this covers the row's own self loops);
    // k-core's result is the final count, so every entry is counted down
    if (kCore && bit_test(peeled, v)) return;
    const uint32_t peers = __match_any_sync(__activemask(), v);
    if (lane_id() != (uint32_t) __ffs(peers) - 1) return;
    const int c = __popc(peers);
    if (!kQueue && v >= ivnum) {
      atomicAdd(ocnt + (v - ivnum), (uint32_t) c);
      if (bit_set_atomic(remote, v)) acc.remote++;
      return;
    }
    const int old = atomicSub(cnt + v, c);
    acc.touched++;
    if (old > L && old - c <= L) {
      if (kCore) {
        core[v] = (uint32_t) L;
        bit_set_atomic(peeled, v);
      }
      if (kQueue) append_active(out, out_n, v);
      else bit_set_atomic(out, v);
      acc.next_count++;
    }
  }
};

// ---------------------------------------------------------------------------
// One fragment: the whole query in one cooperative launch.
// ---------------------------------------------------------------------------
// Counters of one step.  Step t uses c[t % 3]; what it appends (qn, list_n) is
// read during step t + 1; thread 0 zeroes c[(t + 2) % 3] after the grid.sync
// that ends step t, one grid.sync before step t + 2 uses it.
struct CoreStep {
  ScanCtrl sc;
  unsigned int qn;       // vertices appended to the queue step t + 1 scans
  unsigned int list_n;   // survivors written by a list compaction
  unsigned int min_key;  // max of ~count over the remaining vertices (0: none remain)
  unsigned int pad;
};
struct CoreFusedCtl {
  CoreStep c[3];
  unsigned long long subrounds, levels, peeled, scanned, touched;
  unsigned long long level_ns, subround_ns;   // thread 0's device time in level steps / sub-rounds
};

struct CoreFusedArgs {
  EdgeRange er;
  uint32_t n;
  int L0;   // k-core: k - 1
  int32_t* cnt;
  uint32_t* core;
  uint32_t* peeled;
  uint32_t* queue[2];
  uint32_t* list[2];
  CoreFusedCtl* ctl;
  HubItem* hubs;
  uint32_t hub_cap, hub_deg;
};

template <bool kCore>
__global__ void __launch_bounds__(kTB, GL_CORE_FUSED_CTAS) k_core_fused(CoreFusedArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ ScanSmem<uint32_t> sm;
  __shared__ uint32_t s_item;
  CoreFusedCtl* ctl = a.ctl;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nthr = gridDim.x * blockDim.x;
  int L = kCore ? -1 : a.L0;
  uint32_t t = 0;
  auto end_step = [&]() {
    grid.sync();
    if (gtid == 0) ctl->c[(t + 2) % 3] = CoreStep();
    ++t;
  };
  // step 0: counts; the non-isolated vertices form the remaining list (core
  // decomposition) or the vertices with count <= L are the seeds (k-core)
  for (uint32_t base = blockIdx.x * blockDim.x; base < a.n; base += nthr) {   // warp-uniform bound
    const uint32_t v = base + threadIdx.x;
    bool put = false;
    if (v < a.n) {
      const int d = core_init_vertex<kCore>(v, a.er.rp, a.cnt, a.core, a.peeled);
      put = kCore ? d > 0 : d <= L;
    }
    queue_append_warp(kCore ? a.list[0] : a.queue[0], kCore ? &ctl->c[0].list_n : &ctl->c[0].qn, put, v);
  }
  uint32_t list_n = 0, remaining = 0, lsel = 0;
  end_step();
  if (kCore) list_n = remaining = ((volatile CoreStep*) &ctl->c[0])->list_n;
  for (;;) {
    if (kCore) {
      // level step: grid min of the remaining counts (compacting the list when it has halved), then
      // the seeds of level L = max(L + 1, min)
      const unsigned long long t0 = gtid == 0 ? global_ns() : 0;
      CoreStep* C = &ctl->c[t % 3];
      const bool compact = 2ull * remaining <= list_n;
      const uint32_t* src = lsel ? a.list[1] : a.list[0];
      uint32_t* dst = lsel ? a.list[0] : a.list[1];
      uint32_t best = 0;
      for (uint32_t base = blockIdx.x * blockDim.x; base < list_n; base += nthr) {
        const uint32_t i = base + threadIdx.x;
        uint32_t v = 0;
        bool live = false;
        if (i < list_n) {
          v = src[i];
          live = !bit_test_cg(a.peeled, v);
          if (live) best = max(best, ~(uint32_t) __ldcg(a.cnt + v));
        }
        if (compact) queue_append_warp(dst, &C->list_n, live, v);
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
      if (lane_id() == 0 && best) atomicMax(&C->min_key, best);
      grid.sync();
      const uint32_t key = ((volatile CoreStep*) C)->min_key;
      if (key == 0) break;   // nothing remains
      L = max(L + 1, (int) ~key);
      if (compact) {
        lsel ^= 1;
        list_n = ((volatile CoreStep*) C)->list_n;
      }
      const uint32_t* lst = lsel ? a.list[1] : a.list[0];
      uint32_t* q = (t & 1) ? a.queue[1] : a.queue[0];
      for (uint32_t base = blockIdx.x * blockDim.x; base < list_n; base += nthr) {
        const uint32_t i = base + threadIdx.x;
        bool seed = false;
        uint32_t v = 0;
        if (i < list_n) {
          v = lst[i];
          seed = !bit_test_cg(a.peeled, v) && __ldcg(a.cnt + v) <= L;
          if (seed) {
            a.core[v] = (uint32_t) L;
            bit_set_atomic(a.peeled, v);
          }
        }
        queue_append_warp(q, &C->qn, seed, v);
      }
      end_step();
      if (gtid == 0) {
        ctl->levels++;
        ctl->level_ns += global_ns() - t0;
      }
    }
    // sub-rounds: step t scans the queue step t - 1 appended
    for (;;) {
      const uint32_t n = ((volatile CoreStep*) &ctl->c[(t + 2) % 3])->qn;
      if (n == 0) break;
      remaining -= n;
      const unsigned long long t0 = gtid == 0 ? global_ns() : 0;
      CoreStep* C = &ctl->c[t % 3];
      uint32_t* qin = (t & 1) ? a.queue[0] : a.queue[1];
      uint32_t* qout = (t & 1) ? a.queue[1] : a.queue[0];
      OpPeel<kCore, true> op{a.cnt, a.core, a.peeled, qout, &C->qn, nullptr, nullptr, a.n, L};
      ScanAcc acc;
      queue_scan_phase<OpPeel<kCore, true>>(sm, ArraySrc{qin}, n, a.er, op, &C->sc, a.hubs,
                                            a.hub_cap, a.hub_deg, acc);
      grid.sync();
      hub_scan_phase<OpPeel<kCore, true>>(&s_item, a.er, op, &C->sc, a.hubs, a.hub_cap, acc);
      flush_acc(acc, &C->sc);
      grid.sync();
      if (gtid == 0) {
        const volatile ScanCtrl* VC = &C->sc;
        ctl->subrounds++;
        ctl->peeled += n;
        ctl->scanned += VC->scanned;
        ctl->touched += VC->touched;
        ctl->c[(t + 2) % 3] = CoreStep();
        ctl->subround_ns += global_ns() - t0;
      }
      ++t;
    }
    if (!kCore) break;   // k-core: one level
  }
}

// ---------------------------------------------------------------------------
// Several fragments: one sub-round per superstep.
// ---------------------------------------------------------------------------
template <bool kCore>
__global__ void k_core_init(const uint64_t* rp, uint32_t n, int32_t* cnt, uint32_t* core, uint32_t* peeled) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) core_init_vertex<kCore>(v, rp, cnt, core, peeled);
}

// min_key = max of ~count over the unpeeled inner vertices
__global__ void k_core_min(const int32_t* cnt, const uint32_t* peeled, uint32_t n, unsigned int* min_key) {
  uint32_t best = 0;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    if (!bit_test(peeled, v)) best = max(best, ~(uint32_t) cnt[v]);
#pragma unroll
  for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane_id() == 0 && best) atomicMax(min_key, best);
}

// the seeds of level L: (unpeeled) inner vertices with count <= L
template <bool kCore>
__global__ void k_core_seed(const int32_t* cnt, uint32_t* core, uint32_t* peeled, uint32_t n, int L, uint32_t* front) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n || cnt[v] > L) return;
  if (kCore) {
    if (bit_test(peeled, v)) return;
    core[v] = (uint32_t) L;
    bit_set_atomic(peeled, v);
  }
  bit_set_atomic(front, v);
}

struct CorePayload {   // (lid at the owner, entries owed), then the count is cleared
  uint32_t* ocnt;
  uint32_t ivnum;
  GL_DEV ItemU32U32 operator()(uint32_t v, uint32_t lid) const {
    const uint32_t c = ocnt[v - ivnum];
    ocnt[v - ivnum] = 0;
    return ItemU32U32{lid, c};
  }
};
template <bool kCore>
struct CoreApply {
  int32_t* cnt;
  uint32_t* core;
  uint32_t* peeled;
  uint32_t* front;
  int L;
  GL_DEV void operator()(const ItemU32U32& it, ScanAcc& acc) const {
    const int c = (int) it.val;
    const int old = atomicSub(cnt + it.lid, c);
    if (old > L && old - c <= L) {
      if (kCore) {
        core[it.lid] = (uint32_t) L;
        bit_set_atomic(peeled, it.lid);
      }
      bit_set_atomic(front, it.lid);
      acc.aux++;
    }
  }
};

template <typename T>
__global__ void k_core_out(const T* val, uint32_t n, int64_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int64_t) val[i];
}

template <bool kCore>
struct CoreApp : gl_app {
  DevBuf<int32_t> cnt;
  DevBuf<uint32_t> core, peeled;
  DevBuf<int64_t> out64;
  // one fragment
  DevBuf<uint32_t> queue[2], list[2];
  DevBuf<CoreFusedCtl> d_ctl;
  PinnedBuf<CoreFusedCtl> h_ctl;
  cudaEvent_t ev_done = nullptr;
  int fused_grid = 0;
  // several fragments
  DevBuf<uint32_t> in_q, out_local, remote, ocnt;
  DevBuf<unsigned int> d_key;
  PinnedBuf<unsigned int> h_key;
  size_t words = 0;
  int L = -1;
  bool seeded = false;
  uint64_t pending = 0;      // inner vertices peeled by the last scan (this fragment)
  uint64_t subrounds = 0;

  ~CoreApp() override {
    if (ev_done) cudaEventDestroy(ev_done);
  }

  size_t ResultElemBytes() const override { return sizeof(int64_t); }

  int Setup() override {
    // the reference apps load kOnlyOut and are undirected-only
    if (fv.directed) {
      set_error("%s needs an undirected fragment", kCore ? "core decomposition" : "k-core");
      return GL_ERR_ARG;
    }
    const uint32_t iv = std::max<uint32_t>(fv.ivnum, 1);
    words = bm_words(fv.ivnum + fv.ovnum) + 1;
    GL_CUDA(cnt.alloc(iv));
    if (kCore) GL_CUDA(core.alloc(iv));
    GL_CUDA(peeled.alloc(words));
    GL_CUDA(out64.alloc(iv));
    if (fv.fnum == 1) {
      for (int i = 0; i < 2; ++i) {
        GL_CUDA(queue[i].alloc(iv));
        if (kCore) GL_CUDA(list[i].alloc(iv));
      }
      GL_CUDA(d_ctl.alloc(1));
      GL_CUDA(h_ctl.alloc(1));
      return GL_OK;
    }
    GL_CUDA(in_q.alloc(words));
    GL_CUDA(out_local.alloc(words));
    GL_CUDA(remote.alloc(words));
    GL_CUDA(ocnt.alloc(std::max<uint32_t>(fv.ovnum, 1)));
    GL_CUDA(d_key.alloc(1));
    GL_CUDA(h_key.alloc(1));
    return mm.Init(comm, fv, sizeof(ItemU32U32));
  }

  // k-core peels at L = k - 1 (k travels in max_round); core decomposition starts below level 0
  int first_level() const { return kCore ? -1 : (int) std::max<int64_t>((int64_t) cfg.max_round - 1, INT32_MIN); }

  int Init() override {
    cudaStream_t s = eng.stream;
    L = first_level();
    seeded = false;
    pending = 0;
    subrounds = 0;
    GL_CUDA(cudaMemsetAsync(peeled, 0, sizeof(uint32_t) * words, s));
    if (fv.fnum > 1) {
      GL_CUDA(cudaMemsetAsync(in_q, 0, sizeof(uint32_t) * words, s));
      GL_CUDA(cudaMemsetAsync(out_local, 0, sizeof(uint32_t) * words, s));
      GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
      GL_CUDA(cudaMemsetAsync(ocnt, 0, sizeof(uint32_t) * std::max<uint32_t>(fv.ovnum, 1), s));
    }
    return GL_OK;
  }

  int PEval() override {
    cudaStream_t s = eng.stream;
    if (fv.fnum > 1) {
      if (fv.ivnum)
        GL_LAUNCH(k_core_init<kCore>, (fv.ivnum + 255) / 256, 256, s, fv.oe_rp, fv.ivnum, cnt, core, peeled);
      mm.ForceContinue();   // the first IncEval seeds the first level
      return GL_OK;
    }
    GL_CUDA(cudaMemsetAsync(d_ctl, 0, sizeof(CoreFusedCtl), s));
    CoreFusedArgs a;
    a.er = EdgeRange{fv.oe_rp, fv.oe_col, nullptr};
    a.n = fv.ivnum;
    a.L0 = L;
    a.cnt = cnt;
    a.core = core;
    a.peeled = peeled;
    for (int i = 0; i < 2; ++i) {
      a.queue[i] = queue[i];
      a.list[i] = list[i];
    }
    a.ctl = d_ctl;
    a.hubs = eng.hubs;
    a.hub_cap = eng.hub_cap;
    a.hub_deg = eng.hub_deg;
    if (!fused_grid) fused_grid = persistent_grid(k_core_fused<kCore>, eng.sm_count);
    void* args[] = {&a};
    GL_CUDA(cudaLaunchCooperativeKernel((void*) k_core_fused<kCore>, dim3(fused_grid), dim3(kTB), args, 0, s));
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaMemcpyAsync(h_ctl, d_ctl, sizeof(CoreFusedCtl), cudaMemcpyDeviceToHost, s));
    if (!ev_done) GL_CUDA(cudaEventCreate(&ev_done));
    GL_CUDA(cudaEventRecord(ev_done, s));   // the query's last device operation
    GL_CUDA(cudaStreamSynchronize(s));
    subrounds = h_ctl->subrounds;
    if (getenv("GL_KTIME"))
      fprintf(stderr, "[gl-ktime] %s: %llu level steps %.3f ms, %llu sub-rounds %.3f ms (thread 0, device timer)\n",
              kCore ? "core_decomposition" : "kcore", h_ctl->levels, h_ctl->level_ns * 1e-6, h_ctl->subrounds,
              h_ctl->subround_ns * 1e-6);
    note_step(h_ctl->scanned, (uint32_t) std::min<uint64_t>(h_ctl->peeled, 0xFFFFFFFFu), 0);
    q_touched += h_ctl->touched;
    query_end = ev_done;
    return GL_OK;   // no ForceContinue: the query ends with this round
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    // apply the counts received for this fragment's vertices, then vote on the level
    GL_TRY(eng.reset_ctrl());
    GL_LAUNCH((k_unpack<ItemU32U32, CoreApply<kCore>>), eng.sm_count * 4, kTB, s, mm.view(),
              CoreApply<kCore>{cnt, core, peeled, in_q, L}, eng.ctrl);
    GL_CUDA(cudaMemsetAsync(d_key, 0, sizeof(unsigned int), s));
    if (kCore && fv.ivnum)
      GL_LAUNCH(k_core_min, std::min<uint32_t>((fv.ivnum + 255) / 256, eng.sm_count * 8), 256, s, cnt, peeled,
                fv.ivnum, d_key);
    GL_CUDA(cudaMemcpyAsync(h_key, d_key, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    GL_TRY(eng.fetch_ctrl());
    // [0] -1 while some fragment has a frontier; [1] the smallest remaining count
    int64_t vote[2] = {(pending + eng.h_ctrl->aux) ? -1 : 0, *h_key ? (int64_t) (uint32_t) ~*h_key : INT64_MAX};
    GL_TRY(mm.AllReduceI64(vote, 2, 1));
    if (vote[0] == 0) {
      // no frontier and no message anywhere: the level is finished
      if (kCore ? vote[1] == INT64_MAX : seeded) return GL_OK;   // the peel is over: nothing sent, no vote to continue
      if (kCore) L = std::max<int>(L + 1, (int) vote[1]);
      seeded = true;
      if (fv.ivnum)
        GL_LAUNCH(k_core_seed<kCore>, (fv.ivnum + 255) / 256, 256, s, cnt, core, peeled, fv.ivnum, L, in_q);
    }
    GL_TRY(eng.reset_ctrl());
    OpPeel<kCore, false> op{cnt, core, peeled, out_local, nullptr, ocnt, remote, fv.ivnum, L};
    GL_TRY(run_frontier_scan(eng, in_q, fv.ivnum, EdgeRange{fv.oe_rp, fv.oe_col, nullptr}, op));
    GL_LAUNCH((k_pack_outer<ItemU32U32, CorePayload>), eng.sm_count * 4, kTB, s, remote, fv.ivnum, fv.ovnum,
              fv.ovgid, mm.view(), CorePayload{ocnt, fv.ivnum}, 1, remote);
    GL_CUDA(cudaMemsetAsync(in_q, 0, sizeof(uint32_t) * words, s));
    GL_TRY(eng.fetch_ctrl());
    const ScanCtrl& c = *eng.h_ctrl;
    note_step(c.scanned, (uint32_t) std::min<uint64_t>(c.frontier, 0xFFFFFFFFu), 0);
    q_touched += c.touched;
    pending = c.next_count;
    ++subrounds;
    std::swap(out_local, in_q);
    mm.ForceContinue();
    return GL_OK;
  }

  void FillStats(gl_query_stats* st) override { st->supersteps = (int) subrounds; }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    if (kCore) GL_LAUNCH(k_core_out<uint32_t>, (fv.ivnum + 255) / 256, 256, eng.stream, core, fv.ivnum, out64);
    else GL_LAUNCH(k_core_out<int32_t>, (fv.ivnum + 255) / 256, 256, eng.stream, cnt, fv.ivnum, out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(int64_t) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_core_decomposition() { return new CoreApp<true>; }
gl_app* make_kcore() { return new CoreApp<false>; }

}  // namespace gl
