// app_wcc.cu — weakly connected components by min-label propagation.
//
// Behaviour follows examples/analytical_apps/cuda/wcc/wcc.h:24-221: PEval
// (:92-114) labels every local vertex with its gid and activates all of them;
// IncEval (:116-219) applies received labels with atomicMin, pushes
// label[u] along out- (and, when directed, in-) edges of the active vertices,
// reports improved outer vertices to their owners and continues while any
// inner vertex changed.  The fixpoint (component minimum) is order
// independent => bit-exact.
//
// Result: int64 per inner vertex = oid of the minimum-gid vertex of its
// component.  With the order-preserving segmented partitioner used here
// gid order == oid order, so this equals the CPU app's min-oid label
// (wcc/wcc.h:139-153) as well as the GPU app's min-gid label.
#include "apps_common.cuh"
#include "dense.cuh"

namespace gl {
namespace {

// (A hub-first relabelled shadow CSR like the BFS one was measured here and
// for SSSP: with DENSE frontiers it concentrates every heavy row in the first
// tiles, and round 1 went from 4.9 ms to 36 ms on R-MAT-24 — not used.)
struct OpWcc {
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* label;
  uint32_t* out_local;
  uint32_t* remote;
  uint32_t ivnum;
  GL_DEV Meta assign(uint32_t u) const { return label[u]; }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W, ScanAcc& acc) const {
    if (!(m < label[v])) return;
    if (m < atomicMin(label + v, m)) {
      acc.touched++;
      if (v < ivnum) {
        if (bit_set_atomic(out_local, v)) acc.next_count++;
      } else {
        if (bit_set_atomic(remote, v)) acc.remote++;
      }
    }
  }
};

// dense rounds as an edge-balanced pull sweep (dense.cuh): label[row] =
// min(label[row], min over the row's neighbours).  On a symmetric adjacency
// this covers every push of wcc.h:166-198 without one atomic per edge.
struct OpWccPull {
  using Val = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* label;
  uint32_t* out_local;
  GL_DEV Val identity() const { return 0xFFFFFFFFu; }
  GL_DEV Val entry(uint32_t v, W) const { return __ldcg(label + v); }
  GL_DEV Val combine(Val a, Val b) const { return a < b ? a : b; }
  GL_DEV void flush(uint32_t row, Val part, ScanAcc& acc) const {
    if (part < label[row]) {
      if (part < atomicMin(label + row, part)) {
        acc.touched++;
        if (bit_set_atomic(out_local, row)) acc.next_count++;
      }
    }
  }
};

__global__ void k_wcc_init(uint32_t* label, uint32_t ivnum, uint32_t ovnum,
                           const uint32_t* ovgid, uint32_t fid, int fid_offset,
                           uint32_t* in_q, uint32_t words) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum) label[i] = (fid << fid_offset) | i;       // Vertex2Gid, inner
  else if (i < ivnum + ovnum) label[i] = ovgid[i - ivnum];  // outer
  if (i < words) {
    // all inner vertices active
    uint32_t lo = i * 32;
    uint32_t w = 0;
    if (lo + 32 <= ivnum) w = 0xFFFFFFFFu;
    else if (lo < ivnum) w = (1u << (ivnum - lo)) - 1u;
    in_q[i] = w;
  }
}

struct WccPayload {
  const uint32_t* label;
  GL_DEV ItemU32U32 operator()(uint32_t v, uint32_t lid) const {
    return ItemU32U32{lid, label[v]};
  }
};
struct WccApply {
  uint32_t* label;
  uint32_t* in_q;
  GL_DEV void operator()(const ItemU32U32& it, ScanAcc& acc) const {
    if (it.val < atomicMin(label + it.lid, it.val)) {
      if (bit_set_atomic(in_q, it.lid)) acc.aux++;
    }
  }
};

__global__ void k_wcc_out(const uint32_t* label, uint32_t n, LabelMap lm, int64_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = lm.oid(label[i]);
}

struct WccApp : gl_app {
  DevBuf<uint32_t> label, in_q, out_local, remote;
  DevBuf<int64_t> out64;
  size_t words = 0;
  uint32_t tvnum = 0;
  uint64_t active_estimate = 0;   // vertices active in the coming round

  size_t ResultElemBytes() const override { return sizeof(int64_t); }

  int Setup() override {
    // weak connectivity needs both edge directions (wcc.h:181-197 scans ie and oe):
    // a directed fragment created without an ie CSR cannot provide them
    if (fv.directed && frag->ie_alias_oe) {
      set_error("WCC on a directed fragment needs the incoming adjacency (gl_frag_desc.ie / kBothOutIn)");
      return GL_ERR_ARG;
    }
    tvnum = fv.ivnum + fv.ovnum;
    words = bm_words(tvnum) + 1;
    GL_CUDA(label.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(in_q.alloc(words));
    GL_CUDA(out_local.alloc(words));
    GL_CUDA(remote.alloc(words));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    return mm.Init(comm, fv, sizeof(ItemU32U32));
  }

  int Init() override {
    cudaStream_t s = eng.stream;
    GL_CUDA(cudaMemsetAsync(out_local, 0, sizeof(uint32_t) * words, s));
    GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
    l2_persist_window(s, label, sizeof(uint32_t) * (size_t) tvnum);   // random label[v] probes stay in L2
    return GL_OK;
  }

  int PEval() override {
    uint32_t n = (uint32_t) std::max<size_t>(tvnum, words);
    GL_LAUNCH(k_wcc_init, (n + 255) / 256, 256, eng.stream, label, fv.ivnum, fv.ovnum,
              fv.ovgid, fv.fid, fv.fid_offset, in_q, (uint32_t) words);
    active_estimate = fv.ivnum;
    mm.ForceContinue();
    return GL_OK;
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    GL_TRY(eng.reset_ctrl());
    if (fv.fnum > 1) {
      MsgView mv = mm.view();
      WccApply ap{label, in_q};
      GL_LAUNCH((k_unpack<ItemU32U32, WccApply>), eng.sm_count * 4, kTB, s, mv, ap, eng.ctrl);
      GL_TRY(eng.reset_ctrl());
    }
    OpWcc op{label, out_local, remote, fv.ivnum};
    EdgeRange er{fv.oe_rp, fv.oe_col, nullptr};
    // cfg.reserved[0] = 1 selects the pull sweep for dense rounds (measured
    // slower than the push scan on R-MAT-24: 8.5 ms vs 4.9 ms per round, so
    // it is off by default)
    const bool dense = cfg.reserved[0] == 1 && fv.fnum == 1 && !fv.directed && frag->oe_ntiles > 0 &&
                       active_estimate > (uint64_t) fv.ivnum / 8;
    if (dense) {
      static thread_local int gd = 0;
      if (!gd) gd = persistent_grid(k_dense_pull<OpWccPull>, eng.sm_count);
      OpWccPull pop{label, out_local};
      int grid = (int) std::min<uint32_t>((uint32_t) gd, frag->oe_ntiles);
      GL_LAUNCH(k_dense_pull<OpWccPull>, grid, kTB, s, fv.oe_rp, fv.oe_col, (const void*) nullptr,
                frag->oe_tile_row, frag->oe_ntiles, fv.ivnum, (uint64_t) frag->oe.entries, pop, eng.ctrl);
    } else {
      GL_TRY(run_frontier_scan(eng, in_q, fv.ivnum, er, op));
    }
    if (fv.directed && !frag->ie_alias_oe) {
      // second pass over the incoming adjacency (wcc.h:181-197); the tile
      // ticket must restart
      GL_CUDA(cudaMemsetAsync(&eng.ctrl->tile_ticket, 0, 16, s));
      EdgeRange ei{fv.ie_rp, fv.ie_col, nullptr};
      GL_TRY(run_frontier_scan(eng, in_q, fv.ivnum, ei, op));
    }
    if (fv.fnum > 1) {
      MsgView mv = mm.view();
      GL_LAUNCH((k_pack_outer<ItemU32U32, WccPayload>), eng.sm_count * 4, kTB, s, remote,
                fv.ivnum, fv.ovnum, fv.ovgid, mv, WccPayload{label}, 0, nullptr);
      GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
    }
    GL_CUDA(cudaMemsetAsync(in_q, 0, sizeof(uint32_t) * words, s));
    GL_TRY(eng.fetch_ctrl());
    const ScanCtrl& c = *eng.h_ctrl;
    // a dense round sweeps every inner vertex (the sweep keeps no frontier count)
    note_step(c.scanned, dense ? fv.ivnum : (uint32_t) std::min<uint64_t>(c.frontier, 0xFFFFFFFFu), dense ? 2 : 0);
    q_touched += c.touched;
    active_estimate = c.next_count;
    std::swap(out_local, in_q);
    if (c.next_count > 0) mm.ForceContinue();
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    l2_persist_clear(eng.stream);
    GL_LAUNCH(k_wcc_out, (fv.ivnum + 255) / 256, 256, eng.stream, label, fv.ivnum, label_map(*this), out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(int64_t) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_wcc() { return new WccApp; }

}  // namespace gl
