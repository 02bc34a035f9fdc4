// app_cdlp.cu — community detection by synchronous label propagation.
//
// Semantics of examples/analytical_apps/cdlp/cdlp.h:45-161 + cdlp_utils.h:35-73
// (and the GPU app cuda/cdlp/cdlp.h:27-784): labels start as the vertex id;
// for max_round rounds every vertex with out-edges takes the most frequent
// label among its out-neighbours (multi-edges count), ties -> smallest label;
// all vertices update simultaneously.  Integer-only => bit-exact.
//
// Re-design: labels are kept as 32-bit gids (gid order == oid order under
// the segmented partitioner, so "smallest label" is preserved; this is the
// reference's own GID_AS_LABEL build, cdlp.h:109-115) and mapped to oids on
// output.  One round = (1) gather neighbour labels with coalesced column
// reads into a scratch CSR, (2) one device-wide segmented radix sort,
// (3) a flat run-length pass that elects (count, min label) per row with a
// packed 64-bit atomicMax.
#include <cub/cub.cuh>

#include "cdlp_common.cuh"

namespace gl {
namespace {

// warp per row over the sorted labels: every run end votes (count, label)
__global__ void __launch_bounds__(256)
k_cdlp_mode(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ sorted,
            uint32_t ivnum, const uint32_t* __restrict__ label, uint32_t* next) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const uint64_t b = rp[v], e = rp[v + 1];
    if (b == e) {
      if (lane_id() == 0) next[v] = label[v];  // no out-edges: keep (cdlp.h:62-64)
      continue;
    }
    unsigned long long best = 0;
    for (uint64_t i = b + lane_id(); i < e; i += 32) {
      uint32_t x = sorted[i];
      if (i + 1 == e || sorted[i + 1] != x) {
        // run end: find the run start by binary search in [b, i]
        uint64_t lo = b, hi = i;
        while (lo < hi) {
          uint64_t mid = (lo + hi) >> 1;
          if (sorted[mid] < x) lo = mid + 1; else hi = mid;
        }
        unsigned long long cand = ((unsigned long long) (i - lo + 1) << 32) | (0xFFFFFFFFu - x);
        best = cand > best ? cand : best;
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
      best = t > best ? t : best;
    }
    if (lane_id() == 0) next[v] = 0xFFFFFFFFu - (uint32_t) best;
  }
}

struct CdlpApp : gl_app {
  DevBuf<uint32_t> label, next, scratch, sorted;
  DevBuf<int64_t> out64;
  DevBuf<char> sort_tmp;
  size_t sort_bytes = 0;
  uint32_t tvnum = 0;
  int step = 0;

  size_t ResultElemBytes() const override { return sizeof(int64_t); }

  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    const uint64_t m = frag->oe.entries;
    GL_CUDA(label.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(next.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(scratch.alloc(std::max<uint64_t>(m, 4)));
    GL_CUDA(sorted.alloc(std::max<uint64_t>(m, 4)));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, sort_bytes, scratch.get(), sorted.get(), (int64_t) m,
                                               (int64_t) fv.ivnum, fv.oe_rp, fv.oe_rp + 1, eng.stream));
    GL_CUDA(sort_tmp.alloc(std::max<size_t>(sort_bytes, 16)));
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32U32)));
    // outer copies read their owner's label every round (dense mirror sync;
    // the reference ships changed labels with SendMsgThroughOEdges, cdlp.h:69-70)
    if (fv.fnum > 1) GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
    return GL_OK;
  }

  int Init() override {
    step = 0;
    return GL_OK;
  }

  int Propagate() {
    cudaStream_t s = eng.stream;
    const uint64_t m = frag->oe.entries;
    if (fv.fnum > 1 && step > 1) GL_TRY(mm.SyncValuesToGhosts(s, label, 4));
    if (m) {
      GL_LAUNCH(k_cdlp_gather, eng.sm_count * 8, 256, s, fv.oe_col, m, label, scratch);
      GL_CUDA(cub::DeviceSegmentedSort::SortKeys(sort_tmp, sort_bytes, scratch.get(), sorted.get(), (int64_t) m,
                                                 (int64_t) fv.ivnum, fv.oe_rp, fv.oe_rp + 1, s));
      g_kernel_launches += 3;  // cub's partition + large/small segment kernels
    }
    if (fv.ivnum) GL_LAUNCH(k_cdlp_mode, eng.sm_count * 8, 256, s, fv.oe_rp, sorted, fv.ivnum, label, next);
    std::swap(label, next);
    note_step(m, fv.ivnum, 2);
    q_touched += fv.ivnum;
    return GL_OK;
  }

  int PEval() override {
    // cdlp.h:103-131
    // (labels are initialised before the round check so that max_round = 0
    // yields the identity labelling instead of the reference's
    // uninitialised context data)
    if (tvnum) GL_LAUNCH(k_cdlp_init, (tvnum + 255) / 256, 256, eng.stream, label, fv.ivnum, fv.ovnum, fv.ovgid, fv.fid, fv.fid_offset);
    ++step;
    if (step > cfg.max_round) return GL_OK;
    mm.ForceContinue();
    return Propagate();
  }

  int IncEval() override {
    // cdlp.h:133-161
    ++step;
    if (step > cfg.max_round) return GL_OK;
    mm.ForceContinue();
    return Propagate();
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_LAUNCH(k_cdlp_out, (fv.ivnum + 255) / 256, 256, eng.stream, label, fv.ivnum, label_map(*this), out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(int64_t) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_cdlp() { return new CdlpApp; }

}  // namespace gl
