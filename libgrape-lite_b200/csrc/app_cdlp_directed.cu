// app_cdlp_directed.cu — community detection by synchronous label propagation on a directed graph,
// over the in- and out-neighbours of every vertex.
//
// Semantics of the GPU app cuda/cdlp/cdlp.h on a kBothOutIn fragment (PropagateLabel_first_d and the
// isDirected branches of PropagateLabel_lo / _hi), the LDBC Graphalytics directed CDLP: labels start as
// the vertex id; for max_round rounds every vertex takes the most frequent label of the multiset
// ie(v) + oe(v) (a reciprocal pair and a self loop count twice, every repeated edge once per copy),
// ties -> smallest label; all vertices update at once.  A vertex with no in- and no out-edges keeps its
// label, one with only in-edges updates (GL_APP_CDLP keeps the label of a vertex without out-edges).
// Labels are 32-bit gids, as in app_cdlp.cu, and mapped to oids on output.
//
// One round: (1) the labels of the in-row and of the out-row are gathered into two scratch arrays
// with the coalesced k_cdlp_gather and (2) each is sorted per row by a segmented radix sort over the
// fragment's own ie_rp / oe_rp; (3) a vote pass walks the two sorted halves A (in-labels) and B
// (out-labels) of a row together: every run end in A at label x votes runA(x) + |equal_range(B, x)|,
// every run end in B at a label y absent from A votes runB(y), and the packed (count << 32 | ~label)
// maximum wins.  Rows of up to kCdlpdWarpRow entries are voted by a warp, longer ones (R-MAT hubs) by
// a CTA, through a list of those rows built once in Setup.  Several fragments: outer copies read their
// owner's label every round after the first (dense mirror sync, which covers the outer copies seen
// only through in-edges).
#include <cub/cub.cuh>

#include "cdlp_common.cuh"

namespace gl {
namespace {

constexpr uint64_t kCdlpdWarpRow = 1024;   // rows with more in + out entries are voted by a whole CTA

// first position in [lo, hi) of sorted a holding a value >= x (upper: > x)
template <bool kUpper>
GL_DEV uint64_t bound_u32(const uint32_t* a, uint64_t lo, uint64_t hi, uint32_t x) {
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (kUpper ? a[mid] <= x : a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

GL_DEV unsigned long long cdlpd_pack(uint64_t count, uint32_t label) {
  return ((unsigned long long) count << 32) | (0xFFFFFFFFu - label);
}

// One row's sorted in-labels A and out-labels B.
struct CdlpdRow {
  const uint32_t* A;
  const uint32_t* B;
  uint64_t na, nb;
  // the vote of entry k of A ++ B: (count, label) at the run end that owns a label, 0 elsewhere
  GL_DEV unsigned long long vote(uint64_t k) const {
    if (k < na) {
      const uint32_t x = A[k];
      if (k + 1 < na && A[k + 1] == x) return 0;
      const uint64_t lb = bound_u32<false>(B, 0, nb, x);
      const uint64_t in_b = bound_u32<true>(B, lb, nb, x) - lb;
      return cdlpd_pack(k + 1 - bound_u32<false>(A, 0, k, x) + in_b, x);
    }
    k -= na;
    const uint32_t y = B[k];
    if (k + 1 < nb && B[k + 1] == y) return 0;
    const uint64_t la = bound_u32<false>(A, 0, na, y);
    if (la < na && A[la] == y) return 0;   // voted at its run end in A
    return cdlpd_pack(k + 1 - bound_u32<false>(B, 0, k, y), y);
  }
};

struct CdlpdRows {
  const uint64_t *ie_rp, *oe_rp;
  const uint32_t *in, *out;   // sorted labels of every in-row / out-row
  GL_DEV CdlpdRow row(uint32_t v) const {
    const uint64_t ib = ie_rp[v], ob = oe_rp[v];
    return CdlpdRow{in + ib, out + ob, ie_rp[v + 1] - ib, oe_rp[v + 1] - ob};
  }
};

GL_DEV unsigned long long warp_max_u64(unsigned long long x) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, x, o);
    x = t > x ? t : x;
  }
  return x;
}

// rows of up to kCdlpdWarpRow entries: one warp per row
__global__ void __launch_bounds__(256)
k_cdlpd_vote_warp(CdlpdRows a, uint32_t ivnum, const uint32_t* __restrict__ label, uint32_t* next) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const CdlpdRow r = a.row(v);
    const uint64_t n = r.na + r.nb;
    if (n > kCdlpdWarpRow) continue;
    if (n == 0) {
      if (lane_id() == 0) next[v] = label[v];   // no in- and no out-edges: keep
      continue;
    }
    unsigned long long best = 0;
    for (uint64_t k = lane_id(); k < n; k += 32) {
      const unsigned long long c = r.vote(k);
      best = c > best ? c : best;
    }
    best = warp_max_u64(best);
    if (lane_id() == 0) next[v] = 0xFFFFFFFFu - (uint32_t) best;
  }
}

// longer rows, listed in `rows`: one CTA per row
__global__ void __launch_bounds__(kTB)
k_cdlpd_vote_cta(CdlpdRows a, const uint32_t* __restrict__ rows, uint32_t nrows, uint32_t* next) {
  __shared__ unsigned long long s_best[kTB / 32];
  for (uint32_t t = blockIdx.x; t < nrows; t += gridDim.x) {
    const uint32_t v = rows[t];
    const CdlpdRow r = a.row(v);
    const uint64_t n = r.na + r.nb;
    unsigned long long best = 0;
    for (uint64_t k = threadIdx.x; k < n; k += kTB) {
      const unsigned long long c = r.vote(k);
      best = c > best ? c : best;
    }
    best = warp_max_u64(best);
    if (lane_id() == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kTB / 32; ++w) best = s_best[w] > best ? s_best[w] : best;
      next[v] = 0xFFFFFFFFu - (uint32_t) best;
    }
    __syncthreads();
  }
}

__global__ void k_cdlpd_long_rows(const uint64_t* __restrict__ ie_rp, const uint64_t* __restrict__ oe_rp,
                                  uint32_t ivnum, uint32_t* rows, uint32_t* count) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < ivnum && (ie_rp[v + 1] - ie_rp[v]) + (oe_rp[v + 1] - oe_rp[v]) > kCdlpdWarpRow)
    rows[atomicAdd(count, 1u)] = v;
}

struct CdlpDirectedApp : gl_app {
  DevBuf<uint32_t> label, next, scratch, sorted_in, sorted_out, long_rows;
  DevBuf<int64_t> out64;
  DevBuf<char> sort_tmp;
  size_t sort_bytes = 0;
  uint32_t tvnum = 0, nlong = 0;
  int step = 0;

  size_t ResultElemBytes() const override { return sizeof(int64_t); }

  int Setup() override {
    // the reference runs its directed CDLP on kBothOutIn fragments
    if (!fv.directed) {
      set_error("cdlp_directed needs a directed fragment; GL_APP_CDLP is the label propagation of an undirected one");
      return GL_ERR_ARG;
    }
    if (frag->ie_alias_oe) {
      set_error("cdlp_directed needs the incoming adjacency (gl_frag_desc.ie / kBothOutIn)");
      return GL_ERR_ARG;
    }
    tvnum = fv.ivnum + fv.ovnum;
    const uint64_t mi = frag->ie.entries, mo = frag->oe.entries;
    GL_CUDA(label.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(next.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(scratch.alloc(std::max<uint64_t>(std::max(mi, mo), 4)));
    GL_CUDA(sorted_in.alloc(std::max<uint64_t>(mi, 4)));
    GL_CUDA(sorted_out.alloc(std::max<uint64_t>(mo, 4)));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    size_t bi = 0, bo = 0;
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bi, scratch.get(), sorted_in.get(), (int64_t) mi,
                                               (int64_t) fv.ivnum, fv.ie_rp, fv.ie_rp + 1, eng.stream));
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bo, scratch.get(), sorted_out.get(), (int64_t) mo,
                                               (int64_t) fv.ivnum, fv.oe_rp, fv.oe_rp + 1, eng.stream));
    sort_bytes = std::max(bi, bo);
    GL_CUDA(sort_tmp.alloc(std::max<size_t>(sort_bytes, 16)));
    // the rows the CTA vote takes, once: they do not change between queries
    if (fv.ivnum) {
      DevBuf<uint32_t> rows, count;
      GL_CUDA(rows.alloc(fv.ivnum));
      GL_CUDA(count.alloc(1));
      GL_CUDA(cudaMemsetAsync(count, 0, sizeof(uint32_t), eng.stream));
      GL_LAUNCH(k_cdlpd_long_rows, (fv.ivnum + 255) / 256, 256, eng.stream, fv.ie_rp, fv.oe_rp, fv.ivnum, rows.get(),
                count.get());
      GL_CUDA(cudaMemcpyAsync(&nlong, count, sizeof(uint32_t), cudaMemcpyDeviceToHost, eng.stream));
      GL_CUDA(cudaStreamSynchronize(eng.stream));
      if (nlong) {
        GL_CUDA(long_rows.alloc(nlong));
        GL_CUDA(cudaMemcpyAsync(long_rows, rows, sizeof(uint32_t) * nlong, cudaMemcpyDeviceToDevice, eng.stream));
        GL_CUDA(cudaStreamSynchronize(eng.stream));
      }
    }
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32U32)));
    // outer copies, also those reached only through in-edges, read their owner's label every round
    if (fv.fnum > 1) GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
    return GL_OK;
  }

  int Init() override {
    step = 0;
    return GL_OK;
  }

  // gather + per-row sort of one adjacency's labels into `sorted`
  int SortedLabels(const uint64_t* rp, const uint32_t* col, uint64_t m, uint32_t* sorted) {
    if (!m) return GL_OK;
    cudaStream_t s = eng.stream;
    GL_LAUNCH(k_cdlp_gather, eng.sm_count * 8, 256, s, col, m, label, scratch);
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(sort_tmp, sort_bytes, scratch.get(), sorted, (int64_t) m,
                                               (int64_t) fv.ivnum, rp, rp + 1, s));
    g_kernel_launches += 3;  // cub's partition + large/small segment kernels
    return GL_OK;
  }

  int Propagate() {
    cudaStream_t s = eng.stream;
    const uint64_t mi = frag->ie.entries, mo = frag->oe.entries;
    if (fv.fnum > 1 && step > 1) GL_TRY(mm.SyncValuesToGhosts(s, label, 4));
    GL_TRY(SortedLabels(fv.ie_rp, fv.ie_col, mi, sorted_in));
    GL_TRY(SortedLabels(fv.oe_rp, fv.oe_col, mo, sorted_out));
    const CdlpdRows rows{fv.ie_rp, fv.oe_rp, sorted_in, sorted_out};
    if (fv.ivnum) GL_LAUNCH(k_cdlpd_vote_warp, eng.sm_count * 8, 256, s, rows, fv.ivnum, label, next);
    if (nlong)
      GL_LAUNCH(k_cdlpd_vote_cta, std::min<uint32_t>(nlong, eng.sm_count * 4), kTB, s, rows, long_rows, nlong, next);
    std::swap(label, next);
    note_step(mi + mo, fv.ivnum, 2);
    q_touched += fv.ivnum;
    return GL_OK;
  }

  int PEval() override {
    // labels are initialised before the round check, so max_round = 0 yields the identity labelling
    if (tvnum) GL_LAUNCH(k_cdlp_init, (tvnum + 255) / 256, 256, eng.stream, label, fv.ivnum, fv.ovnum, fv.ovgid, fv.fid, fv.fid_offset);
    ++step;
    if (step > cfg.max_round) return GL_OK;
    mm.ForceContinue();
    return Propagate();
  }

  int IncEval() override {
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

gl_app* make_cdlp_directed() { return new CdlpDirectedApp; }

}  // namespace gl
