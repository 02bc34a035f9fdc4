// app_pagerank_directed.cu — the directed PageRank of LDBC Graphalytics (the reference's
// PageRankDirected, examples/analytical_apps/pagerank/pagerank_directed.h, run_app_opt --application
// pagerank --directed) on a kBothOutIn fragment.
//
// x[v] holds rank / deg(v) (the rank itself when v is dangling, deg(v) = 0), as the reference's
// result array does between rounds.  A round is one pull over the in-rows:
//   c(v) = d * (sum of x[w] over ie(v)) + base,   base = (1 - d)/N + d * S/N,
//   x'[v] = c(v) / deg(v), or c(v) when v is dangling,
// and S, the mass the dangling vertices hold, is the sum of their c(v) for the next round.  A sink
// keeps what arrives over its in-edges, so the ranks of the group sum to 1 (GL_APP_PAGERANK on a
// directed fragment follows pagerank_parallel.h instead, where a sink is reset to base).
//
// The in-row sums use the row tiers of row_tiers.cuh, so every sum has one fixed order and the output
// is bit-identical from run to run.  The epilogue (c, x', the vertex's share of S) runs in the tiers'
// row consumer; a CTA reduces its dangling share in a fixed tree order into one partial, and one
// thread folds the partials in CTA order into S and the next base.  On one fragment S and base stay on
// the device and the rounds are enqueued back to back: the whole query is PEval's, with no host
// synchronisation between rounds.  Several fragments: x reaches the outer copies (also those seen only
// through in-edges) by the dense mirror sync after PEval and after rounds 1..R-1; the dangling count D
// is all-reduced once in Setup and S after rounds 1..R-1, each as a left fold in fid order.
#include "row_tiers.cuh"

namespace gl {
namespace {

constexpr int kPrdLongTB = 256;   // threads per CTA of the long-row fold

__host__ __device__ inline double prd_base(double S, double N, double d) { return (1.0 - d) / N + d * S / N; }

// the device scalars of a query: S (this fragment's share until it is all-reduced) and base
struct PrdScal {
  double S, base;
};

// the consumer of a finished in-row sum
struct PrdOut {
  const uint64_t* oe_rp;
  double* xn;    // x of the next round
  double* res;   // last round: the output
  double d, base;
  bool last;
  double dangling = 0.0;      // this thread's share of S, in row order
  GL_DEV void operator()(uint32_t v, double sum) {
    const uint64_t deg = oe_rp[v + 1] - oe_rp[v];
    const double c = d * sum + base;
    if (last) {
      res[v] = deg ? c / (double) deg * (double) deg : c;   // the reference's multiply-back
    } else if (deg) {
      xn[v] = c / (double) deg;
    } else {
      xn[v] = c;
      dangling += c;
    }
  }
};

// the CTA's dangling share: warp trees, then the warps in order
GL_DEV void prd_cta_partial(double v, double* part) {
  __shared__ double s_w[32];
  v = warp_sum(v);
  if (lane_id() == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (uint32_t w = 0; w < (blockDim.x >> 5); ++w) s += s_w[w];
    part[blockIdx.x] = s;
  }
}

__global__ void k_prd_init(const uint64_t* __restrict__ oe_rp, uint32_t ivnum, double p, double* __restrict__ x,
                           PrdScal* scal, double base) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < ivnum) {
    const uint64_t deg = oe_rp[v + 1] - oe_rp[v];
    x[v] = deg ? p / (double) deg : p;
  }
  if (v == 0) scal->base = base;
}

// six CTAs per SM: at the eight ptxas aims for by default (32 registers) the loop state spills
__global__ void __launch_bounds__(kTB, 6)
k_prd_pull(const uint64_t* __restrict__ ie_rp, const uint32_t* __restrict__ ie_col, uint32_t ivnum,
           const double* __restrict__ x, PrdOut o, const PrdScal* __restrict__ scal, double* part) {
  PrdOut out{o.oe_rp, o.xn, o.res, o.d, scal->base, o.last};
  tier_rows(ie_rp, ie_col, ivnum, x, out);
  prd_cta_partial(out.dangling, part);
}

__global__ void __launch_bounds__(kTB)
k_prd_chunks(const uint64_t* __restrict__ cb, const uint64_t* __restrict__ ce, uint32_t nitems,
             const uint32_t* __restrict__ ie_col, const double* __restrict__ x, double* __restrict__ csum) {
  tier_chunks(cb, ce, nitems, ie_col, x, csum);
}

__global__ void __launch_bounds__(kPrdLongTB)
k_prd_long(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ off, uint32_t nlong,
           const double* __restrict__ csum, PrdOut o, const PrdScal* __restrict__ scal, double* part) {
  PrdOut out{o.oe_rp, o.xn, o.res, o.d, scal->base, o.last};
  tier_long(rows, off, nlong, csum, out);
  prd_cta_partial(out.dangling, part);
}

// S = the partials in CTA order (the pull's CTAs, then the long-row fold's); base of the next round
__global__ void k_prd_fold(const double* __restrict__ part, uint32_t np, double N, double d, PrdScal* scal) {
  double s = 0.0;
  for (uint32_t i = 0; i < np; ++i) s += part[i];
  scal->S = s;
  scal->base = prd_base(s, N, d);
}

struct PageRankDirectedApp : gl_app {
  DevBuf<double> x[2], res, part;
  DevBuf<PrdScal> scal;
  TierLongRows lr;   // in-rows longer than kTierChunk entries
  uint32_t tvnum = 0;
  int grid_pull = 0, grid_long = 0, grid_chunks = 0;
  int64_t ndangling = 0;   // D, over the group
  uint64_t sync_bytes = 0;

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    if (!fv.directed) {
      set_error("pagerank_directed needs a directed fragment; GL_APP_PAGERANK is the PageRank of an undirected one");
      return GL_ERR_ARG;
    }
    if (frag->ie_alias_oe) {
      set_error("pagerank_directed needs the incoming adjacency (gl_frag_desc.ie / kBothOutIn)");
      return GL_ERR_ARG;
    }
    cudaStream_t s = eng.stream;
    tvnum = fv.ivnum + fv.ovnum;
    GL_CUDA(x[0].alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(x[1].alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(res.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    GL_CUDA(scal.alloc(1));
    if (fv.ivnum) {
      GL_TRY(lr.plan(fv.ie_rp, fv.ivnum));
      static thread_local int gp = 0;
      if (!gp) gp = persistent_grid(k_prd_pull, eng.sm_count);
      grid_pull = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) fv.ivnum + kTB - 1) / kTB);
      grid_chunks = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) lr.nitems * 32 + kTB - 1) / kTB);
      grid_long = (int) ((lr.nlong + kPrdLongTB - 1) / kPrdLongTB);
    }
    GL_CUDA(part.alloc(std::max(grid_pull + grid_long, 1)));
    // D: the vertices with an empty out-row
    long long d0 = 0, d1 = 0;
    if (fv.ivnum) {
      std::vector<uint64_t> rp(fv.ivnum + 1);
      GL_CUDA(cudaMemcpy(rp.data(), fv.oe_rp, sizeof(uint64_t) * (fv.ivnum + 1), cudaMemcpyDeviceToHost));
      for (uint32_t v = 0; v < fv.ivnum; ++v) d0 += rp[v + 1] == rp[v];
    }
    GL_TRY(mm.Init(comm, fv, 8));
    if (fv.fnum > 1) {
      double unused = 0;
      GL_TRY(mm.PeerAllReduce(s, &d0, &d1, &unused, 0));
      // outer copies, also those reached only through in-edges, read their owner's x
      GL_TRY(mm.BuildMirrorPlan(s, fv));
      sync_bytes = 8 * mm.mirror_total;
    }
    ndangling = d0;
    return GL_OK;
  }

  int Init() override {
    if (cfg.max_round <= 0 && fv.ivnum) GL_CUDA(cudaMemsetAsync(res, 0, sizeof(double) * fv.ivnum, eng.stream));
    return GL_OK;
  }

  // x reaches the outer copies (several fragments)
  int sync_x(cudaStream_t s, double* xs) {
    if (fv.fnum == 1) return GL_OK;
    GL_TRY(mm.SyncValuesToGhosts(s, xs, 8));
    mm.bytes_sent += sync_bytes;
    return GL_OK;
  }

  // The whole query: PEval's initialisation and all R rounds (see the file comment).  Each round is
  // recorded as its own step (the events bracket it on the stream), so the statistics read as R + 1
  // supersteps (FillStats).
  int PEval() override {
    const int R = cfg.max_round;
    if (R <= 0) return GL_OK;
    cudaStream_t s = eng.stream;
    const double N = (double) fv.total_vnum, d = cfg.pr_delta, p = 1.0 / N;
    // PEval: x = p / deg (p when dangling), S = p * D
    GL_LAUNCH(k_prd_init, std::max<uint32_t>((fv.ivnum + 255) / 256, 1), 256, s, fv.oe_rp, fv.ivnum, p, x[0], scal,
              prd_base(p * (double) ndangling, N, d));
    GL_TRY(sync_x(s, x[0]));
    GL_CUDA(cudaEventRecord(rec.next(), s));
    int cur = 0;
    for (int k = 1; k <= R; ++k) {
      const bool last = k == R;
      PrdOut out{fv.oe_rp, x[cur ^ 1], res, d, 0.0, last};
      if (fv.ivnum) {
        GL_LAUNCH(k_prd_pull, grid_pull, kTB, s, fv.ie_rp, fv.ie_col, fv.ivnum, x[cur], out, scal, part);
        if (lr.nlong) {
          GL_LAUNCH(k_prd_chunks, grid_chunks, kTB, s, lr.cb, lr.ce, lr.nitems, fv.ie_col, x[cur], lr.csum);
          GL_LAUNCH(k_prd_long, grid_long, kPrdLongTB, s, lr.rows, lr.off, lr.nlong, lr.csum, out, scal,
                    part.get() + grid_pull);
        }
      }
      if (!last) {
        GL_LAUNCH(k_prd_fold, 1, 1, s, part, (uint32_t) (grid_pull + grid_long), N, d, scal);
        if (fv.fnum > 1) {
          // S over the group, folded in fid order on every rank
          PrdScal h;
          GL_CUDA(cudaMemcpyAsync(&h, scal, sizeof(h), cudaMemcpyDeviceToHost, s));
          GL_CUDA(cudaStreamSynchronize(s));
          long long i0 = 0, i1 = 0;
          GL_TRY(mm.PeerAllReduce(s, &i0, &i1, &h.S, 0));
          mm.bytes_sent += 8 * (fv.fnum - 1);
          h.base = prd_base(h.S, N, d);
          GL_CUDA(cudaMemcpyAsync(scal, &h, sizeof(h), cudaMemcpyHostToDevice, s));
        }
        GL_TRY(sync_x(s, x[cur ^ 1]));
      }
      cur ^= 1;
      GL_CUDA(cudaEventRecord(rec.next(), s));
      note_step(frag->ie.entries, fv.ivnum, 2);
      q_touched += fv.ivnum;
    }
    return GL_OK;
  }

  int IncEval() override { return GL_OK; }

  void FillStats(gl_query_stats* st) override {
    const int R = cfg.max_round;
    if (R <= 0) return;
    st->supersteps = R + 1;
    st->n_steps = std::min(R + 1, GL_MAX_STEP_STATS);
    // the worker's closing interval (its round barrier) is not a step of its own
    if (R + 1 < GL_MAX_STEP_STATS) {
      st->step_ms[R + 1] = 0.f;
      st->step_entries[R + 1] = 0;
      st->step_frontier[R + 1] = 0;
      st->step_mode[R + 1] = 0;
    }
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_CUDA(cudaMemcpyAsync(host_out, res, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_pagerank_directed() { return new PageRankDirectedApp; }

}  // namespace gl
