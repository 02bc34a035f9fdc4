// app_pagerank_local.cu — un-normalised PageRank (the reference's PageRankLocal,
// examples/analytical_apps/pagerank/pagerank_local.h, run_app --application pagerank_local) on an
// undirected or a directed fragment.
//
// x[v] holds c(v) / deg(v) (c(v) itself when deg(v) = 0), deg(v) the length of v's out-row.  PEval
// sets x[v] = 1 / deg(v) (1 when deg(v) = 0); a round is one pull over the out-rows:
//   c(v) = (1 - d) + d * (sum of x[u] over the entries u of v's out-row),
//   x'[v] = c(v) / deg(v), or c(v) when deg(v) = 0,
// and the last round writes c(v) itself.  There is no normalisation by N and no dangling mass, so the
// ranks sum to about N.
//
// The out-row sums use the row tiers of row_tiers.cuh, so every sum has one fixed order and the output
// is bit-identical from run to run; the epilogue (c, x' or the output) runs in the tiers' row consumer.
// A round has no global scalar, so there is no fold and no all-reduce: all R rounds are enqueued back
// to back in PEval with no host synchronisation.  Several fragments: x reaches the outer copies by the
// dense mirror sync (planned once in Setup) after PEval and after rounds 1..R-1.
#include "row_tiers.cuh"

namespace gl {
namespace {

constexpr int kPrlLongTB = 256;   // threads per CTA of the long-row fold

// the consumer of a finished out-row sum
struct PrlOut {
  const uint64_t* oe_rp;
  double* xn;    // x of the next round
  double* res;   // last round: the output
  double d;
  bool last;
  GL_DEV void operator()(uint32_t v, double sum) const {
    const double c = (1.0 - d) + d * sum;
    if (last) {
      res[v] = c;
    } else {
      const uint64_t deg = oe_rp[v + 1] - oe_rp[v];
      xn[v] = deg ? c / (double) deg : c;
    }
  }
};

__global__ void k_prl_init(const uint64_t* __restrict__ oe_rp, uint32_t ivnum, double* __restrict__ x) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < ivnum) {
    const uint64_t deg = oe_rp[v + 1] - oe_rp[v];
    x[v] = deg ? 1.0 / (double) deg : 1.0;
  }
}

// eight CTAs per SM: with no dangling share to carry (unlike k_prd_pull) the loop fits the 32
// registers ptxas aims for at full occupancy without spilling, and the gather is latency-bound
__global__ void __launch_bounds__(kTB, 8)
k_prl_pull(const uint64_t* __restrict__ oe_rp, const uint32_t* __restrict__ oe_col, uint32_t ivnum,
           const double* __restrict__ x, PrlOut out) {
  tier_rows(oe_rp, oe_col, ivnum, x, out);
}

__global__ void __launch_bounds__(kTB)
k_prl_chunks(const uint64_t* __restrict__ cb, const uint64_t* __restrict__ ce, uint32_t nitems,
             const uint32_t* __restrict__ oe_col, const double* __restrict__ x, double* __restrict__ csum) {
  tier_chunks(cb, ce, nitems, oe_col, x, csum);
}

__global__ void __launch_bounds__(kPrlLongTB)
k_prl_long(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ off, uint32_t nlong,
           const double* __restrict__ csum, PrlOut out) {
  tier_long(rows, off, nlong, csum, out);
}

struct PageRankLocalApp : gl_app {
  DevBuf<double> x[2], res;
  TierLongRows lr;   // out-rows longer than kTierChunk entries
  int grid_pull = 0, grid_long = 0, grid_chunks = 0;
  uint64_t sync_bytes = 0;

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    if (cfg.max_round <= 0) {
      set_error("pagerank_local needs max_round >= 1 (the output is c of round max_round)");
      return GL_ERR_ARG;
    }
    const uint32_t tvnum = fv.ivnum + fv.ovnum;
    GL_CUDA(x[0].alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(x[1].alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(res.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    if (fv.ivnum) {
      GL_TRY(lr.plan(fv.oe_rp, fv.ivnum));
      static thread_local int gp = 0;
      if (!gp) gp = persistent_grid(k_prl_pull, eng.sm_count);
      grid_pull = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) fv.ivnum + kTB - 1) / kTB);
      grid_chunks = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) lr.nitems * 32 + kTB - 1) / kTB);
      grid_long = (int) ((lr.nlong + kPrlLongTB - 1) / kPrlLongTB);
    }
    GL_TRY(mm.Init(comm, fv, 8));
    if (fv.fnum > 1) {
      GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
      sync_bytes = 8 * mm.mirror_total;
    }
    return GL_OK;
  }

  int Init() override { return GL_OK; }

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
    cudaStream_t s = eng.stream;
    GL_LAUNCH(k_prl_init, std::max<uint32_t>((fv.ivnum + 255) / 256, 1), 256, s, fv.oe_rp, fv.ivnum, x[0]);
    GL_TRY(sync_x(s, x[0]));
    GL_CUDA(cudaEventRecord(rec.next(), s));
    int cur = 0;
    for (int k = 1; k <= R; ++k) {
      const bool last = k == R;
      const PrlOut out{fv.oe_rp, x[cur ^ 1], res, cfg.pr_delta, last};
      if (fv.ivnum) {
        GL_LAUNCH(k_prl_pull, grid_pull, kTB, s, fv.oe_rp, fv.oe_col, fv.ivnum, x[cur], out);
        if (lr.nlong) {
          GL_LAUNCH(k_prl_chunks, grid_chunks, kTB, s, lr.cb, lr.ce, lr.nitems, fv.oe_col, x[cur], lr.csum);
          GL_LAUNCH(k_prl_long, grid_long, kPrlLongTB, s, lr.rows, lr.off, lr.nlong, lr.csum, out);
        }
      }
      if (!last) GL_TRY(sync_x(s, x[cur ^ 1]));
      cur ^= 1;
      GL_CUDA(cudaEventRecord(rec.next(), s));
      note_step(frag->oe.entries, fv.ivnum, 2);
      q_touched += fv.ivnum;
    }
    return GL_OK;
  }

  int IncEval() override { return GL_OK; }

  void FillStats(gl_query_stats* st) override {
    const int R = cfg.max_round;
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

gl_app* make_pagerank_local() { return new PageRankLocalApp; }

}  // namespace gl
