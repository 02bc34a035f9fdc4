// app_pagerank.cu — PageRank, fixed number of rounds.
//
// Push formulation of examples/analytical_apps/cuda/pagerank/pagerank.h:37-252:
// PEval (:137-151) sets rank = 1/N; each IncEval (:153-249) first adds the
// partial sums received for its inner vertices, then (for max_iter rounds)
// computes the dangling mass (:183-193, all-reduced), initialises
//   next[v] = (1-d)/N + d*dangling/N                         (:196-200)
// pushes d*rank[u]/deg(u) along every out-edge with atomicAdd (:207-221) and
// ships the partial sums accumulated on outer vertices to their owners
// (:227-238).  Arithmetic is fp64 (the reference uses f32 for undirected
// graphs; the north-star tolerance of 1e-6 needs f64 accumulation).
// cfg.pr_pull = 1 selects a deterministic pull step (single fragment):
//   next[v] = base + d * sum_{u in N(v)} rank[u]/deg(u)
// which is the CPU app's formulation (pagerank/pagerank.h:102-154).
#include <cub/cub.cuh>

#include "apps_common.cuh"
#include "dense.cuh"

namespace gl {
namespace {

struct OpPrPush {
  using Meta = double;
  using W = float;
  static constexpr bool kWeighted = false;
  const double* rank;
  double* next;
  const uint64_t* rp;
  double delta;
  GL_DEV Meta assign(uint32_t u) const {
    uint64_t dg = rp[u + 1] - rp[u];
    return dg ? delta * rank[u] / (double) dg : 0.0;
  }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W, ScanAcc&) const {
    atomicAdd(next + v, m);
  }
};

__global__ void k_pr_init(double* rank, double* next, uint32_t ivnum,
                          uint32_t tvnum, double p) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < tvnum) {
    rank[i] = i < ivnum ? p : 0.0;
    next[i] = 0.0;
  }
}

__global__ void k_pr_dangling(const double* rank, const uint64_t* rp,
                              uint32_t ivnum, double* out) {
  double s = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ivnum;
       i += gridDim.x * blockDim.x)
    if (rp[i + 1] == rp[i]) s += rank[i];
  s = warp_sum(s);
  if (lane_id() == 0 && s != 0.0) atomicAdd(out, s);
}

// Directed fragments follow the reference's directed app (pagerank_parallel.h:52-205, pinned by
// dataset/p2p-31-PR-directed): a vertex WITHOUT out-edges keeps rank = base -- what arrives over
// its in-edges is dropped -- so the dangling mass of a round is base * N_dangling.
__global__ void k_pr_fix_dangling(double* rank, const uint64_t* rp, uint32_t ivnum, double base) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum && rp[i + 1] == rp[i]) rank[i] = base;
}

__global__ void k_pr_base(double* next, uint32_t ivnum, double base) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum) next[i] = base;
}

// pull as an edge-balanced dense sweep: next[row] += delta * sum contrib[col]
// CT = double, or float: the gathered array then is 4 B per vertex (67 MB at
// 2^24 vertices: half the bytes of the f64 one; neither fits H100's 50 MB L2 whole).  Sums stay f64;
// every term carries a relative rounding error <= 2^-24, so after the damped
// iteration the result is within 2^-24 / (1 - delta) = 4e-7 of the f64 run
// (parity bar: 1e-6).
template <typename CT>
struct OpPrPull {
  using Val = double;
  using W = float;
  static constexpr bool kWeighted = false;
  const CT* contrib;
  double* next;
  double delta;
  GL_DEV Val identity() const { return 0.0; }
  GL_DEV Val entry(uint32_t v, W) const { return (double) __ldcg(contrib + v); }
  GL_DEV Val combine(Val a, Val b) const { return a + b; }
  GL_DEV void flush(uint32_t row, Val part, ScanAcc&) const { atomicAdd(next + row, delta * part); }
};

// contrib[slot(u)] = rank[u]/deg(u).  slot = identity, or the hub-first
// permutation: the gathered array is then ordered by descending degree, so the
// few thousand hub entries that receive most of the 5e8 random reads of a
// sweep are contiguous and stay in L1/L2 (the 134 MB array does not fit L2).
template <typename CT>
__global__ void k_pr_contrib(const double* rank, const uint64_t* rp,
                             uint32_t ivnum, const uint32_t* __restrict__ perm, CT* contrib) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum) {
    uint64_t dg = rp[i + 1] - rp[i];
    contrib[perm ? perm[i] : i] = (CT) (dg ? rank[i] / (double) dg : 0.0);
  }
}
__global__ void k_pr_permute_cols(const uint32_t* __restrict__ col, uint64_t m,
                                  const uint32_t* __restrict__ perm, uint32_t n, uint32_t* out) {
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t) gridDim.x * blockDim.x) {
    uint32_t c = col[i];
    out[i] = c < n ? perm[c] : c;
  }
}


// ---------------------------------------------------------------------------
// Pull sweep with the hub contributions in shared memory.
//
// Why: every formulation of the PageRank round (f64 atomics, f64 / f32 gathers)
// is bound by the L1TEX divergent-request rate (about one 128-byte line per two
// cycles per SM), not by HBM.  Only shared memory serves 32 random lanes in a few cycles.  In the
// hub-first id space (perm) the first kPrHub = 45056 contributions (176 KB of
// f32) are the sources of ~43 % of all CSR entries of an R-MAT graph, so every
// CTA keeps them in shared memory and only the remaining entries pay a global
// (67 MB, partly L2-resident) gather.  One CTA of 1024 threads per SM, column tiles
// staged by the TMA engine (cp.async.bulk + mbarrier, double buffered).
// ---------------------------------------------------------------------------
constexpr int kPrTB = 1024;
constexpr int kPrHub = 45056;                 // f32 contributions kept in shared memory (176 KB)
constexpr int kPrEPT = kDenseTile / kPrTB;    // 4 consecutive entries per thread
struct PrHubSmem {
  float hub[kPrHub];
  uint32_t col[2][kDenseTile];
  uint64_t rp[kDenseRows + 2];
  uint64_t bar[2];
};

__global__ void __launch_bounds__(kPrTB, 1)
k_pr_pull_hub(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col_p,
              const uint32_t* __restrict__ tile_row, uint32_t ntiles, uint32_t nrows, uint64_t m,
              const float* __restrict__ contrib, uint32_t nhub, double* next, double delta, ScanCtrl* ctrl) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  PrHubSmem& sm = *reinterpret_cast<PrHubSmem*>(smem_raw);
  if (threadIdx.x == 0) {
    mbar_init(&sm.bar[0], 1);
    mbar_init(&sm.bar[1], 1);
    mbar_fence_init();
  }
  for (uint32_t i = threadIdx.x; i < nhub; i += kPrTB) sm.hub[i] = contrib[i];
  __syncthreads();

  auto issue = [&](uint32_t tile, int stage) {
    const uint64_t e0 = (uint64_t) tile * kDenseTile;
    const uint32_t n = (uint32_t) ((m - e0) < (uint64_t) kDenseTile ? (m - e0) : (uint64_t) kDenseTile);
    const uint32_t bytes = ((n * 4u) + 15u) & ~15u;
    mbar_expect_tx(&sm.bar[stage], bytes);
    tma_load_1d(&sm.col[stage][0], col_p + e0, bytes, &sm.bar[stage]);
  };

  uint32_t it = 0;
  uint32_t tile = blockIdx.x;
  if (tile < ntiles && threadIdx.x == 0) issue(tile, 0);
  for (; tile < ntiles; tile += gridDim.x, ++it) {
    const int stage = it & 1;
    const uint32_t nexttile = tile + gridDim.x;
    if (nexttile < ntiles && threadIdx.x == 0) issue(nexttile, stage ^ 1);
    const uint64_t e0 = (uint64_t) tile * kDenseTile;
    const uint32_t n = (uint32_t) ((m - e0) < (uint64_t) kDenseTile ? (m - e0) : (uint64_t) kDenseTile);
    const uint32_t r0 = tile_row[tile];
    uint32_t r1 = tile_row[tile + 1];
    if (r1 >= nrows) r1 = nrows - 1;
    const uint32_t nr = r1 - r0 + 1;
    const bool fits = nr <= (uint32_t) kDenseRows;
    if (fits)
      for (uint32_t i = threadIdx.x; i <= nr; i += kPrTB) sm.rp[i] = rp[r0 + i];
    __syncthreads();
    mbar_wait_parity(&sm.bar[stage], (it >> 1) & 1);

    const uint32_t le = threadIdx.x * kPrEPT;
    const uint4 c = *(const uint4*) &sm.col[stage][le];
    const uint32_t cs[4] = {c.x, c.y, c.z, c.w};
    // global gathers first (in flight together), shared-memory hits afterwards
    float gv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) gv[k] = (le + k < n && cs[k] >= nhub) ? __ldcg(contrib + cs[k]) : 0.0f;
    double ev[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) ev[k] = (le + k < n) ? (double) (cs[k] < nhub ? sm.hub[cs[k]] : gv[k]) : 0.0;

    uint32_t row = 0xFFFFFFFFu;
    double part = 0.0;
    if (le < n) {
      const uint64_t e = e0 + le;
      if (fits) {
        uint32_t lo = 0, hi = nr + 1;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (sm.rp[mid] <= e) lo = mid + 1; else hi = mid;
        }
        row = r0 + lo - 1;
      } else {
        uint32_t lo = r0, hi = r1 + 2;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (rp[mid] <= e) lo = mid + 1; else hi = mid;
        }
        row = lo - 1;
      }
      uint64_t row_end = fits ? sm.rp[row - r0 + 1] : rp[row + 1];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (le + k < n) {
          const uint64_t ek = e + k;
          if (ek >= row_end) {
            atomicAdd(next + row, delta * part);
            part = 0.0;
            do {
              ++row;
              row_end = fits ? sm.rp[row - r0 + 1] : rp[row + 1];
            } while (ek >= row_end);
          }
          part += ev[k];
        }
      }
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t orow = __shfl_up_sync(0xffffffffu, row, o);
      const double oval = __shfl_up_sync(0xffffffffu, part, o);
      if (lane_id() >= (uint32_t) o && orow == row) part += oval;
    }
    {
      const uint32_t nrow = __shfl_down_sync(0xffffffffu, row, 1);
      const bool tail = (lane_id() == 31) || (nrow != row);
      if (tail && row != 0xFFFFFFFFu) atomicAdd(next + row, delta * part);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && blockIdx.x == 0) atomicAdd(&ctrl->scanned, (unsigned long long) m);
}

__global__ void __launch_bounds__(kTB)
k_pr_send(double* next, uint32_t ivnum, uint32_t ovnum,
          const uint32_t* __restrict__ ovgid, MsgView mv) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t rounds = (ovnum + stride - 1) / stride;
  uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t r = 0; r < rounds; ++r, o += stride) {
    bool pred = false;
    uint32_t dst = 0;
    ItemU32F64 it{0, 0, 0.0};
    if (o < ovnum) {
      double x = next[ivnum + o];
      if (x > 0) {
        uint32_t gid = ovgid[o];
        dst = gid >> mv.fid_offset;
        it.lid = gid & mv.id_mask;
        it.val = x;
        next[ivnum + o] = 0.0;
        pred = true;
      }
    }
    msg_send<ItemU32F64>(mv, pred, dst, it);
  }
}
struct PrApply {
  double* rank;
  GL_DEV void operator()(const ItemU32F64& it, ScanAcc&) const {
    atomicAdd(rank + it.lid, it.val);
  }
};

__global__ void k_ones(uint32_t* bm, uint32_t nbits, uint32_t words) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= words) return;
  uint32_t lo = i * 32, w = 0;
  if (lo + 32 <= nbits) w = 0xFFFFFFFFu;
  else if (lo < nbits) w = (1u << (nbits - lo)) - 1u;
  bm[i] = w;
}

struct PageRankApp : gl_app {
  DevBuf<double> rank, next, contrib, d_dangling;
  DevBuf<uint32_t> all_inner;
  DevBuf<uint32_t> perm, col_p;   // hub-first gather order (pull, one fragment): perm[u] = rank of u by descending degree; col_p = perm[col]
  size_t words = 0;
  uint32_t tvnum = 0;
  int curr_iter = 0;
  double last_base = 0;
  // The pull sweep gathers along oe rows, which are the IN-neighbours only when
  // the fragment is undirected; on a directed fragment pr_pull falls back to the
  // push formulation (same ranks, pagerank.h:207-221), never a wrong gather.
  bool use_pull() const { return cfg.pr_pull && !fv.directed; }

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    words = bm_words(fv.ivnum) + 1;
    GL_CUDA(rank.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(next.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(d_dangling.alloc(1));
    GL_CUDA(all_inner.alloc(words));
    GL_LAUNCH(k_ones, (unsigned) ((words + 255) / 256), 256, eng.stream, all_inner, fv.ivnum, (uint32_t) words);
    if (use_pull()) {
      GL_CUDA(contrib.alloc(std::max<uint32_t>(tvnum, 1)));
      if (fv.fnum == 1 && fv.ivnum) {
        const uint64_t m = frag->oe.entries;
        GL_TRY(build_hub_order(eng.stream, fv.oe_rp, fv.ivnum, &perm, nullptr));
        GL_CUDA(col_p.alloc(m + 16));
        if (m) GL_LAUNCH(k_pr_permute_cols, eng.sm_count * 8, 256, eng.stream, fv.oe_col, m, perm, fv.ivnum, col_p);
        GL_CUDA(cudaStreamSynchronize(eng.stream));
      }
    }
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32F64)));
    if (use_pull() && fv.fnum > 1) GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
    return GL_OK;
  }

  int Init() override {
    curr_iter = 0;
    return GL_OK;
  }

  int PEval() override {
    double p = 1.0 / (double) fv.total_vnum;
    if (tvnum) GL_LAUNCH(k_pr_init, (tvnum + 255) / 256, 256, eng.stream, rank, next, fv.ivnum, tvnum, p);
    mm.ForceContinue();
    return GL_OK;
  }

  // contributions -> (mirror sync) -> next = base + delta * gathered sums
  template <typename CT>
  int pull_sweep(cudaStream_t s, double base) {
    CT* cb = (CT*) contrib.get();
    l2_persist_window(s, cb, sizeof(CT) * (size_t) tvnum);   // the gathered array stays in L2, the CSR streams through
    if (fv.ivnum) GL_LAUNCH(k_pr_contrib<CT>, (fv.ivnum + 255) / 256, 256, s, rank, fv.oe_rp, fv.ivnum, perm, cb);
    // outer copies take their owner's contribution (dense mirror sync)
    if (fv.fnum > 1) GL_TRY(mm.SyncValuesToGhosts(s, cb, (int) sizeof(CT)));
    if (fv.ivnum) {
      // next = base, then the TMA-staged dense sweep folds the gathered sums in
      GL_LAUNCH(k_pr_base, (fv.ivnum + 255) / 256, 256, s, next, fv.ivnum, base);
      static thread_local int gd = 0;
      if (!gd) gd = persistent_grid(k_dense_pull<OpPrPull<CT>>, eng.sm_count);
      if (frag->oe_ntiles && std::is_same<CT, float>::value && col_p && cfg.reserved[4] == 0) {
        // hub-first gather order: the first kPrHub contributions live in shared memory
        static thread_local int configured = 0;
        if (!configured) {
          GL_CUDA(cudaFuncSetAttribute(k_pr_pull_hub, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(PrHubSmem)));
          configured = 1;
        }
        const uint32_t nhub = std::min<uint32_t>((uint32_t) kPrHub, fv.ivnum);
        const int grid = (int) std::min<uint32_t>((uint32_t) eng.sm_count, frag->oe_ntiles);
        k_pr_pull_hub<<<grid, kPrTB, sizeof(PrHubSmem), s>>>(fv.oe_rp, col_p, frag->oe_tile_row, frag->oe_ntiles, fv.ivnum,
                                                              (uint64_t) frag->oe.entries, (const float*) cb, nhub, next,
                                                              cfg.pr_delta, eng.ctrl);
        GL_COUNT_LAUNCH();
        GL_CUDA(cudaGetLastError());
      } else if (frag->oe_ntiles) {
        OpPrPull<CT> op{cb, next, cfg.pr_delta};
        int grid = (int) std::min<uint32_t>((uint32_t) gd, frag->oe_ntiles);
        GL_LAUNCH(k_dense_pull<OpPrPull<CT>>, grid, kTB, s, fv.oe_rp, col_p ? col_p : fv.oe_col, (const void*) nullptr,
                  frag->oe_tile_row, frag->oe_ntiles, fv.ivnum, (uint64_t) frag->oe.entries, op, eng.ctrl);
      }
    }
    return GL_OK;
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    if (fv.fnum > 1) {
      MsgView mv = mm.view();
      PrApply ap{rank};
      GL_LAUNCH((k_unpack<ItemU32F64, PrApply>), eng.sm_count * 4, kTB, s, mv, ap, eng.ctrl);
    }
    if (fv.directed && curr_iter > 0 && fv.ivnum)
      GL_LAUNCH(k_pr_fix_dangling, (fv.ivnum + 255) / 256, 256, s, rank, fv.oe_rp, fv.ivnum, last_base);
    if (curr_iter++ >= cfg.max_round) return GL_OK;
    mm.ForceContinue();
    GL_TRY(eng.reset_ctrl());
    // dangling mass (pagerank.h:183-193)
    double dangling = 0;
    GL_CUDA(cudaMemsetAsync(d_dangling, 0, sizeof(double), s));
    if (fv.ivnum) GL_LAUNCH(k_pr_dangling, eng.sm_count * 4, 256, s, rank, fv.oe_rp, fv.ivnum, d_dangling);
    GL_CUDA(cudaMemcpyAsync(&dangling, d_dangling, sizeof(double), cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    GL_TRY(mm.AllReduceF64(&dangling, 1, 0));
    const double N = (double) fv.total_vnum;
    const double base = (1.0 - cfg.pr_delta) / N + cfg.pr_delta * dangling / N;
    last_base = base;
    if (use_pull()) {
      if (cfg.reserved[5] == 1) GL_TRY(pull_sweep<float>(s, base));
      else GL_TRY(pull_sweep<double>(s, base));
    } else {
      if (fv.ivnum) GL_LAUNCH(k_pr_base, (fv.ivnum + 255) / 256, 256, s, next, fv.ivnum, base);
      // (an L2 persistence window over `next` was measured to HURT the atomic push: 7.0 -> 9.6 ms per round)
      OpPrPush op{rank, next, fv.oe_rp, cfg.pr_delta};
      EdgeRange er{fv.oe_rp, fv.oe_col, nullptr};
      GL_TRY(run_frontier_scan(eng, all_inner, fv.ivnum, er, op));
      if (fv.fnum > 1) {
        MsgView mv = mm.view();
        GL_LAUNCH(k_pr_send, eng.sm_count * 4, kTB, s, next, fv.ivnum, fv.ovnum, fv.ovgid, mv);
      }
    }
    GL_TRY(eng.fetch_ctrl());
    note_step(eng.h_ctrl->scanned, fv.ivnum, 2);
    q_touched += fv.ivnum;
    std::swap(rank, next);
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    l2_persist_clear(eng.stream);
    GL_CUDA(cudaMemcpyAsync(host_out, rank, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_pagerank() { return new PageRankApp; }

}  // namespace gl
