// app_kclique.cu — k-clique counting (examples/analytical_apps/kclique/, run_app --application kclique
// --kclique_k K).
//
// Result: the number of k-cliques of the SIMPLE graph underneath the fragment group (self loops
// ignored, a pair joined by several CSR entries is one edge), summed in uint64 (wraps modulo 2^64, like
// the reference's size_t), the same value on every rank.  On a simple graph this is what the reference
// prints; on a multigraph the reference weights cliques by edge multiplicities in an order that depends
// on the fragment count, and this library deliberately does not.
//
// Re-design (the reference walks a depth-first search per vertex through std::set and a byte table,
// kclique_utils.h):
//   1. DAG: every simple edge is oriented from the lower to the higher (degree, gid), degree = CSR row
//      length; rows hold gids, sorted and unique.  A k-clique is counted once, at its lowest vertex v,
//      through the oriented edge (v, u) to its second-lowest vertex u: the other k - 2 vertices form a
//      (k-2)-clique of the DAG induced on I = N+(v) ∩ N+(u).
//   2. k = 3: one warp per oriented edge adds |I|.
//   3. k >= 4: the same warp pass computes s = |I| and picks a tier from s alone:
//        (a) s <= kKcWarpMax: the warp builds the induced DAG on I as 32 one-word rows in its slice of
//            shared memory and its lanes walk the first level in parallel;
//        (b) s <= kKcCtaMax: one CTA builds an s x 1024-bit matrix (one 32-bit word per lane and row)
//            in shared memory; its warps split the first level and walk candidate bitmaps depth-first;
//        (c) larger s: one CTA walks sorted candidate arrays depth-first in a global scratch of
//            (k - 2) x (longest DAG row) entries and hands every sub-problem of at most kKcCtaMax
//            vertices to the code of (b).
//      A branch is pruned when its candidate set is smaller than the number of vertices still needed.
//   4. fnum > 1: degrees of the outer copies come from the dense mirror sync; every fragment builds the
//      rows of its inner vertices and replicates the peers' rows (PeerCsr); a fragment counts the
//      cliques whose lowest vertex is one of its inner vertices; one peer all-reduce sums the counts.
#include <cstring>

#include "dag_common.cuh"

namespace gl {
namespace {

constexpr int kKcWarpMax = 32;     // tier (a): one 32-bit row per candidate
constexpr int kKcCtaMax = 1024;    // tier (b): one 32-bit word per lane and row, 128 KB of rows
constexpr int kKcWarps = kTB / 32;
static_assert(GL_KCLIQUE_MAX_K >= 4, "");

// DFS stack levels per walker: a walk that still needs nd <= k - 3 vertices pushes while nd - d - 1 >= 2
__host__ __device__ inline int kc_levels(int k) { return k > 5 ? k - 4 : 1; }   // max(k - 4, 1)

// dynamic shared memory of the two kernels (32-bit words)
__host__ __device__ inline size_t kc_warp_smem_words(int k) { return (size_t) kKcWarps * 32 * (2 + 2 * kc_levels(k)); }
__host__ __device__ inline size_t kc_cta_smem_words(int k) {
  return (size_t) kKcCtaMax * 32 + kKcCtaMax + (size_t) kKcWarps * 64 * kc_levels(k) + kKcWarps + 2 * GL_KCLIQUE_MAX_K;
}

struct KcCtl {
  unsigned long long total;     // cliques found by this fragment
  unsigned long long scanned;   // DAG entries iterated by the intersections
  unsigned long long tier_a;    // items counted by tier (a)
  unsigned int q_b, q_c;        // items queued for tier (b) (from the front) and (c) (from the back)
  unsigned int max_row;         // longest DAG row of this fragment
  unsigned int max_s;           // largest |I|
};

// the DAG rows of the whole group, by gid
struct Dag {
  const uint64_t* const* rp;
  const uint32_t* const* key;
  int fid_offset;
  uint32_t id_mask;
  GL_DEV const uint32_t* row(uint32_t g, uint32_t* n) const {
    const uint64_t* r = rp[g >> fid_offset];
    const uint32_t l = g & id_mask;
    const uint64_t b = r[l];
    *n = (uint32_t) (r[l + 1] - b);
    return key[g >> fid_offset] + b;
  }
};

GL_DEV uint32_t lower_bound(const uint32_t* a, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
GL_DEV bool contains(const uint32_t* a, uint32_t n, uint32_t x) {
  const uint32_t p = lower_bound(a, n, x);
  return p < n && a[p] == x;
}

// v -> u is kept when v ranks below u; a self loop and all but the first copy of a multi-edge are dropped
struct KcKeep {
  GL_DEV bool operator()(const uint32_t* col, uint64_t b, uint64_t p, uint32_t v, uint32_t u, uint32_t dv,
                         uint32_t du, uint32_t gv, uint32_t gu) const {
    return u != v && (p == b || col[p - 1] != u) && (dv < du || (dv == du && gv < gu));
  }
};

struct KcArgs {
  Dag dag;
  const uint64_t* orp;     // this fragment's rows (inner lids)
  const uint32_t* okey;
  const uint32_t* osrc;
  uint64_t om;
  int k;
  uint32_t* queue;         // tier (b) items from the front, tier (c) items from the back
  uint64_t qcap;
  uint32_t* scratch;       // tier (c): per CTA, (k - 2) lists of `stride` entries
  uint32_t stride;
  KcCtl* ctl;
};

// Number of nd-cliques (nd >= 1) of the DAG `row` (one-word rows) inside `cand`, walked by one lane;
// so / sr: this lane's stack of (candidate set, not yet tried) words, stride 32.
GL_DEV unsigned long long lane_count(uint32_t cand, int nd, const uint32_t* row, uint32_t* so, uint32_t* sr) {
  if (nd == 1) return __popc(cand);
  if (__popc(cand) < nd) return 0;
  unsigned long long tot = 0;
  int d = 0;
  uint32_t orig = cand, rem = cand;
  while (true) {
    if (rem == 0) {
      if (d == 0) break;
      --d;
      orig = so[d * 32];
      rem = sr[d * 32];
      continue;
    }
    const int j = __ffs(rem) - 1;
    rem &= rem - 1;
    const uint32_t nc = orig & row[j];
    const int need = nd - d - 1;
    if (need == 1) {
      tot += __popc(nc);
      continue;
    }
    if (__popc(nc) < need) continue;
    so[d * 32] = orig;
    sr[d * 32] = rem;
    ++d;
    orig = rem = nc;
  }
  return tot;
}

// The same walk by a whole warp over bitmaps of up to 1024 bits: lane l holds word l of every set, and
// row j of the matrix is rows[j * 32 .. j * 32 + 32).  Every lane returns the count.
GL_DEV unsigned long long warp_count(uint32_t cand, int nd, const uint32_t* rows, uint32_t* so, uint32_t* sr) {
  const uint32_t lane = lane_id();
  const uint32_t c0 = warp_sum((uint32_t) __popc(cand));
  if (nd == 1) return c0;
  if (c0 < (uint32_t) nd) return 0;
  unsigned long long tot = 0;
  int d = 0;
  uint32_t orig = cand, rem = cand;
  while (true) {
    const uint32_t any = __ballot_sync(0xffffffffu, rem != 0);
    if (!any) {
      if (d == 0) break;
      --d;
      orig = so[d * 32 + lane];
      rem = sr[d * 32 + lane];
      continue;
    }
    const int ln = __ffs(any) - 1;
    const uint32_t wv = __shfl_sync(0xffffffffu, rem, ln);
    const int j = ln * 32 + __ffs(wv) - 1;
    if ((int) lane == ln) rem &= rem - 1;
    const uint32_t nc = orig & rows[j * 32 + lane];
    const int need = nd - d - 1;
    const uint32_t c = warp_sum((uint32_t) __popc(nc));
    if (need == 1) {
      tot += c;
      continue;
    }
    if (c < (uint32_t) need) continue;
    so[d * 32 + lane] = orig;
    sr[d * 32 + lane] = rem;
    ++d;
    orig = rem = nc;
  }
  return tot;
}

// k = 3: sum of |I|.  k >= 4: tier (a) inline, tiers (b) / (c) queued.  One warp per oriented edge.
__global__ void __launch_bounds__(kTB) k_kc_edges(KcArgs a) {
  extern __shared__ uint32_t smem[];
  const uint32_t lane = lane_id(), wib = threadIdx.x >> 5;
  uint32_t* I = smem + (size_t) wib * 32 * (2 + 2 * kc_levels(a.k));
  uint32_t* row = I + 32;
  uint32_t* so = row + 32 + lane;
  uint32_t* sr = so + 32 * kc_levels(a.k);
  const uint64_t warps = ((uint64_t) gridDim.x * blockDim.x) >> 5;
  const int r = a.k - 2;   // vertices to pick inside I
  unsigned long long tot = 0, scanned = 0, tier_a = 0;
  uint32_t max_s = 0;
  for (uint64_t ei = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; ei < a.om; ei += warps) {
    const uint32_t v = a.osrc[ei];
    const uint64_t vb = a.orp[v];
    const uint32_t* A = a.okey + vb;
    uint32_t na = (uint32_t) (a.orp[v + 1] - vb), nb;
    const uint32_t* B = a.dag.row(a.okey[ei], &nb);
    // iterate the shorter row, search the longer one; I comes out sorted by gid
    if (nb < na) {
      const uint32_t* t = A; A = B; B = t;
      const uint32_t tn = na; na = nb; nb = tn;
    }
    uint32_t s = 0;
    for (uint32_t p0 = 0; p0 < na; p0 += 32) {
      const uint32_t p = p0 + lane;
      uint32_t x = 0;
      const bool f = p < na && contains(B, nb, x = A[p]);
      const uint32_t m = __ballot_sync(0xffffffffu, f);
      if (f) {
        const uint32_t at = s + __popc(m & ((1u << lane) - 1));
        if (at < kKcWarpMax) I[at] = x;
      }
      s += __popc(m);
    }
    scanned += na;
    max_s = max(max_s, s);
    if (r == 1) {
      if (lane == 0) tot += s;
      continue;
    }
    if (s < (uint32_t) r) continue;
    if (s > kKcWarpMax) {
      if (lane == 0) {
        if (s <= kKcCtaMax) a.queue[atomicAdd(&a.ctl->q_b, 1u)] = (uint32_t) ei;
        else a.queue[a.qcap - 1 - atomicAdd(&a.ctl->q_c, 1u)] = (uint32_t) ei;
      }
      continue;
    }
    // tier (a): row i = the members of I in N+(I[i]), one binary search per lane
    __syncwarp();
    const uint32_t mine = lane < s ? I[lane] : 0;
    for (uint32_t i = 0; i < s; ++i) {
      uint32_t nw;
      const uint32_t* W = a.dag.row(I[i], &nw);
      const uint32_t bits = __ballot_sync(0xffffffffu, lane < s && contains(W, nw, mine));
      if (lane == 0) row[i] = bits;
    }
    scanned += s;
    __syncwarp();
    if (lane < s) tot += lane_count(row[lane], r - 1, row, so, sr);
    ++tier_a;
    __syncwarp();
  }
  tot = warp_sum(tot);
  max_s = __reduce_max_sync(0xffffffffu, max_s);
  if (lane == 0) {
    if (tot) atomicAdd(&a.ctl->total, tot);
    if (scanned) atomicAdd(&a.ctl->scanned, scanned);
    if (tier_a) atomicAdd(&a.ctl->tier_a, tier_a);
    if (max_s) atomicMax(&a.ctl->max_s, max_s);
  }
}

struct CtaSmem {
  uint32_t* rows;   // [kKcCtaMax][32]
  uint32_t* L;      // [kKcCtaMax]
  uint32_t* stk;    // [warps][2][levels][32]
  uint32_t* wcnt;   // [warps]
  uint32_t* pos;    // [GL_KCLIQUE_MAX_K]
  uint32_t* len;    // [GL_KCLIQUE_MAX_K]
};

// out = A ∩ B in ascending order (both sorted); every thread returns the size.  Ends with a barrier.
GL_DEV uint32_t cta_intersect(const uint32_t* A, uint32_t na, const uint32_t* B, uint32_t nb, uint32_t* out,
                              const CtaSmem& sm, unsigned long long* scanned) {
  if (nb < na) {
    const uint32_t* t = A; A = B; B = t;
    const uint32_t tn = na; na = nb; nb = tn;
  }
  const uint32_t lane = lane_id(), wib = threadIdx.x >> 5;
  uint32_t base = 0;
  for (uint32_t p0 = 0; p0 < na; p0 += kTB) {
    const uint32_t p = p0 + threadIdx.x;
    uint32_t x = 0;
    const bool f = p < na && contains(B, nb, x = A[p]);
    const uint32_t m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) sm.wcnt[wib] = __popc(m);
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (uint32_t w = 0; w < kKcWarps; ++w) {
      const uint32_t c = sm.wcnt[w];
      before += w < wib ? c : 0;
      all += c;
    }
    if (f) out[base + before + __popc(m & ((1u << lane) - 1))] = x;
    base += all;
    __syncthreads();
  }
  if (threadIdx.x == 0) *scanned += na;
  __syncthreads();
  return base;
}

// r-cliques (r >= 2) of the DAG induced on the sorted list L of n <= kKcCtaMax gids; every lane returns
// its warp's share.  Ends with a barrier.
GL_DEV unsigned long long cta_bitmap_count(const uint32_t* L, uint32_t n, int r, const Dag& dag, const CtaSmem& sm,
                                           int levels, unsigned long long* scanned) {
  const uint32_t lane = lane_id(), wib = threadIdx.x >> 5;
  for (uint32_t t = threadIdx.x; t < n; t += kTB) sm.L[t] = L[t];
  for (uint32_t t = threadIdx.x; t < n * 32; t += kTB) sm.rows[t] = 0;
  __syncthreads();
  for (uint32_t i = wib; i < n; i += kKcWarps) {
    uint32_t nw;
    const uint32_t* W = dag.row(sm.L[i], &nw);
    for (uint32_t p = lane; p < nw; p += 32) {
      const uint32_t x = W[p];
      const uint32_t j = lower_bound(sm.L, n, x);
      if (j < n && sm.L[j] == x) atomicOr(&sm.rows[i * 32 + (j >> 5)], 1u << (j & 31));
    }
    if (lane == 0) *scanned += nw;
  }
  __syncthreads();
  uint32_t* so = sm.stk + (size_t) wib * 64 * levels;
  uint32_t* sr = so + 32 * levels;
  unsigned long long tot = 0;
  for (uint32_t i = wib; i < n; i += kKcWarps) tot += warp_count(sm.rows[i * 32 + lane], r - 1, sm.rows, so, sr);
  __syncthreads();
  return tot;
}

// tiers (b) and (c): one CTA per queued item
__global__ void __launch_bounds__(kTB, 1) k_kc_cta(KcArgs a, uint32_t n_b, uint32_t n_c) {
  extern __shared__ uint32_t smem[];
  const int levels = kc_levels(a.k);
  CtaSmem sm;
  sm.rows = smem;
  sm.L = sm.rows + (size_t) kKcCtaMax * 32;
  sm.stk = sm.L + kKcCtaMax;
  sm.wcnt = sm.stk + (size_t) kKcWarps * 64 * levels;
  sm.pos = sm.wcnt + kKcWarps;
  sm.len = sm.pos + GL_KCLIQUE_MAX_K;
  const int r0 = a.k - 2;
  uint32_t* scratch = a.scratch + (size_t) blockIdx.x * r0 * a.stride;
  unsigned long long tot = 0, scanned = 0;
  for (uint32_t t = blockIdx.x; t < n_b + n_c; t += gridDim.x) {
    const uint64_t ei = t < n_b ? a.queue[t] : a.queue[a.qcap - 1 - (t - n_b)];
    const uint32_t v = a.osrc[ei];
    uint32_t nb;
    const uint32_t* B = a.dag.row(a.okey[ei], &nb);
    const uint32_t n0 = cta_intersect(a.okey + a.orp[v], (uint32_t) (a.orp[v + 1] - a.orp[v]), B, nb, scratch, sm,
                                      &scanned);
    if (n0 <= kKcCtaMax) {
      tot += cta_bitmap_count(scratch, n0, r0, a.dag, sm, levels, &scanned);
      continue;
    }
    // tier (c): depth-first over sorted lists; list d lives at scratch + d * stride
    if (threadIdx.x == 0) {
      sm.len[0] = n0;
      sm.pos[0] = 0;
    }
    __syncthreads();
    int d = 0;
    while (d >= 0) {
      const uint32_t p = sm.pos[d], n = sm.len[d];
      if (p == n) {
        --d;
        continue;
      }
      __syncthreads();   // everybody has read pos[d]
      if (threadIdx.x == 0) sm.pos[d] = p + 1;
      const uint32_t* Ld = scratch + (size_t) d * a.stride;
      uint32_t* Ln = scratch + (size_t) (d + 1) * a.stride;
      uint32_t nw;
      const uint32_t* W = a.dag.row(Ld[p], &nw);
      const uint32_t nn = cta_intersect(Ld, n, W, nw, Ln, sm, &scanned);
      const int need = r0 - d - 1;
      if (need == 1) {
        if (threadIdx.x == 0) tot += nn;
        continue;
      }
      if (nn < (uint32_t) need) continue;
      if (nn <= kKcCtaMax) {
        tot += cta_bitmap_count(Ln, nn, need, a.dag, sm, levels, &scanned);
        continue;
      }
      if (threadIdx.x == 0) {
        sm.len[d + 1] = nn;
        sm.pos[d + 1] = 0;
      }
      __syncthreads();
      ++d;
    }
    __syncthreads();
  }
  // tot: thread 0 holds the list-level counts, lane 0 of every warp its warp's bitmap counts
  if (lane_id() == 0) {
    if (tot) atomicAdd(&a.ctl->total, tot);
    if (scanned) atomicAdd(&a.ctl->scanned, scanned);
  }
}

struct KCliqueApp : gl_app {
  int k = 0;
  DevBuf<uint32_t> deg, okey, osrc, queue, scratch;
  DevBuf<uint64_t> cnt, orp;
  DevBuf<KcCtl> d_ctl;
  PinnedBuf<KcCtl> h_ctl;
  PeerCsr dag;
  uint64_t om = 0;
  size_t scratch_words = 0;
  int64_t result = 0;
  KcCtl last{};
  int cta_grid = 0;

  size_t ResultElemBytes() const override { return sizeof(int64_t); }
  size_t ResultCount() const override { return 1; }

  int Setup() override {
    // the reference app loads kOnlyOut and "can work on undirected graph"
    if (fv.directed) {
      set_error("kclique needs an undirected fragment");
      return GL_ERR_ARG;
    }
    k = cfg.max_round;
    if (k < 3 || k > GL_KCLIQUE_MAX_K) {
      set_error("kclique: k = %d is outside [3, %d] (k travels in gl_app_config.max_round)", k, GL_KCLIQUE_MAX_K);
      return GL_ERR_ARG;
    }
    const uint32_t tvnum = fv.ivnum + fv.ovnum;
    GL_CUDA(deg.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(cnt.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(orp.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(d_ctl.alloc(1));
    GL_CUDA(h_ctl.alloc(1));
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32I64)));
    if (fv.fnum > 1) GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
    // the attribute belongs to the kernel, not to this app: every app sets the bound of the largest k, so
    // apps with different k can live side by side
    GL_CUDA(cudaFuncSetAttribute(k_kc_edges, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int) (4 * kc_warp_smem_words(GL_KCLIQUE_MAX_K))));
    GL_CUDA(cudaFuncSetAttribute(k_kc_cta, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int) (4 * kc_cta_smem_words(GL_KCLIQUE_MAX_K))));
    return GL_OK;
  }

  int Init() override { return GL_OK; }

  int fetch(KcCtl* out) {
    GL_CUDA(cudaMemcpyAsync(h_ctl, d_ctl, sizeof(KcCtl), cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    *out = *h_ctl;
    return GL_OK;
  }

  // the degree-ordered DAG of this fragment's inner vertices, rows of gids sorted and unique
  int build_dag() {
    cudaStream_t s = eng.stream;
    const GidOf gid{fv.ivnum, fv.fid, fv.fid_offset, fv.ovgid};
    if (fv.ivnum) GL_LAUNCH(k_row_length<uint32_t>, (fv.ivnum + 255) / 256, 256, s, fv.oe_rp, fv.ivnum, deg.get());
    if (fv.fnum > 1) GL_TRY(mm.SyncValuesToGhosts(s, deg, 4));
    GL_LAUNCH(k_dag_count<KcKeep>, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, KcKeep{}, cnt,
              &d_ctl.get()->max_row);
    uint64_t total = 0;
    GL_TRY(dag_scan(s, cnt, orp, fv.ivnum, &total));
    // every rank takes the same decision, so no rank is left waiting in the next collective
    long long most = (long long) total, unused = 0;
    double unused_d = 0;
    if (fv.fnum > 1) GL_TRY(mm.PeerAllReduce(s, &most, &unused, &unused_d, 2));
    if ((unsigned long long) most > 0xFFFFFFFFull) {
      set_error("kclique: %llu oriented edges in one fragment of the group; at most 2^32 - 1 are supported",
                (unsigned long long) most);
      return GL_ERR_ARG;
    }
    if (total != om || !okey) {
      okey.reset();
      osrc.reset();
      queue.reset();
      om = total;
      GL_CUDA(okey.alloc(std::max<uint64_t>(om, 4)));
      GL_CUDA(osrc.alloc(std::max<uint64_t>(om, 4)));
      GL_CUDA(queue.alloc(std::max<uint64_t>(om, 4)));
    }
    if (fv.ivnum && om) {
      GL_LAUNCH(k_dag_fill<KcKeep>, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, KcKeep{}, orp,
                okey, nullptr, osrc);
      // several fragments: outer gids do not follow lid order
      if (fv.fnum > 1) GL_TRY(sort_csr_rows(s, orp, fv.ivnum, om, &okey));
    }
    return dag.replicate(mm, s, fv, orp, okey, om);
  }

  int PEval() override {
    cudaStream_t s = eng.stream;
    GL_CUDA(cudaMemsetAsync(d_ctl, 0, sizeof(KcCtl), s));
    GL_TRY(build_dag());
    KcArgs a;
    a.dag = Dag{dag.d_rp, dag.d_col, fv.fid_offset, fv.id_mask};
    a.orp = orp;
    a.okey = okey;
    a.osrc = osrc;
    a.om = om;
    a.k = k;
    a.queue = queue;
    a.qcap = std::max<uint64_t>(om, 4);
    a.scratch = nullptr;
    a.stride = 0;
    a.ctl = d_ctl;
    if (om) {
      k_kc_edges<<<eng.sm_count * 8, kTB, 4 * kc_warp_smem_words(k), s>>>(a);
      GL_COUNT_LAUNCH();
      GL_CUDA(cudaGetLastError());
    }
    KcCtl c;
    GL_TRY(fetch(&c));
    if (c.q_b + c.q_c) {
      const size_t smem = 4 * kc_cta_smem_words(k);
      if (!cta_grid) {
        int per_sm = 0;
        GL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_kc_cta, kTB, smem));
        cta_grid = std::max(per_sm, 1) * eng.sm_count;
      }
      const uint32_t grid = std::min<uint32_t>(c.q_b + c.q_c, (uint32_t) cta_grid);
      a.stride = std::max<uint32_t>(c.max_row, 1);
      const size_t need = (size_t) grid * (k - 2) * a.stride;
      if (need > scratch_words) {
        scratch.reset();
        GL_CUDA(scratch.alloc(need));
        scratch_words = need;
      }
      a.scratch = scratch;
      k_kc_cta<<<grid, kTB, smem, s>>>(a, c.q_b, c.q_c);
      GL_COUNT_LAUNCH();
      GL_CUDA(cudaGetLastError());
      GL_TRY(fetch(&c));
    }
    last = c;
    long long sum = (long long) c.total, unused = 0;
    double unused_d = 0;
    if (fv.fnum > 1) GL_TRY(mm.PeerAllReduce(s, &sum, &unused, &unused_d, 0));
    result = (int64_t) sum;
    q_entries += c.scanned;
    q_frontier += om;
    return GL_OK;   // the query ends with this round
  }

  int IncEval() override { return GL_OK; }

  void FillStats(gl_query_stats* st) override {
    st->step_frontier[0] = last.max_s;
    st->step_frontier[1] = (uint32_t) std::min<unsigned long long>(last.tier_a, 0xFFFFFFFFull);
    st->step_frontier[2] = last.q_b;
    st->step_frontier[3] = last.q_c;
  }

  int Result(void* host_out, size_t) override {
    memcpy(host_out, &result, sizeof(result));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_kclique() { return new KCliqueApp; }

}  // namespace gl
