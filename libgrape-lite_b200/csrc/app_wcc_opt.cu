// app_wcc_opt.cu — weakly connected components by union-find ("wcc_opt").
//
// The reference's WCCOpt (examples/analytical_apps/cuda/wcc/wcc_opt.h:25-294)
// converts the fragment to COO, hooks the higher root under the lower one with
// atomicCAS (:150-172), compresses paths (:174-184), keeps a parents array of
// the WHOLE graph on every fragment and funnels (offset, parent) pairs to
// fragment 0 (:187-199, :228-247), which alone writes the result.
//
// Re-design
//  * hook/compress run on the CSR that is already resident (no COO copy);
//  * neighbour sampling (Sutton et al., "Afforest"): two rounds hook every
//    vertex to its first / second neighbour; after a compress the giant
//    component is identified from 1024 samples and ONLY vertices outside it
//    scan the rest of their row (on a symmetric adjacency an edge between the
//    giant component and the rest is seen from the other endpoint).  On
//    R-MAT-24 this skips > 99 % of the 5.4e8 CSR entries;
//  * several fragments: every fragment contracts its LOCAL components (inner
//    vertices + outer copies) first; afterwards only component labels cross the
//    cut: an outer copy whose component label improved reports it to its owner
//    ((lid, label) items over the NVLink landing slots, like wcc.h:200-218), the
//    owner folds it into its own component's label.  A round costs O(outer
//    copies + items), not O(edges), and every fragment returns the labels of its
//    own inner vertices (no funnel through fragment 0).
//
// Result: int64 per inner vertex = oid of the minimum-gid vertex of its
// component — identical to the "wcc" app (and to the CPU app's min-oid label with
// the order-preserving partitioner), hence bit-exact against the same oracle.
#include "apps_common.cuh"

namespace gl {
namespace {

// parent pointers only ever move from "root" to an ancestor with a smaller
// index, so a stale (L1) read is still an ancestor-or-self: finds stay correct,
// and a stale "is root" belief is caught by the CAS, which reads L2.
GL_DEV uint32_t uf_find(uint32_t* par, uint32_t x) {
  uint32_t p = par[x];
  while (p != x) {
    const uint32_t gp = par[p];
    if (gp == p) return p;
    par[x] = gp;   // path halving: gp is an ancestor of x
    x = gp;
    p = par[x];
  }
  return x;
}
GL_DEV void uf_hook(uint32_t* par, uint32_t a, uint32_t b) {
  uint32_t ra = uf_find(par, a), rb = uf_find(par, b);
  while (ra != rb) {
    const uint32_t hi = ra > rb ? ra : rb, lo = ra ^ rb ^ hi;
    const uint32_t old = atomicCAS(par + hi, hi, lo);   // wcc_opt.h:163 (HookHighToLowAtomic)
    if (old == hi) return;
    ra = uf_find(par, old);
    rb = uf_find(par, lo);
  }
}

__global__ void k_uf_init(uint32_t* par, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) par[i] = i;
}

// sampling round r: hook every inner vertex to its r-th neighbour
__global__ void __launch_bounds__(256)
k_uf_sample_round(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint32_t ivnum,
                  uint32_t r, uint32_t* par) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < ivnum; v += gridDim.x * blockDim.x) {
    const uint64_t b = rp[v], e = rp[v + 1];
    if (b + r < e) uf_hook(par, v, col[b + r]);
  }
}

// full compression (MultiJumpCompress, wcc_opt.h:174-184)
__global__ void __launch_bounds__(256) k_uf_compress(uint32_t* par, uint32_t n) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    uint32_t p = par[v], pp = par[p];
    while (p != pp) {
      p = pp;
      pp = par[p];
    }
    par[v] = p;
  }
}

// most frequent root among 1024 pseudo-random inner vertices (one CTA)
__global__ void __launch_bounds__(1024) k_uf_giant(const uint32_t* __restrict__ par, uint32_t ivnum, uint32_t* giant) {
  __shared__ uint32_t keys[2048];
  __shared__ uint32_t cnts[2048];
  __shared__ unsigned long long best;
  for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x) {
    keys[i] = 0xFFFFFFFFu;
    cnts[i] = 0;
  }
  if (threadIdx.x == 0) best = 0;
  __syncthreads();
  if (ivnum) {
    unsigned long long z = (threadIdx.x + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const uint32_t r = par[(uint32_t) (z % ivnum)];
    uint32_t h = (r * 2654435761u) >> 21;   // 11 bits
    for (;;) {
      const uint32_t k = atomicCAS(&keys[h], 0xFFFFFFFFu, r);
      if (k == 0xFFFFFFFFu || k == r) {
        atomicAdd(&cnts[h], 1u);
        break;
      }
      h = (h + 1) & 2047;
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x)
    if (cnts[i]) atomicMax(&best, ((unsigned long long) cnts[i] << 32) | (0xFFFFFFFFu - keys[i]));
  __syncthreads();
  if (threadIdx.x == 0) *giant = best ? 0xFFFFFFFFu - (uint32_t) best : 0xFFFFFFFFu;
}

// vertices that still have unseen row entries: outside the giant component
// (or everybody when the adjacency is not symmetric), degree > sampled rounds
__global__ void k_uf_rest_bitmap(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ par,
                                 const uint32_t* __restrict__ giant, uint32_t ivnum, uint32_t sampled,
                                 int can_skip, uint32_t* bm, uint32_t words) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool on = false;
  if (i < ivnum) {
    const uint64_t dg = rp[i + 1] - rp[i];
    on = dg > sampled && !(can_skip && par[i] == *giant);
  }
  const uint32_t w = __ballot_sync(0xffffffffu, on);
  if ((threadIdx.x & 31) == 0 && (i >> 5) < words) bm[i >> 5] = w;
}
// (directed graphs, incoming adjacency: every non-giant vertex with in-edges)
__global__ void k_uf_rest_bitmap_in(const uint64_t* __restrict__ irp, const uint32_t* __restrict__ par,
                                    const uint32_t* __restrict__ giant, uint32_t ivnum, int can_skip,
                                    uint32_t* bm, uint32_t words) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool on = false;
  if (i < ivnum) on = irp[i + 1] > irp[i] && !(can_skip && par[i] == *giant);
  const uint32_t w = __ballot_sync(0xffffffffu, on);
  if ((threadIdx.x & 31) == 0 && (i >> 5) < words) bm[i >> 5] = w;
}

// Outer copies have no row of their own: the edges (u, g) of a giant-component
// vertex u are skipped, so every outer copy g looks for ONE inner neighbour in
// the giant component through its reverse adjacency (ovie) and hooks to it;
// edges to vertices outside the giant component are hooked from their side.
__global__ void __launch_bounds__(256)
k_uf_attach_outer(const uint64_t* __restrict__ orp, const uint32_t* __restrict__ ocol, uint32_t ivnum,
                  uint32_t ovnum, const uint32_t* __restrict__ giant, uint32_t* par) {
  const uint32_t gi = *giant;
  for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < ovnum; o += gridDim.x * blockDim.x) {
    const uint64_t b = orp[o], e = orp[o + 1];
    for (uint64_t p = b; p < e; ++p) {
      const uint32_t u = ocol[p];
      if (par[u] == gi) {   // (par is compressed: a stale value only costs a later candidate)
        uf_hook(par, ivnum + o, u);
        break;
      }
    }
  }
}

struct OpUfHook {
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* par;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  GL_DEV void edge(uint32_t u, Meta, uint32_t v, W, ScanAcc& acc) const {
    if (u != v) uf_hook(par, u, v);
    acc.touched++;
  }
};

// clabel[root] = min gid over the local component
__global__ void k_uf_labels_init(uint32_t* clabel, uint32_t ivnum, uint32_t ovnum, const uint32_t* ovgid,
                                 uint32_t fid, int fid_offset) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum) clabel[i] = (fid << fid_offset) | i;
  else if (i < ivnum + ovnum) clabel[i] = ovgid[i - ivnum];
}
// The root is the member with the smallest local index, i.e. the smallest gid
// among the INNER members; only outer copies (gids of other fragments) can
// lower the label.  The plain pre-check keeps the atomics off the hot word of
// the giant component (16 M atomicMin on one address cost 5 ms).
__global__ void k_uf_labels_fold(const uint32_t* __restrict__ par, uint32_t* clabel, uint32_t ivnum, uint32_t tvnum) {
  const uint32_t i = ivnum + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tvnum) return;
  const uint32_t r = par[i];
  if (r == i) return;
  const uint32_t g = clabel[i];   // clabel[i] of a non-root is still its own gid here
  if (g < __ldcg(clabel + r)) atomicMin(clabel + r, g);
}

// an outer copy whose component label is better than what its owner was told
__global__ void k_uf_mark_outer(const uint32_t* __restrict__ par, const uint32_t* __restrict__ clabel,
                                uint32_t* sent, uint32_t ivnum, uint32_t ovnum, uint32_t* remote) {
  const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= ovnum) return;
  const uint32_t v = ivnum + o;
  const uint32_t l = clabel[par[v]];
  if (l < sent[o]) {
    sent[o] = l;
    bit_set_atomic(remote, v);
  }
}
struct UfPayload {
  const uint32_t* sent;
  uint32_t ivnum;
  GL_DEV ItemU32U32 operator()(uint32_t v, uint32_t lid) const { return ItemU32U32{lid, sent[v - ivnum]}; }
};
struct UfApply {
  const uint32_t* par;
  uint32_t* clabel;
  GL_DEV void operator()(const ItemU32U32& it, ScanAcc& acc) const {
    const uint32_t r = par[it.lid];
    if (!(it.val < __ldcg(clabel + r))) return;   // keep failing atomics off the giant component's word
    if (it.val < atomicMin(clabel + r, it.val)) acc.aux++;
  }
};

__global__ void k_uf_out(const uint32_t* par, const uint32_t* clabel, uint32_t n, LabelMap lm, int64_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = lm.oid(clabel[par[i]]);
}

struct WccOptApp : gl_app {
  DevBuf<uint32_t> par, clabel, sent, rest, remote, d_giant;
  DevBuf<int64_t> out64;
  uint32_t tvnum = 0;
  size_t words = 0;
  static constexpr uint32_t kSampled = 2;

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
    GL_CUDA(par.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(clabel.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(sent.alloc(std::max<uint32_t>(fv.ovnum, 1)));
    GL_CUDA(rest.alloc(words));
    GL_CUDA(remote.alloc(words));
    GL_CUDA(d_giant.alloc(1));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    return mm.Init(comm, fv, sizeof(ItemU32U32));
  }

  int Init() override {
    GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, eng.stream));
    return GL_OK;
  }

  // one engine scan over `er` of the vertices in `rest`
  int scan_rest(EdgeRange er) {
    GL_TRY(eng.reset_ctrl());
    OpUfHook op{par};
    GL_TRY(run_frontier_scan(eng, rest, fv.ivnum, er, op));
    GL_TRY(eng.fetch_ctrl());
    note_step(eng.h_ctrl->scanned, (uint32_t) std::min<uint64_t>(eng.h_ctrl->frontier, 0xFFFFFFFFu), 0);
    return GL_OK;
  }

  // outer copies with a better component label -> their owners
  int report_outer() {
    cudaStream_t s = eng.stream;
    if (fv.ovnum) GL_LAUNCH(k_uf_mark_outer, (fv.ovnum + 255) / 256, 256, s, par, clabel, sent, fv.ivnum, fv.ovnum, remote);
    MsgView mv = mm.view();
    GL_LAUNCH((k_pack_outer<ItemU32U32, UfPayload>), eng.sm_count * 4, kTB, s, remote, fv.ivnum, fv.ovnum, fv.ovgid,
              mv, UfPayload{sent, fv.ivnum}, 1, remote);
    return GL_OK;
  }

  int PEval() override {
    cudaStream_t s = eng.stream;
    const int g256 = eng.sm_count * 8;
    if (tvnum) GL_LAUNCH(k_uf_init, g256, 256, s, par, tvnum);
    const bool has_in = fv.directed && !frag->ie_alias_oe && fv.ie_rp != nullptr;
    // skipping the giant component needs every edge to be visible from both endpoints
    // (several fragments + a separate incoming adjacency: outer copies that are only
    //  reachable through skipped in-rows would be missed, so nothing is skipped)
    const int can_skip = (!fv.directed || frag->ie_alias_oe || (has_in && fv.fnum == 1)) ? 1 : 0;
    if (fv.ivnum) {
      for (uint32_t r = 0; r < kSampled; ++r)
        GL_LAUNCH(k_uf_sample_round, g256, 256, s, fv.oe_rp, fv.oe_col, fv.ivnum, r, par);
      GL_LAUNCH(k_uf_compress, g256, 256, s, par, tvnum);
      GL_LAUNCH(k_uf_giant, 1, 1024, s, par, fv.ivnum, d_giant);
      const uint32_t nb = (uint32_t) ((std::max<size_t>(fv.ivnum, (words - 1) * 32) + 255) / 256);
      GL_CUDA(cudaMemsetAsync(rest, 0, sizeof(uint32_t) * words, s));
      GL_LAUNCH(k_uf_rest_bitmap, nb, 256, s, fv.oe_rp, par, d_giant, fv.ivnum, kSampled, can_skip, rest, (uint32_t) words);
      if (can_skip && fv.ovnum && fv.ovie_rp)
        GL_LAUNCH(k_uf_attach_outer, g256, 256, s, fv.ovie_rp, fv.ovie_col, fv.ivnum, fv.ovnum, d_giant, par);
      GL_TRY(scan_rest(EdgeRange{fv.oe_rp, fv.oe_col, nullptr}));
      if (has_in) {
        // incoming adjacency of the vertices outside the giant component (wcc.h:181-197)
        GL_CUDA(cudaMemsetAsync(rest, 0, sizeof(uint32_t) * words, s));
        GL_LAUNCH(k_uf_rest_bitmap_in, nb, 256, s, fv.ie_rp, par, d_giant, fv.ivnum, can_skip, rest, (uint32_t) words);
        GL_TRY(scan_rest(EdgeRange{fv.ie_rp, fv.ie_col, nullptr}));
      }
    }
    if (tvnum) {
      GL_LAUNCH(k_uf_compress, g256, 256, s, par, tvnum);
      GL_LAUNCH(k_uf_labels_init, (tvnum + 255) / 256, 256, s, clabel, fv.ivnum, fv.ovnum, fv.ovgid, fv.fid, fv.fid_offset);
      if (fv.ovnum) GL_LAUNCH(k_uf_labels_fold, (fv.ovnum + 255) / 256, 256, s, par, clabel, fv.ivnum, tvnum);
    }
    q_touched += fv.ivnum;
    peval_entries = q_entries + (uint64_t) kSampled * fv.ivnum;
    if (fv.fnum > 1) {
      // the owner knows its own gid: that is what every outer copy has "sent" so far
      if (fv.ovnum) GL_CUDA(cudaMemcpyAsync(sent, fv.ovgid, sizeof(uint32_t) * fv.ovnum, cudaMemcpyDeviceToDevice, s));
      GL_TRY(report_outer());
      mm.ForceContinue();   // every fragment runs at least one exchange round
    }
    return GL_OK;
  }

  // only on several fragments: fold received labels, report improvements
  int IncEval() override {
    cudaStream_t s = eng.stream;
    GL_TRY(eng.reset_ctrl());
    MsgView mv = mm.view();
    GL_LAUNCH((k_unpack<ItemU32U32, UfApply>), eng.sm_count * 4, kTB, s, mv, UfApply{par, clabel}, eng.ctrl);
    GL_TRY(report_outer());
    GL_TRY(eng.fetch_ctrl());
    note_step(0, (uint32_t) std::min<uint64_t>(eng.h_ctrl->aux, 0xFFFFFFFFu), 0);
    // (items sent this round keep the query alive through the round vote)
    return GL_OK;
  }

  // the whole contraction happens in PEval (step 0): CSR entries it looked at
  void FillStats(gl_query_stats* st) override {
    if (st->n_steps < 1) return;
    st->step_entries[0] = peval_entries;
    st->step_frontier[0] = fv.ivnum;
    st->entries_scanned = peval_entries;
  }
  uint64_t peval_entries = 0;

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_LAUNCH(k_uf_out, (fv.ivnum + 255) / 256, 256, eng.stream, par, clabel, fv.ivnum, label_map(*this), out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(int64_t) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_wcc_opt() { return new WccOptApp; }

}  // namespace gl
