// app_pagerank_vc.cu — PageRank on a vertex-cut fragment (the reference's PageRankVC, run_app --vc;
// examples/analytical_apps/pagerank/pagerank_vc.h, grape/parallel/gather_scatter_message_manager.h).
//
// Each round is one pull sweep over the fragment's local CSR: next[v] = sum of curr[u] over v's
// entries, where curr already holds rank / degree (the reference's master_result before a scatter).
// The partial sums of a master vertex are then GATHERED to its owner, folded in fid order, turned
// into the new rank / degree and SCATTERED back to every fragment holding the vertex.
//
// Every sum has one fixed order, so the output is bit-identical from run to run (the reference adds
// with f64 atomics in thread order): the row tiers of row_tiers.cuh (a thread, a warp, or chunks
// folded in chunk order by a second kernel).
//
// Gather / scatter (F > 1) are dense peer stores into the communicator's mirror slots: a fragment
// stores the partial-sum slice of every other fragment's master range it holds into that owner's
// slot (parity 0, src = me); a device-side barrier; the owner folds its own partials and the received
// slices in fid order and stores the new values into every holder's slot (parity 1, src = owner);
// a barrier; holders copy the slices into their local copies.  A slice is at most mvc doubles, so the
// slots need mirror_bytes >= 8 * mvc.  The two parities keep a round's scatter from overwriting a
// gather slice that its owner has not folded yet; the next round's gather stores start only after
// every fragment has passed the scatter barrier, i.e. after every fold has read its slices.
#include <cmath>

#include "row_tiers.cuh"
#include "vcfrag.h"

namespace gl {
namespace {

struct VcSlice {
  double* ptr;     // peer slot (put) or my slot (copy-in)
  uint64_t off;    // local id of the slice's first vertex
  uint64_t cnt;
};

struct VcStore {
  double* next;
  GL_DEV void operator()(uint32_t r, double s) const { next[r] = s; }
};

__global__ void __launch_bounds__(kTB)
k_vc_pull(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint32_t nl,
          const double* __restrict__ curr, double* __restrict__ next) {
  VcStore out{next};
  tier_rows(rp, col, nl, curr, out);
}

__global__ void __launch_bounds__(kTB)
k_vc_chunks(const uint64_t* __restrict__ cb, const uint64_t* __restrict__ ce, uint32_t nitems,
            const uint32_t* __restrict__ col, const double* __restrict__ curr, double* __restrict__ csum) {
  tier_chunks(cb, ce, nitems, col, curr, csum);
}

__global__ void k_vc_long(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ off, uint32_t nlong,
                          const double* __restrict__ csum, double* __restrict__ next) {
  VcStore out{next};
  tier_long(rows, off, nlong, csum, out);
}

// dense slices of `src` into peer slots (blockIdx.y = slice)
__global__ void k_vc_put(const double* __restrict__ src, const VcSlice* __restrict__ t) {
  const VcSlice sl = t[blockIdx.y];
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < sl.cnt; i += (uint64_t) gridDim.x * blockDim.x)
    sl.ptr[i] = src[sl.off + i];
}

// received slices into the local copies (blockIdx.y = slice)
__global__ void k_vc_copy_in(double* __restrict__ curr, const VcSlice* __restrict__ t) {
  const VcSlice sl = t[blockIdx.y];
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < sl.cnt; i += (uint64_t) gridDim.x * blockDim.x)
    curr[sl.off + i] = sl.ptr[i];
}

enum { kPEval = 0, kRound = 1, kLast = 2 };

// Owner side: fold the partial sums of every holder (fid order), then
//   kPEval: deg = sum, mr = p / deg (p when dangling), count the dangling masters;
//   kRound: mr = (base + delta * sum) / deg (base when dangling);
//   kLast:  res = sum * delta + base.
// kPEval / kRound write mr into the own local copy and store it into every other holder's slot.
struct VcMasterArgs {
  const double* const* fold;   // [nfold] partial-sum slices, fid order
  uint32_t nfold;
  double* const* scat;         // [nscat] peer slots of the other holders
  uint32_t nscat;
  uint64_t nm;
  double* deg;
  double* curr_own;
  double* res;
  double p, base, delta;
  unsigned long long* ndangling;
};
__global__ void k_vc_master(VcMasterArgs a, int mode) {
  uint32_t dangling = 0;
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < a.nm; i += (uint64_t) gridDim.x * blockDim.x) {
    double sum = a.fold[0][i];
    for (uint32_t k = 1; k < a.nfold; ++k) sum += a.fold[k][i];
    if (mode == kLast) {
      a.res[i] = sum * a.delta + a.base;
      continue;
    }
    double mr;
    if (mode == kPEval) {
      a.deg[i] = sum;
      mr = sum > 0 ? a.p / sum : a.p;
      dangling += sum > 0 ? 0u : 1u;
    } else {
      const double d = a.deg[i];
      mr = d > 0 ? (a.base + a.delta * sum) / d : a.base;
    }
    a.curr_own[i] = mr;
    for (uint32_t k = 0; k < a.nscat; ++k) a.scat[k][i] = mr;
  }
  if (mode == kPEval) {
    const unsigned long long c = warp_sum((unsigned long long) dangling);
    if (lane_id() == 0 && c) atomicAdd(a.ndangling, c);
  }
}

struct PageRankVcApp : gl_app {
  gl_vcfrag* vf = nullptr;
  uint32_t nl = 0;
  uint64_t nm = 0, mlid = 0;   // own masters and the local id of the first
  DevBuf<double> curr, next, deg, res;
  DevBuf<unsigned long long> d_ndangling;
  TierLongRows lr;   // rows longer than kTierChunk entries
  // gather / scatter tables (F > 1)
  DevBuf<VcSlice> d_put, d_copy;
  uint32_t nput = 0, ncopy = 0;
  uint64_t max_slice = 0;
  DevBuf<const double*> d_fold;
  DevBuf<double*> d_scat;
  uint32_t nfold = 1, nscat = 0;
  uint64_t gather_bytes = 0, scatter_bytes = 0;
  int step = 0;
  int64_t ndangling = 0;
  double dangling_sum = 0;

  explicit PageRankVcApp(gl_vcfrag* f) : vf(f) {}

  size_t ResultElemBytes() const override { return sizeof(double); }
  size_t ResultCount() const override { return nm; }
  int ResultOids(int64_t* out, size_t count) override {
    GL_ARG(count >= nm, "result_oids buffer too small");
    const uint64_t mb = vf->master_begin(vf->fid);
    for (uint64_t i = 0; i < nm; ++i) out[i] = (int64_t) (mb + i);
    return GL_OK;
  }

  int Setup() override {
    nl = vf->nlocal;
    const uint64_t mb = vf->master_begin(vf->fid);
    nm = vf->master_end(vf->fid) - mb;
    mlid = nm ? vf->lid(mb) : 0;
    GL_CUDA(curr.alloc(std::max<uint32_t>(nl, 1)));
    GL_CUDA(next.alloc(std::max<uint32_t>(nl, 1)));
    GL_CUDA(deg.alloc(std::max<uint64_t>(nm, 1)));
    GL_CUDA(res.alloc(std::max<uint64_t>(nm, 1)));
    GL_CUDA(d_ndangling.alloc(1));
    GL_TRY(lr.plan(vf->rp, nl));
    if (vf->fnum > 1) {
      const uint64_t need = 8 * vf->mvc;
      if (!comm || !comm->opened || comm->fnum != vf->fnum || comm->fid != vf->fid) {
        set_error("a vertex-cut fragment with fnum=%u needs an opened communicator of the same fid / fnum", vf->fnum);
        return GL_ERR_ARG;
      }
      if (comm->mirror_bytes < need) {
        set_error("mirror_bytes %zu < 8 * mvc = %llu", comm->mirror_bytes, (unsigned long long) need);
        return GL_ERR_ARG;
      }
    }
    GL_TRY(mm.Init(comm, fv, 8));
    return plan_gather_scatter();
  }

  int plan_gather_scatter() {
    const uint32_t F = vf->fnum, me = vf->fid;
    std::vector<VcSlice> put, copy;
    std::vector<const double*> fold;
    std::vector<double*> scat;
    for (uint32_t g = 0; g < F; ++g) {
      const uint64_t gb = vf->master_begin(g), cnt = vf->master_end(g) - gb;
      if (g == me) {
        fold.push_back(next.get() + mlid);
        continue;
      }
      // g's masters lie in chunk g / side: I hold them when that chunk is one of my two ranges
      if (cnt && vf->holds_chunk(g / vf->side)) {
        put.push_back({(double*) (comm->peer_base[g] + comm->mirror_off(0, me)), vf->lid(gb), cnt});
        copy.push_back({(double*) (comm->local_base + comm->mirror_off(1, g)), vf->lid(gb), cnt});
        gather_bytes += 8 * cnt;
        max_slice = std::max(max_slice, cnt);
      }
      // g holds my masters (chunk me / side)
      const uint32_t c = vf->chunk_of_src();
      if (nm && (g / vf->side == c || g % vf->side == c)) {
        fold.push_back((const double*) (comm->local_base + comm->mirror_off(0, g)));
        scat.push_back((double*) (comm->peer_base[g] + comm->mirror_off(1, me)));
        scatter_bytes += 8 * nm;
      }
    }
    nput = (uint32_t) put.size();
    ncopy = (uint32_t) copy.size();
    nfold = (uint32_t) fold.size();
    nscat = (uint32_t) scat.size();
    GL_CUDA(d_fold.alloc(nfold));
    GL_CUDA(cudaMemcpy(d_fold, fold.data(), sizeof(double*) * nfold, cudaMemcpyHostToDevice));
    GL_CUDA(d_scat.alloc(std::max<uint32_t>(nscat, 1)));
    if (nscat) GL_CUDA(cudaMemcpy(d_scat, scat.data(), sizeof(double*) * nscat, cudaMemcpyHostToDevice));
    GL_CUDA(d_put.alloc(std::max<uint32_t>(nput, 1)));
    GL_CUDA(d_copy.alloc(std::max<uint32_t>(ncopy, 1)));
    if (nput) GL_CUDA(cudaMemcpy(d_put, put.data(), sizeof(VcSlice) * nput, cudaMemcpyHostToDevice));
    if (ncopy) GL_CUDA(cudaMemcpy(d_copy, copy.data(), sizeof(VcSlice) * ncopy, cudaMemcpyHostToDevice));
    return GL_OK;
  }

  int Init() override {
    step = 0;
    if (nm) GL_CUDA(cudaMemsetAsync(res, 0, sizeof(double) * nm, eng.stream));
    return GL_OK;
  }

  int slice_grid(uint64_t cnt) const {
    return (int) std::max<uint64_t>(1, std::min<uint64_t>((cnt + 255) / 256, (uint64_t) eng.sm_count * 4));
  }

  // gather: partial-sum slices to their owners; barrier; fold + update (+ scatter unless kLast)
  int gather_update(int mode, double base) {
    cudaStream_t s = eng.stream;
    if (vf->fnum > 1) {
      comm->mirror_dirty = true;
      if (nput) GL_LAUNCH(k_vc_put, dim3(slice_grid(max_slice), nput), 256, s, next, d_put);
      mm.bytes_sent += gather_bytes;
      GL_TRY(mm.PeerBarrierAsync(s));
    }
    VcMasterArgs a{d_fold, nfold, d_scat, mode == kLast ? 0u : nscat, nm, deg, curr.get() + mlid, res,
                   1.0 / (double) vf->n, base, cfg.pr_delta, d_ndangling};
    if (nm) GL_LAUNCH(k_vc_master, slice_grid(nm), 256, s, a, mode);
    if (mode != kLast && vf->fnum > 1) {
      mm.bytes_sent += scatter_bytes;
      GL_TRY(mm.PeerBarrierAsync(s));
      if (ncopy) GL_LAUNCH(k_vc_copy_in, dim3(slice_grid(max_slice), ncopy), 256, s, curr, d_copy);
    }
    return GL_OK;
  }

  int PEval() override {
    if (cfg.max_round <= 0) return GL_OK;
    cudaStream_t s = eng.stream;
    GL_CUDA(cudaMemsetAsync(d_ndangling, 0, sizeof(unsigned long long), s));
    // degree partials: the local CSR holds both endpoints of every block edge, so a row's length is
    // the vertex's degree inside the block
    if (nl) GL_LAUNCH(k_row_length<double>, (nl + 255) / 256, 256, s, vf->rp, nl, next);
    GL_TRY(gather_update(kPEval, 0.0));
    unsigned long long nd = 0;
    GL_CUDA(cudaMemcpyAsync(&nd, d_ndangling, sizeof(nd), cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    long long d0 = (long long) nd, d1 = 0;
    double d2 = 0;
    if (vf->fnum > 1) GL_TRY(mm.PeerAllReduce(s, &d0, &d1, &d2, 0));
    ndangling = d0;
    dangling_sum = (1.0 / (double) vf->n) * (double) ndangling;
    mm.ForceContinue();
    return GL_OK;
  }

  int IncEval() override {
    if (step >= cfg.max_round) return GL_OK;
    ++step;
    cudaStream_t s = eng.stream;
    const double N = (double) vf->n;
    const double base = (1.0 - cfg.pr_delta) / N + cfg.pr_delta * dangling_sum / N;
    dangling_sum = base * (double) ndangling;
    if (nl) {
      static thread_local int gp = 0;
      if (!gp) gp = persistent_grid(k_vc_pull, eng.sm_count);
      const int grid = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) nl + kTB - 1) / kTB);
      GL_LAUNCH(k_vc_pull, grid, kTB, s, vf->rp, vf->col, nl, curr, next);
      if (lr.nlong) {
        const int g2 = (int) std::min<uint64_t>((uint64_t) gp, ((uint64_t) lr.nitems * 32 + kTB - 1) / kTB);
        GL_LAUNCH(k_vc_chunks, g2, kTB, s, lr.cb, lr.ce, lr.nitems, vf->col, curr, lr.csum);
        GL_LAUNCH(k_vc_long, (lr.nlong + 255) / 256, 256, s, lr.rows, lr.off, lr.nlong, lr.csum, next);
      }
    }
    const bool last = step == cfg.max_round;
    GL_TRY(gather_update(last ? kLast : kRound, base));
    if (!last) mm.ForceContinue();
    note_step(vf->entries(), nl, 2);
    q_touched += nm;
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (!nm) return GL_OK;
    GL_CUDA(cudaMemcpyAsync(host_out, res, sizeof(double) * nm, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_pagerank_vc(gl_vcfrag* f) { return new PageRankVcApp(f); }

}  // namespace gl
