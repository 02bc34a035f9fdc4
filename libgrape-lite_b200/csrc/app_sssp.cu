// app_sssp.cu — single-source shortest paths, near/far ("delta-stepping")
// Bellman-Ford.
//
// Behaviour follows examples/analytical_apps/cuda/sssp/sssp.h:24-306: PEval
// (:143-171) seeds the source; IncEval (:173-305) applies received distances
// with atomicMin, relaxes the out-edges of the active set, files improved
// inner vertices into `near` (new < prio) or `far`, switches to `far` and
// raises prio by init_prio when `near` is empty (:273-285), and reports
// improved outer vertices to their owners (:295-304).
// init_prio = 32 * avg_weight / avg_degree (:82-92).
//
// Distances: f32 by default like the reference GPU app (run_cuda_app.cu:46);
// cfg.sssp_f64 = 1 computes in fp64 like the CPU app (run_app.cc:49).  The
// result is returned as double; unreachable = DBL_MAX (printed "infinity").
// min over paths of left-to-right sums is order independent, so results are
// bit-exact against the CPU oracle whenever the sums are exact in the chosen
// precision (integer weights in f32, any f32-valued weights in f64).
#include <cfloat>

#include "apps_common.cuh"

namespace gl {
namespace {

template <typename T>
GL_DEV T atomic_min_nonneg(T* a, T v);
template <>
GL_DEV float atomic_min_nonneg<float>(float* a, float v) {
  return atomic_min_f32_nonneg(a, v);
}
template <>
GL_DEV double atomic_min_nonneg<double>(double* a, double v) {
  return atomic_min_f64_nonneg(a, v);
}

template <typename T, typename WT>
struct OpSssp {
  using Meta = T;
  using W = WT;
  static constexpr bool kWeighted = true;
  T* dist;
  uint32_t* near;
  uint32_t* far;
  uint32_t* remote;
  uint32_t ivnum;
  T prio;
  GL_DEV Meta assign(uint32_t u) const { return dist[u]; }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W w, ScanAcc& acc) const {
    T nd = m + (T) w;
    if (!(nd < dist[v])) return;  // cheap filter (stale reads only delay)
    T old = atomic_min_nonneg<T>(dist + v, nd);
    if (nd < old) {
      acc.touched++;
      if (v < ivnum) {
        if (nd < prio) {
          if (bit_set_atomic(near, v)) acc.next_count++;
        } else {
          if (bit_set_atomic(far, v)) acc.aux++;
        }
      } else {
        if (bit_set_atomic(remote, v)) acc.remote++;
      }
    }
  }
};

template <typename T>
__global__ void k_fill(T* a, uint32_t n, T v) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

template <typename T>
__global__ void k_sssp_seed(uint32_t src, T* dist, uint32_t* in_q) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    dist[src] = (T) 0;
    in_q[src >> 5] |= 1u << (src & 31);
  }
}

template <typename WT>
__global__ void k_weight_sum(const WT* w, uint64_t m, double* out) {
  // out[0] += sum of the weights; out[1] = 1 when a weight is negative, -0.0 or
  // NaN: the device atomic-min orders distances by their bit patterns
  // (common.cuh atomic_min_*_nonneg), which is only an order for values >= +0
  double s = 0;
  bool bad = false;
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < m;
       i += (uint64_t) gridDim.x * blockDim.x) {
    const WT x = w[i];
    s += (double) x;
    bad |= !(x >= (WT) 0) || signbit(x);
  }
  s = warp_sum(s);
  if (lane_id() == 0) atomicAdd(out, s);
  if (bad) out[1] = 1.0;
}

template <typename T>
struct ItemDist {
  uint32_t lid;
  uint32_t pad;
  T val;
};
template <>
struct ItemDist<float> {
  uint32_t lid;
  float val;
};

template <typename T>
struct SsspPayload {
  const T* dist;
  GL_DEV ItemDist<T> operator()(uint32_t v, uint32_t lid) const {
    ItemDist<T> it;
    it.lid = lid;
    it.val = dist[v];
    return it;
  }
};
template <typename T>
struct SsspApply {
  T* dist;
  uint32_t* in_q;
  GL_DEV void operator()(const ItemDist<T>& it, ScanAcc& acc) const {
    if (it.val < atomic_min_nonneg<T>(dist + it.lid, it.val)) {
      if (bit_set_atomic(in_q, it.lid)) acc.aux++;
    }
  }
};

template <typename T>
__global__ void k_dist_to_f64(const T* d, uint32_t n, T inf, double* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = d[i] == inf ? DBL_MAX : (double) d[i];
}

template <typename T>
struct SsspApp : gl_app {
  DevBuf<T> dist;
  DevBuf<uint32_t> in_q, near, far, remote;
  DevBuf<double> out64;
  size_t words = 0;
  uint32_t tvnum = 0;
  T init_prio = 0, prio = 0;
  uint64_t far_total = 0;
  static T inf() { return sizeof(T) == 4 ? (T) FLT_MAX : (T) DBL_MAX; }

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    words = bm_words(tvnum) + 1;
    GL_CUDA(dist.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(in_q.alloc(words));
    GL_CUDA(near.alloc(words));
    GL_CUDA(far.alloc(words));
    GL_CUDA(remote.alloc(words));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    // init_prio heuristic (sssp.h:76-92)
    double p = cfg.sssp_prio;
    {
      double wsum = (double) frag->oe.entries;  // unweighted: every edge counts 1
      if (frag->oe.w && frag->oe.entries) {
        double h_sum[2] = {0, 0};
        DevBuf<double> d_sum;
        GL_CUDA(d_sum.alloc(2));
        GL_CUDA(cudaMemsetAsync(d_sum, 0, 16, eng.stream));
        if (fv.edata_bytes == 4) {
          GL_LAUNCH(k_weight_sum<float>, eng.sm_count * 8, 256, eng.stream, (const float*) frag->oe.w, frag->oe.entries, d_sum);
        } else {
          GL_LAUNCH(k_weight_sum<double>, eng.sm_count * 8, 256, eng.stream, (const double*) frag->oe.w, frag->oe.entries, d_sum);
        }
        GL_CUDA(cudaMemcpyAsync(h_sum, d_sum, 16, cudaMemcpyDeviceToHost, eng.stream));
        GL_CUDA(cudaStreamSynchronize(eng.stream));
        d_sum.reset();
        wsum = h_sum[0];
        if (h_sum[1] != 0.0) {
          set_error("SSSP: negative (or -0.0 / NaN) edge weights are not supported");
          return GL_ERR_ARG;
        }
      }
      double m = (double) std::max<uint64_t>(frag->oe.entries, 1);
      double iv = (double) std::max<uint32_t>(fv.ivnum, 1);
      if (p <= 0) p = 32.0 * (wsum / m) / (m / iv);
    }
    init_prio = (T) p;
    return mm.Init(comm, fv, sizeof(ItemDist<T>));
  }

  int Init() override {
    cudaStream_t s = eng.stream;
    if (tvnum) GL_LAUNCH(k_fill<T>, (tvnum + 255) / 256, 256, s, dist, tvnum, inf());
    GL_CUDA(cudaMemsetAsync(in_q, 0, sizeof(uint32_t) * words, s));
    GL_CUDA(cudaMemsetAsync(near, 0, sizeof(uint32_t) * words, s));
    GL_CUDA(cudaMemsetAsync(far, 0, sizeof(uint32_t) * words, s));
    GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
    prio = init_prio;
    far_total = 0;
    l2_persist_window(s, dist, sizeof(T) * (size_t) tvnum);   // random dist[v] probes hit L2 while col / w stream through
    return GL_OK;
  }

  int PEval() override {
    uint32_t src;
    if (gl_frag_oid2lid(frag, cfg.source_oid, &src) == GL_OK)
      GL_LAUNCH(k_sssp_seed<T>, 1, 32, eng.stream, src, dist, in_q);
    mm.ForceContinue();
    return GL_OK;
  }

  template <typename WT>
  int scan(cudaStream_t) {
    OpSssp<T, WT> op{dist, near, far, remote, fv.ivnum, prio};
    EdgeRange er{fv.oe_rp, fv.oe_col, fv.oe_w};
    return run_frontier_scan(eng, in_q, fv.ivnum, er, op);
  }

  int IncEval() override {
    cudaStream_t s = eng.stream;
    GL_TRY(eng.reset_ctrl());
    if (fv.fnum > 1) {
      MsgView mv = mm.view();
      SsspApply<T> ap{dist, in_q};
      GL_LAUNCH((k_unpack<ItemDist<T>, SsspApply<T>>), eng.sm_count * 4, kTB, s, mv, ap, eng.ctrl);
      GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, s));
      GL_TRY(eng.reset_ctrl());
    }
    if (fv.edata_bytes == 8) GL_TRY(scan<double>(s)); else GL_TRY(scan<float>(s));
    GL_CUDA(cudaMemsetAsync(in_q, 0, sizeof(uint32_t) * words, s));
    if (fv.fnum > 1) {
      MsgView mv = mm.view();
      GL_LAUNCH((k_pack_outer<ItemDist<T>, SsspPayload<T>>), eng.sm_count * 4, kTB, s, remote,
                fv.ivnum, fv.ovnum, fv.ovgid, mv, SsspPayload<T>{dist}, 0, nullptr);
    }
    GL_TRY(eng.fetch_ctrl());
    const ScanCtrl& c = *eng.h_ctrl;
    note_step(c.scanned, (uint32_t) std::min<uint64_t>(c.frontier, 0xFFFFFFFFu), 0);
    q_touched += c.touched;
    far_total += c.aux;
    uint64_t local = c.next_count;
    if (local > 0) {
      std::swap(in_q, near);
    } else {
      local = far_total;
      far_total = 0;
      std::swap(in_q, far);
      prio += init_prio;
    }
    if (local > 0) mm.ForceContinue();
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    l2_persist_clear(eng.stream);
    GL_LAUNCH(k_dist_to_f64<T>, (fv.ivnum + 255) / 256, 256, eng.stream, dist, fv.ivnum, inf(), out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_sssp_f32() { return new SsspApp<float>; }
gl_app* make_sssp_f64() { return new SsspApp<double>; }

}  // namespace gl
