// dag_common.cuh — the degree-ordered DAG shared by LCC (app_lcc.cu), directed LCC (app_lcc_directed.cu)
// and k-clique (app_kclique.cu).  A fragment keeps some CSR entries of its inner vertices, each oriented
// one way, as rows of head gids sorted ascending (orp / okey; osrc holds the tail lid of every entry), and
// replicates its peers' rows (PeerCsr).  LCC and directed LCC count triangles over it with one app body,
// TriangleApp.  Every kernel is a template, so a unit compiles only the kernels it launches.
#pragma once
#include <cub/cub.cuh>

#include "apps_common.cuh"

namespace gl {
namespace {

// Keep is the app's rule for entry p of the inner row [b, e) of v, pointing at u (d: degree, g: gid):
//   GL_DEV bool operator()(const uint32_t* col, uint64_t b, uint64_t p, uint32_t v, uint32_t u,
//                          uint32_t dv, uint32_t du, uint32_t gv, uint32_t gu) const;

// cnt[v] = kept entries of the inner row v, cnt[ivnum] = 0; max_row (when non-null) takes the longest row
template <typename Keep>
__global__ void k_dag_count(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                            const uint32_t* __restrict__ deg, GidOf gid, uint32_t ivnum, Keep keep, uint64_t* cnt,
                            unsigned int* max_row) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v <= ivnum; v += warps) {
    if (v == ivnum) {
      if (lane_id() == 0) cnt[v] = 0;
      continue;
    }
    const uint64_t b = rp[v], e = rp[v + 1];
    const uint32_t dv = deg[v], gv = gid(v);
    uint32_t k = 0;
    for (uint64_t p = b + lane_id(); p < e; p += 32) {
      const uint32_t u = col[p];
      k += keep(col, b, p, v, u, dv, deg[u], gv, gid(u));
    }
    k = warp_sum(k);
    if (lane_id() == 0) {
      cnt[v] = k;
      if (max_row && k) atomicMax(max_row, k);
    }
  }
}

// order-preserving fill: okey = gid of the head, osrc = lid of the tail, olid (when non-null) = lid of
// the head
template <typename Keep>
__global__ void k_dag_fill(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                           const uint32_t* __restrict__ deg, GidOf gid, uint32_t ivnum, Keep keep,
                           const uint64_t* __restrict__ orp, uint32_t* okey, uint32_t* olid, uint32_t* osrc) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const uint64_t b = rp[v], e = rp[v + 1];
    const uint32_t dv = deg[v], gv = gid(v);
    uint64_t o = orp[v];
    for (uint64_t p0 = b; p0 < e; p0 += 32) {
      const uint64_t p = p0 + lane_id();
      bool k = false;
      uint32_t u = 0, gu = 0;
      if (p < e) {
        u = col[p];
        gu = gid(u);
        k = keep(col, b, p, v, u, dv, deg[u], gv, gu);
      }
      const uint32_t mask = __ballot_sync(0xffffffffu, k);
      if (k) {
        const uint64_t at = o + __popc(mask & ((1u << lane_id()) - 1));
        okey[at] = gu;
        if (olid) olid[at] = u;
        osrc[at] = v;
      }
      o += __popc(mask);
    }
  }
}

// orp = exclusive scan of the ivnum + 1 row counts in cnt; *total = orp[ivnum]
inline int dag_scan(cudaStream_t s, const uint64_t* cnt, uint64_t* orp, uint32_t ivnum, uint64_t* total) {
  size_t tb = 0;
  GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, orp, (int) (ivnum + 1), s));
  DevBuf<char> tmp;
  GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
  GL_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, orp, (int) (ivnum + 1), s));
  GL_CUDA(cudaMemcpyAsync(total, orp + ivnum, 8, cudaMemcpyDeviceToHost, s));
  GL_CUDA(cudaStreamSynchronize(s));
  return GL_OK;
}

// One warp per oriented edge (v,u) of this fragment: every entry x of N+(u), read from its owner's
// replica, is searched in the sorted N+(v); a common x adds w(v,u) to x, w(v,x) to u and w(u,x) to v in
// 64-bit atomics.  Unweighted: every weight is 1.  olid is the lid of each head, null where gids are lids
// (one fragment).
template <bool kWeighted>
__global__ void __launch_bounds__(256)
k_dag_tri(const uint64_t* __restrict__ orp, const uint32_t* __restrict__ okey, const uint32_t* __restrict__ olid,
          const uint32_t* __restrict__ ow, const uint32_t* __restrict__ osrc, uint64_t om,
          const uint64_t* const* __restrict__ t_orp, const uint32_t* const* __restrict__ t_key,
          const uint32_t* const* __restrict__ t_w, int fid_offset, uint32_t id_mask,
          unsigned long long* tri, ScanCtrl* ctrl) {
  using Sum = std::conditional_t<kWeighted, unsigned long long, uint32_t>;
  const uint64_t warps = ((uint64_t) gridDim.x * blockDim.x) >> 5;
  uint64_t scanned = 0;
  for (uint64_t ei = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; ei < om; ei += warps) {
    const uint32_t v = osrc[ei], ug = okey[ei], ul = olid ? olid[ei] : ug;
    const unsigned long long wvu = kWeighted ? ow[ei] : 1ull;
    const uint64_t vb = orp[v], ve = orp[v + 1];
    const uint32_t g = ug >> fid_offset, l = ug & id_mask;
    const uint64_t* rorp = t_orp[g];
    const uint32_t* rkey = t_key[g];
    const uint32_t* rw = kWeighted ? t_w[g] : nullptr;
    const uint64_t ub = rorp[l], ue = rorp[l + 1];
    Sum to_u = 0, to_v = 0;
    for (uint64_t p = ub + lane_id(); p < ue; p += 32) {
      const uint32_t x = rkey[p];
      uint64_t lo = vb, hi = ve;
      while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (okey[mid] < x) lo = mid + 1; else hi = mid;
      }
      if (lo < ve && okey[lo] == x) {
        atomicAdd(tri + (olid ? olid[lo] : x), wvu);
        to_u += kWeighted ? ow[lo] : 1u;
        if (kWeighted) to_v += rw[p];
      }
    }
    to_u = warp_sum(to_u);
    to_v = kWeighted ? warp_sum(to_v) : to_u;
    if (lane_id() == 0) {
      if (to_u) atomicAdd(tri + ul, (unsigned long long) to_u);
      if (to_v) atomicAdd(tri + v, (unsigned long long) to_v);
      scanned += ue - ub;
    }
  }
  if (lane_id() == 0 && scanned) atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}

// remote bit of every outer copy with a non-zero count
template <typename T>
__global__ void k_mark_nonzero(const T* cnt, uint32_t ivnum, uint32_t ovnum, uint32_t* remote) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ovnum && cnt[ivnum + i]) bit_set_atomic(remote, ivnum + i);
}
struct TriPayload {
  const unsigned long long* tri;
  GL_DEV ItemU32I64 operator()(uint32_t v, uint32_t lid) const { return ItemU32I64{lid, 0u, (int64_t) tri[v]}; }
};
struct TriApply {
  unsigned long long* tri;
  GL_DEV void operator()(const ItemU32I64& it, ScanAcc&) const {
    atomicAdd(tri + it.lid, (unsigned long long) it.val);
  }
};

// out[v] = factor * tri / (d (d - 1)), 0 when d < 2
template <typename T>
__global__ void k_clustering(const uint32_t* d, const T* tri, uint32_t ivnum, double factor, double* out) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= ivnum) return;
  const int64_t dv = d[v];
  out[v] = dv < 2 ? 0.0 : factor * (double) tri[v] / (double) (dv * (dv - 1));
}

// LCC and directed LCC: the app fills the DAG in PEval (deg: its degree of every inner and outer vertex;
// ow: one weight per entry when kWeighted) and writes its result through WriteResult.  A triangle is
// counted once, at the owner of its highest-ranked vertex; counts that land on outer copies go to their
// owners as (lid, count) items.
template <bool kWeighted>
struct TriangleApp : gl_app {
  DevBuf<uint64_t> cnt, orp;
  DevBuf<uint32_t> deg, okey, osrc, remote;
  DevBuf<uint32_t> olid;   // several fragments only: on one fragment the head gids are their lids
  DevBuf<uint32_t> ow;     // kWeighted only
  DevBuf<unsigned long long> tri;
  DevBuf<double> out64;
  uint64_t om = 0;
  int stage = 0;
  uint32_t tvnum = 0;
  size_t words = 0;
  PeerCsr peers;   // every fragment's rows (one fragment: its own)

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    words = bm_words(tvnum) + 1;
    GL_CUDA(cnt.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(orp.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(deg.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(tri.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32I64)));
    if (fv.fnum > 1) {
      GL_CUDA(remote.alloc(words));
      GL_TRY(mm.BuildMirrorPlan(eng.stream, fv));
    }
    return GL_OK;
  }

  int Init() override {
    stage = 0;
    GL_CUDA(cudaMemsetAsync(tri, 0, sizeof(unsigned long long) * std::max<uint32_t>(tvnum, 1), eng.stream));
    if (remote) GL_CUDA(cudaMemsetAsync(remote, 0, sizeof(uint32_t) * words, eng.stream));
    return GL_OK;
  }

  // orp from the row counts in cnt; the DAG arrays sized for its total
  int scan_and_resize() {
    uint64_t total = 0;
    GL_TRY(dag_scan(eng.stream, cnt, orp, fv.ivnum, &total));
    if (total != om || !okey) {
      okey.reset();
      olid.reset();
      ow.reset();
      osrc.reset();
      om = total;
      GL_CUDA(okey.alloc(std::max<uint64_t>(om, 4)));
      GL_CUDA(osrc.alloc(std::max<uint64_t>(om, 4)));
      if (kWeighted) GL_CUDA(ow.alloc(std::max<uint64_t>(om, 4)));
      if (fv.fnum > 1) GL_CUDA(olid.alloc(std::max<uint64_t>(om, 4)));
    }
    return GL_OK;
  }

  // IncEval: triangle counting (stage 1; lcc.h:133-196, lcc_directed.h:241-350), then the counts of outer
  // copies are added at their owners (stage 2; lcc.h:178-196, lcc_directed.h:351-357)
  int IncEval() override {
    cudaStream_t s = eng.stream;
    if (stage == 0) {
      stage = 1;
      GL_TRY(eng.reset_ctrl());
      if (om)
        GL_LAUNCH(k_dag_tri<kWeighted>, eng.sm_count * 8, 256, s, orp, okey, olid, ow, osrc, om, peers.d_rp, peers.d_col,
                  peers.d_w, fv.fid_offset, fv.id_mask, tri, eng.ctrl);
      if (fv.fnum > 1) {
        if (fv.ovnum)
          GL_LAUNCH(k_mark_nonzero<unsigned long long>, (fv.ovnum + 255) / 256, 256, s, tri, fv.ivnum, fv.ovnum,
                    remote);
        MsgView mv = mm.view();
        GL_LAUNCH((k_pack_outer<ItemU32I64, TriPayload>), eng.sm_count * 4, kTB, s, remote, fv.ivnum, fv.ovnum,
                  fv.ovgid, mv, TriPayload{tri}, 0, nullptr);
      }
      GL_TRY(eng.fetch_ctrl());
      note_step(eng.h_ctrl->scanned, fv.ivnum, 2);
      q_touched += fv.ivnum;
      mm.ForceContinue();
    } else {
      if (stage == 1 && fv.fnum > 1) {
        MsgView mv = mm.view();
        GL_LAUNCH((k_unpack<ItemU32I64, TriApply>), eng.sm_count * 4, kTB, s, mv, TriApply{tri}, eng.ctrl);
      }
      stage = 2;
    }
    return GL_OK;
  }

  // the coefficient of every inner vertex from the app's degree d
  int WriteResult(void* host_out, const uint32_t* d, double factor) {
    if (fv.ivnum == 0) return GL_OK;
    GL_LAUNCH(k_clustering<unsigned long long>, (fv.ivnum + 255) / 256, 256, eng.stream, d, tri, fv.ivnum, factor,
              out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace
}  // namespace gl
