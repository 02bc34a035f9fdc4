// app_lcc.cu — local clustering coefficient by oriented triangle counting.
//
// Semantics of examples/analytical_apps/lcc/lcc.h:48-233 + lcc_context.h:52-66
// (GPU apps: cuda/lcc/lcc_preprocess.h:96-188 + lcc_opt.h:183-316):
//   degree(v) = CSR entries of v's row (multi-edges count);
//   N+(v) = { u in N(v) : deg u < deg v, or deg u == deg v and gid(v) > gid(u) }
//   for every v, every u in N+(v) (with multiplicity), every w in N+(u) (with
//   multiplicity): if w is a member of N+(v) then tri[u], tri[v], tri[w] += 1;
//   lcc(v) = 2*tri / (d*(d-1)), 0 when d < 2.
// Integer counting => bit-exact; the final division is fp64 as in the reference.
//
// Re-design: the degree-ordered DAG is built on the device (the reference
// builds it on the CPU with one std::vector per vertex and ships it through
// MPI, lcc_preprocess.h), then one warp per oriented edge (v,u) intersects
// N+(u) against the sorted N+(v) by binary search; counts use 64-bit atomics.
//
// fnum > 1 (lcc.h:96-140 ships the filtered neighbour lists of every inner
// vertex to the fragments mirroring it, through MPI byte archives): here
//   1. degrees of the outer copies come from the dense mirror sync;
//   2. each fragment builds its part of the DAG with GLOBAL ids (rows sorted
//      by gid) and exports the two arrays through CUDA IPC;
//   3. every fragment replicates its peers' parts with bulk NVLink copies
//      (the whole DAG is 4 B per oriented edge — 1 GB at scale 24);
//   4. a triangle is counted once, by the owner of its highest-ranked vertex;
//      counts that land on outer copies go to their owners as (lid, count)
//      items and are added in the next round (the reference's
//      SyncStateOnOuterVertex + sum, lcc.h:178-196).
#include <cub/cub.cuh>

#include <cstring>
#include <vector>

#include "apps_common.cuh"

namespace gl {
namespace {

GL_DEV bool keep_edge(uint64_t dv, uint64_t du, uint32_t v, uint32_t u) {
  return du < dv || (du == dv && v > u);
}

__global__ void k_lcc_count(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                            uint32_t ivnum, uint64_t* cnt) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v <= ivnum; v += warps) {
    if (v == ivnum) {
      if (lane_id() == 0) cnt[v] = 0;
      continue;
    }
    const uint64_t b = rp[v], e = rp[v + 1], dv = e - b;
    uint32_t k = 0;
    for (uint64_t p = b + lane_id(); p < e; p += 32) {
      uint32_t u = col[p];
      uint64_t du = rp[u + 1] - rp[u];
      k += keep_edge(dv, du, v, u);
    }
    k = warp_sum(k);
    if (lane_id() == 0) cnt[v] = k;
  }
}

// order-preserving fill (rows stay sorted by lid)
__global__ void k_lcc_fill(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                           uint32_t ivnum, const uint64_t* __restrict__ orp,
                           uint32_t* ocol, uint32_t* osrc) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const uint64_t b = rp[v], e = rp[v + 1], dv = e - b;
    uint64_t o = orp[v];
    for (uint64_t p0 = b; p0 < e; p0 += 32) {
      uint64_t p = p0 + lane_id();
      bool k = false;
      uint32_t u = 0;
      if (p < e) {
        u = col[p];
        k = keep_edge(dv, rp[u + 1] - rp[u], v, u);
      }
      uint32_t mask = __ballot_sync(0xffffffffu, k);
      if (k) {
        uint64_t at = o + __popc(mask & ((1u << lane_id()) - 1));
        ocol[at] = u;
        osrc[at] = v;
      }
      o += __popc(mask);
    }
  }
}

// one warp per oriented edge (v,u)
__global__ void __launch_bounds__(256)
k_lcc_tri(const uint64_t* __restrict__ orp, const uint32_t* __restrict__ ocol,
          const uint32_t* __restrict__ osrc, uint64_t om,
          unsigned long long* tri, ScanCtrl* ctrl) {
  const uint64_t warps = ((uint64_t) gridDim.x * blockDim.x) >> 5;
  uint64_t scanned = 0;
  for (uint64_t ei = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; ei < om; ei += warps) {
    const uint32_t v = osrc[ei], u = ocol[ei];
    const uint64_t vb = orp[v], ve = orp[v + 1];
    const uint64_t ub = orp[u], ue = orp[u + 1];
    uint32_t found = 0;
    for (uint64_t p = ub + lane_id(); p < ue; p += 32) {
      const uint32_t w = ocol[p];
      uint64_t lo = vb, hi = ve;
      while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (ocol[mid] < w) lo = mid + 1; else hi = mid;
      }
      if (lo < ve && ocol[lo] == w) {
        ++found;
        atomicAdd(tri + w, 1ull);
      }
    }
    found = warp_sum(found);
    if (lane_id() == 0) {
      if (found) {
        atomicAdd(tri + u, (unsigned long long) found);
        atomicAdd(tri + v, (unsigned long long) found);
      }
      scanned += ue - ub;
    }
  }
  if (lane_id() == 0 && scanned) atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}


// ---------------------------------------------------------------- fnum > 1
__global__ void k_lcc_count_m(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                              const uint32_t* __restrict__ deg, GidOf gid, uint32_t ivnum, uint64_t* cnt) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v <= ivnum; v += warps) {
    if (v == ivnum) {
      if (lane_id() == 0) cnt[v] = 0;
      continue;
    }
    const uint64_t b = rp[v], e = rp[v + 1], dv = e - b;
    const uint32_t gv = gid(v);
    uint32_t k = 0;
    for (uint64_t p = b + lane_id(); p < e; p += 32) {
      const uint32_t u = col[p];
      k += keep_edge(dv, deg[u], gv, gid(u));
    }
    k = warp_sum(k);
    if (lane_id() == 0) cnt[v] = k;
  }
}

__global__ void k_lcc_fill_m(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                             const uint32_t* __restrict__ deg, GidOf gid, uint32_t ivnum,
                             const uint64_t* __restrict__ orp, uint32_t* okey, uint32_t* olid, uint32_t* osrc) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < ivnum; v += warps) {
    const uint64_t b = rp[v], e = rp[v + 1], dv = e - b;
    const uint32_t gv = gid(v);
    uint64_t o = orp[v];
    for (uint64_t p0 = b; p0 < e; p0 += 32) {
      uint64_t p = p0 + lane_id();
      bool k = false;
      uint32_t u = 0, gu = 0;
      if (p < e) {
        u = col[p];
        gu = gid(u);
        k = keep_edge(dv, deg[u], gv, gu);
      }
      uint32_t mask = __ballot_sync(0xffffffffu, k);
      if (k) {
        uint64_t at = o + __popc(mask & ((1u << lane_id()) - 1));
        okey[at] = gu;
        olid[at] = u;
        osrc[at] = v;
      }
      o += __popc(mask);
    }
  }
}

// one warp per oriented edge (v,u); N+(u) comes from the owner's replica
__global__ void __launch_bounds__(256)
k_lcc_tri_m(const uint64_t* __restrict__ orp, const uint32_t* __restrict__ okey,
            const uint32_t* __restrict__ olid, const uint32_t* __restrict__ osrc, uint64_t om,
            const uint64_t* const* __restrict__ t_orp, const uint32_t* const* __restrict__ t_key,
            int fid_offset, uint32_t id_mask, unsigned long long* tri, ScanCtrl* ctrl) {
  const uint64_t warps = ((uint64_t) gridDim.x * blockDim.x) >> 5;
  uint64_t scanned = 0;
  for (uint64_t ei = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; ei < om; ei += warps) {
    const uint32_t v = osrc[ei], ug = okey[ei], ul = olid[ei];
    const uint64_t vb = orp[v], ve = orp[v + 1];
    const uint32_t g = ug >> fid_offset, l = ug & id_mask;
    const uint64_t* rorp = t_orp[g];
    const uint32_t* rkey = t_key[g];
    const uint64_t ub = rorp[l], ue = rorp[l + 1];
    uint32_t found = 0;
    for (uint64_t p = ub + lane_id(); p < ue; p += 32) {
      const uint32_t w = rkey[p];
      uint64_t lo = vb, hi = ve;
      while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (okey[mid] < w) lo = mid + 1; else hi = mid;
      }
      if (lo < ve && okey[lo] == w) {
        ++found;
        atomicAdd(tri + olid[lo], 1ull);
      }
    }
    found = warp_sum(found);
    if (lane_id() == 0) {
      if (found) {
        atomicAdd(tri + ul, (unsigned long long) found);
        atomicAdd(tri + v, (unsigned long long) found);
      }
      scanned += ue - ub;
    }
  }
  if (lane_id() == 0 && scanned) atomicAdd(&ctrl->scanned, (unsigned long long) scanned);
}

__global__ void k_lcc_mark_remote(const unsigned long long* tri, uint32_t ivnum, uint32_t ovnum, uint32_t* remote) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ovnum && tri[ivnum + i]) bit_set_atomic(remote, ivnum + i);
}
struct LccPayload {
  const unsigned long long* tri;
  GL_DEV ItemU32I64 operator()(uint32_t v, uint32_t lid) const {
    return ItemU32I64{lid, 0u, (int64_t) tri[v]};
  }
};
struct LccApply {
  unsigned long long* tri;
  GL_DEV void operator()(const ItemU32I64& it, ScanAcc&) const {
    atomicAdd(tri + it.lid, (unsigned long long) it.val);
  }
};

__global__ void k_lcc_out(const uint64_t* rp, const unsigned long long* tri,
                          uint32_t ivnum, double* out) {
  uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= ivnum) return;
  int64_t d = (int64_t) (rp[v + 1] - rp[v]);
  out[v] = d < 2 ? 0.0 : 2.0 * (double) tri[v] / (double) (d * (d - 1));
}

struct LccApp : gl_app {
  DevBuf<uint64_t> cnt, orp;
  DevBuf<uint32_t> ocol, osrc;   // fnum > 1: ocol holds gids (sorted per row)
  DevBuf<uint32_t> olid, deg, remote;
  DevBuf<unsigned long long> tri;
  DevBuf<double> out64;
  uint64_t om = 0;
  int stage = 0;
  uint32_t tvnum = 0;
  size_t words = 0;
  PeerCsr peers;   // fnum > 1: every fragment's part of the DAG

  size_t ResultElemBytes() const override { return sizeof(double); }

  int Setup() override {
    tvnum = fv.ivnum + fv.ovnum;
    words = bm_words(tvnum) + 1;
    GL_CUDA(cnt.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(orp.alloc((size_t) fv.ivnum + 1));
    GL_CUDA(tri.alloc(std::max<uint32_t>(tvnum, 1)));
    GL_CUDA(out64.alloc(std::max<uint32_t>(fv.ivnum, 1)));
    GL_TRY(mm.Init(comm, fv, sizeof(ItemU32I64)));
    if (fv.fnum > 1) {
      GL_CUDA(deg.alloc(std::max<uint32_t>(tvnum, 1)));
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

  int scan_counts(uint64_t* total) {
    cudaStream_t s = eng.stream;
    size_t tb = 0;
    GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.get(), orp.get(), (int) (fv.ivnum + 1), s));
    DevBuf<char> tmp;
    GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
    GL_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt.get(), orp.get(), (int) (fv.ivnum + 1), s));
    GL_CUDA(cudaMemcpyAsync(total, orp + fv.ivnum, 8, cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    return GL_OK;
  }
  int resize_dag(uint64_t total) {
    if (total != om || !ocol) {
      ocol.reset();
      osrc.reset();
      olid.reset();
      om = total;
      GL_CUDA(ocol.alloc(std::max<uint64_t>(om, 4)));
      GL_CUDA(osrc.alloc(std::max<uint64_t>(om, 4)));
      if (fv.fnum > 1) GL_CUDA(olid.alloc(std::max<uint64_t>(om, 4)));
    }
    return GL_OK;
  }

  // PEval: degrees + degree-ordered DAG (lcc.h:48-74 and stage 0, :84-132)
  int PEval() override {
    cudaStream_t s = eng.stream;
    if (fv.fnum > 1) return PEvalMulti();
    GL_LAUNCH(k_lcc_count, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, fv.ivnum, cnt);
    uint64_t total = 0;
    GL_TRY(scan_counts(&total));
    GL_TRY(resize_dag(total));
    if (fv.ivnum) GL_LAUNCH(k_lcc_fill, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, fv.ivnum, orp, ocol, osrc);
    mm.ForceContinue();
    return GL_OK;
  }

  int PEvalMulti() {
    cudaStream_t s = eng.stream;
    const GidOf gid{fv.ivnum, fv.fid, fv.fid_offset, fv.ovgid};
    // 1. degrees: own rows, then the owners' values for the outer copies
    if (fv.ivnum) GL_LAUNCH(k_row_length<uint32_t>, (fv.ivnum + 255) / 256, 256, s, fv.oe_rp, fv.ivnum, deg.get());
    GL_TRY(mm.SyncValuesToGhosts(s, deg, 4));
    // 2. my part of the DAG, global ids, rows sorted by gid
    GL_LAUNCH(k_lcc_count_m, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, cnt);
    uint64_t total = 0;
    GL_TRY(scan_counts(&total));
    GL_TRY(resize_dag(total));
    if (fv.ivnum && om) {
      DevBuf<uint32_t> key_u, lid_u;
      GL_CUDA(key_u.alloc(om));
      GL_CUDA(lid_u.alloc(om));
      GL_LAUNCH(k_lcc_fill_m, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, orp, key_u, lid_u, osrc);
      size_t sb = 0;
      GL_CUDA(cub::DeviceSegmentedSort::SortPairs(nullptr, sb, key_u.get(), ocol.get(), lid_u.get(), olid.get(), (int64_t) om,
                                                  (int64_t) fv.ivnum, orp.get(), orp + 1, s));
      DevBuf<char> st;
      GL_CUDA(st.alloc(std::max<size_t>(sb, 16)));
      GL_CUDA(cub::DeviceSegmentedSort::SortPairs(st, sb, key_u.get(), ocol.get(), lid_u.get(), olid.get(), (int64_t) om,
                                                  (int64_t) fv.ivnum, orp.get(), orp + 1, s));
      GL_CUDA(cudaStreamSynchronize(s));
    }
    // 3. replicate the peers' parts (bulk NVLink copies)
    GL_TRY(peers.replicate(mm, s, fv, orp, ocol, om));
    mm.ForceContinue();
    return GL_OK;
  }

  // IncEval: triangle counting (stage 1, lcc.h:133-196), then the counts of
  // outer copies are added at their owners (stage 2)
  int IncEval() override {
    cudaStream_t s = eng.stream;
    if (stage == 0) {
      stage = 1;
      GL_TRY(eng.reset_ctrl());
      if (fv.fnum == 1) {
        if (om) GL_LAUNCH(k_lcc_tri, eng.sm_count * 8, 256, s, orp, ocol, osrc, om, tri, eng.ctrl);
      } else {
        if (om) GL_LAUNCH(k_lcc_tri_m, eng.sm_count * 8, 256, s, orp, ocol, olid, osrc, om, peers.d_rp, peers.d_col,
                          fv.fid_offset, fv.id_mask, tri, eng.ctrl);
        if (fv.ovnum) GL_LAUNCH(k_lcc_mark_remote, (fv.ovnum + 255) / 256, 256, s, tri, fv.ivnum, fv.ovnum, remote);
        MsgView mv = mm.view();
        GL_LAUNCH((k_pack_outer<ItemU32I64, LccPayload>), eng.sm_count * 4, kTB, s, remote, fv.ivnum, fv.ovnum,
                  fv.ovgid, mv, LccPayload{tri}, 0, nullptr);
      }
      GL_TRY(eng.fetch_ctrl());
      note_step(eng.h_ctrl->scanned, fv.ivnum, 2);
      q_touched += fv.ivnum;
      mm.ForceContinue();
    } else {
      if (stage == 1 && fv.fnum > 1) {
        MsgView mv = mm.view();
        GL_LAUNCH((k_unpack<ItemU32I64, LccApply>), eng.sm_count * 4, kTB, s, mv, LccApply{tri}, eng.ctrl);
      }
      stage = 2;
    }
    return GL_OK;
  }

  int Result(void* host_out, size_t) override {
    if (fv.ivnum == 0) return GL_OK;
    GL_LAUNCH(k_lcc_out, (fv.ivnum + 255) / 256, 256, eng.stream, fv.oe_rp, tri, fv.ivnum, out64);
    GL_CUDA(cudaMemcpyAsync(host_out, out64, sizeof(double) * fv.ivnum, cudaMemcpyDeviceToHost, eng.stream));
    GL_CUDA(cudaStreamSynchronize(eng.stream));
    return GL_OK;
  }
};

}  // namespace

gl_app* make_lcc() { return new LccApp; }

}  // namespace gl
