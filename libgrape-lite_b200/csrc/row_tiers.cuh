// row_tiers.cuh — deterministic row sums sum(val[col[p]]) over the rows of a CSR, in three tiers by
// row length, shared by the PageRank variants that must give bit-identical output from run to run.
//
// Every row has one fixed summation order, whatever the scheduling: a row of up to kTierShort
// entries is summed by one thread in sequence, a row of up to kTierChunk entries by one warp (lane
// stride 32, then the xor-shuffle tree of warp_sum), and a longer row in kTierChunk-entry chunks (a
// warp each, as the medium tier) whose sums are folded in chunk order.  k_dense_pull's atomic row
// flushes land in scheduling order, which is why these apps do not use it.
//
// The tiers hand each finished row sum to a consumer, `out(row, sum)`, called once per row by the
// thread that holds the sum; a consumer may keep per-thread state (it is a local of the kernel).
// The callers wrap the device functions below in their own kernels, so each app keeps kernel names
// of its own in profiles.
#pragma once
#include <vector>

#include "apps_common.cuh"

namespace gl {

constexpr uint32_t kTierShort = 32;     // rows up to this length: one thread, sequential sum
constexpr uint32_t kTierChunk = 4096;   // rows up to this length: one warp; longer: chunks of this many entries

// Short and medium rows of [0, nl), grid-stride over groups of 32 rows per warp.  Long rows are
// skipped (TierLongRows).  Every lane of a warp runs the same number of iterations.
template <typename Out>
GL_DEV void tier_rows(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint32_t nl,
                      const double* __restrict__ val, Out& out) {
  const uint32_t lane = lane_id();
  const uint64_t nwarps = (uint64_t) gridDim.x * (blockDim.x / 32);
  for (uint64_t g = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) / 32; g * 32 < nl; g += nwarps) {
    const uint64_t r = g * 32 + lane;
    const bool ok = r < nl;
    const uint64_t b = ok ? rp[r] : 0, e = ok ? rp[r + 1] : 0;
    const uint64_t deg = e - b;
    double s = 0.0;
    if (deg <= kTierShort)
      for (uint64_t p = b; p < e; ++p) s += val[col[p]];
    uint32_t med = __ballot_sync(0xffffffffu, ok && deg > kTierShort && deg <= kTierChunk);
    while (med) {
      const int j = __ffs(med) - 1;
      med &= med - 1;
      const uint64_t rb = __shfl_sync(0xffffffffu, b, j), re = __shfl_sync(0xffffffffu, e, j);
      double t = 0.0;
      for (uint64_t p = rb + lane; p < re; p += 32) t += val[col[p]];
      t = warp_sum(t);
      if ((int) lane == j) s = t;
    }
    if (ok && deg <= kTierChunk) out((uint32_t) r, s);
  }
}

// one warp per kTierChunk-entry chunk [cb[i], ce[i]) of a long row: csum[i] = its sum
GL_DEV void tier_chunks(const uint64_t* __restrict__ cb, const uint64_t* __restrict__ ce, uint32_t nitems,
                        const uint32_t* __restrict__ col, const double* __restrict__ val, double* __restrict__ csum) {
  const uint32_t lane = lane_id();
  const uint32_t nwarps = gridDim.x * (blockDim.x / 32);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) / 32; i < nitems; i += nwarps) {
    double t = 0.0;
    for (uint64_t p = cb[i] + lane; p < ce[i]; p += 32) t += val[col[p]];
    t = warp_sum(t);
    if (lane == 0) csum[i] = t;
  }
}

// one thread per long row j: its chunk sums [off[j], off[j+1]) folded in chunk order (threads past
// nlong fall through, so a caller may synchronise its CTA afterwards)
template <typename Out>
GL_DEV void tier_long(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ off, uint32_t nlong,
                      const double* __restrict__ csum, Out& out) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < nlong) {
    double s = 0.0;
    for (uint32_t i = off[j]; i < off[j + 1]; ++i) s += csum[i];
    out(rows[j], s);
  }
}

// The rows longer than kTierChunk entries and their chunks, planned once from the row pointers.
struct TierLongRows {
  DevBuf<uint64_t> cb, ce;      // chunk items [cb, ce)
  DevBuf<uint32_t> rows, off;   // per long row: its row and its item range [off[j], off[j+1])
  DevBuf<double> csum;          // per item: its sum
  uint32_t nitems = 0, nlong = 0;

  int plan(const uint64_t* d_rp, uint32_t nl) {
    std::vector<uint64_t> rp(nl + 1);
    GL_CUDA(cudaMemcpy(rp.data(), d_rp, sizeof(uint64_t) * (nl + 1), cudaMemcpyDeviceToHost));
    std::vector<uint64_t> b, e;
    std::vector<uint32_t> r, o(1, 0);
    for (uint32_t v = 0; v < nl; ++v) {
      if (rp[v + 1] - rp[v] <= kTierChunk) continue;
      for (uint64_t c = rp[v]; c < rp[v + 1]; c += kTierChunk) {
        b.push_back(c);
        e.push_back(std::min<uint64_t>(c + kTierChunk, rp[v + 1]));
      }
      r.push_back(v);
      o.push_back((uint32_t) b.size());
    }
    nitems = (uint32_t) b.size();
    nlong = (uint32_t) r.size();
    if (!nlong) return GL_OK;
    GL_CUDA(cb.alloc(nitems));
    GL_CUDA(ce.alloc(nitems));
    GL_CUDA(csum.alloc(nitems));
    GL_CUDA(rows.alloc(nlong));
    GL_CUDA(off.alloc(nlong + 1));
    GL_CUDA(cudaMemcpy(cb, b.data(), sizeof(uint64_t) * nitems, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(ce, e.data(), sizeof(uint64_t) * nitems, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(rows, r.data(), sizeof(uint32_t) * nlong, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(off, o.data(), sizeof(uint32_t) * (nlong + 1), cudaMemcpyHostToDevice));
    return GL_OK;
  }
};

}  // namespace gl
