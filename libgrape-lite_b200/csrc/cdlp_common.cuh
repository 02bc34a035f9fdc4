// cdlp_common.cuh — the label kernels shared by CDLP (app_cdlp.cu) and directed CDLP
// (app_cdlp_directed.cu): labels are 32-bit gids, initialised to the vertex's own gid, gathered
// per CSR entry before the sort, and mapped to oids on output.
#pragma once
#include "apps_common.cuh"

namespace gl {
namespace {

__global__ void k_cdlp_init(uint32_t* label, uint32_t ivnum, uint32_t ovnum,
                            const uint32_t* ovgid, uint32_t fid, int fid_offset) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ivnum) label[i] = (fid << fid_offset) | i;
  else if (i < ivnum + ovnum) label[i] = ovgid[i - ivnum];
}

// scratch[e] = label[col[e]] for every CSR entry (row order preserved)
__global__ void __launch_bounds__(256)
k_cdlp_gather(const uint32_t* __restrict__ col, uint64_t m,
              const uint32_t* __restrict__ label, uint32_t* scratch) {
  const uint64_t stride = (uint64_t) gridDim.x * blockDim.x * 4;
  for (uint64_t i = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) * 4; i < m; i += stride) {
    if (i + 4 <= m) {
      uint4 c = ld_stream_u4((const uint4*) (col + i));
      uint4 o;
      o.x = label[c.x];
      o.y = label[c.y];
      o.z = label[c.z];
      o.w = label[c.w];
      *(uint4*) (scratch + i) = o;
    } else {
      for (uint64_t j = i; j < m; ++j) scratch[j] = label[col[j]];
    }
  }
}

__global__ void k_cdlp_out(const uint32_t* label, uint32_t n, LabelMap lm, int64_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = lm.oid(label[i]);
}

}  // namespace
}  // namespace gl
