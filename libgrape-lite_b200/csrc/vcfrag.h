// vcfrag.h — device-resident vertex-cut fragment (ImmutableVertexcutFragment with the 2-D
// VCPartitioner, grape/fragment/immutable_vertexcut_fragment.h, grape/vertex_map/partitioner.h).
#pragma once
#include <algorithm>

#include "common.cuh"

namespace gl {
// The local id space of a vertex-cut fragment: range A = [a_begin, a_end) first, then range B
// (which starts at b_begin; empty on a diagonal block).  Shared by the host and the build kernels.
struct VcRanges {
  uint64_t a_begin, a_end, b_begin;
  __host__ __device__ uint32_t lid(uint64_t v) const {
    return (uint32_t) (v < a_end && v >= a_begin ? v - a_begin : (a_end - a_begin) + (v - b_begin));
  }
};
}  // namespace gl

struct gl_vcfrag {
  uint32_t fid = 0, fnum = 1, side = 1;  // side = sqrt(fnum)
  uint64_t n = 0, mvc = 0, vchunk = 0;
  // local vertices: range A then range B (A is the lower chunk; B is empty on a diagonal block)
  uint64_t a_begin = 0, a_end = 0, b_begin = 0, b_end = 0;
  uint64_t block_edges = 0;
  uint32_t nlocal = 0;
  gl::DevBuf<uint64_t> rp;   // [nlocal + 1]
  gl::DevBuf<uint32_t> col;  // [2 * block_edges] local ids of the other endpoints, rows sorted
  uint64_t entries() const { return 2 * block_edges; }
  uint32_t chunk_of_src() const { return fid / side; }
  uint32_t chunk_of_dst() const { return fid % side; }
  uint64_t chunk_begin(uint64_t c) const { return std::min<uint64_t>(c * vchunk, n); }
  uint64_t chunk_end(uint64_t c) const { return std::min<uint64_t>((c + 1) * vchunk, n); }
  uint64_t master_begin(uint32_t f) const { return std::min<uint64_t>((uint64_t) f * mvc, n); }
  uint64_t master_end(uint32_t f) const { return std::min<uint64_t>((uint64_t) (f + 1) * mvc, n); }
  bool holds_chunk(uint32_t c) const { return c == chunk_of_src() || c == chunk_of_dst(); }
  // local id of an oid inside this fragment's local range
  gl::VcRanges ranges() const { return {a_begin, a_end, b_begin}; }
  uint32_t lid(uint64_t v) const { return ranges().lid(v); }
};
