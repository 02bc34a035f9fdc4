// vcfrag.cu — device-side construction of a vertex-cut fragment.
//
// Replaces ImmutableVertexcutFragment::Init with the 2-D VCPartitioner
// (grape/fragment/immutable_vertexcut_fragment.h, grape/vertex_map/partitioner.h) for the GPU path:
// filter the block, count both endpoints per local vertex, scan, fill a local CSR of other-endpoint
// local ids, sort the rows.  The reference tiles its edge list into bucket_num x bucket_num buckets
// (GetEdgesOfBucket) so that CPU threads write disjoint vertex ranges; the CSR makes each vertex's
// entries one row, which is what a pull sweep on the GPU reads.
#include <cub/cub.cuh>

#include <cmath>

#include "apps_common.cuh"
#include "rmat.h"
#include "vcfrag.h"

namespace gl {
namespace {

struct VcPart {
  uint64_t n, vchunk;
  uint32_t cs, cd;
  VcRanges r;
  GL_DEV bool in_block(uint64_t a, uint64_t b) const { return a / vchunk == cs && b / vchunk == cd; }
  GL_DEV uint32_t lid(uint64_t v) const { return r.lid(v); }
};

// edge e of a host-supplied list (staged on the device); false when an endpoint is outside [0, n)
struct ListEdges {
  const int64_t* s;
  const int64_t* d;
  GL_DEV bool operator()(uint64_t e, uint64_t n, uint64_t* a, uint64_t* b) const {
    const int64_t x = s[e], y = d[e];
    *a = (uint64_t) x;
    *b = (uint64_t) y;
    return x >= 0 && y >= 0 && (uint64_t) x < n && (uint64_t) y < n;
  }
};
struct RmatEdges {
  int scale;
  uint64_t seed;
  GL_DEV bool operator()(uint64_t e, uint64_t, uint64_t* a, uint64_t* b) const {
    rmat_edge(e, scale, seed, a, b);
    return true;
  }
};

template <class Src>
__global__ void k_vc_count(Src src, uint64_t m, VcPart p, unsigned long long* cnt, unsigned long long* nblock,
                           int* bad) {
  unsigned long long mine = 0;
  for (uint64_t e = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (uint64_t) gridDim.x * blockDim.x) {
    uint64_t a, b;
    if (!src(e, p.n, &a, &b)) {
      *bad = 1;
      continue;
    }
    if (!p.in_block(a, b)) continue;
    atomicAdd(cnt + p.lid(a), 1ull);
    atomicAdd(cnt + p.lid(b), 1ull);
    ++mine;
  }
  mine = warp_sum(mine);
  if (lane_id() == 0 && mine) atomicAdd(nblock, mine);
}

template <class Src>
__global__ void k_vc_fill(Src src, uint64_t m, VcPart p, unsigned long long* cursor, uint32_t* col) {
  for (uint64_t e = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (uint64_t) gridDim.x * blockDim.x) {
    uint64_t a, b;
    if (!src(e, p.n, &a, &b) || !p.in_block(a, b)) continue;
    const uint32_t la = p.lid(a), lb = p.lid(b);
    col[atomicAdd(cursor + la, 1ull)] = lb;
    col[atomicAdd(cursor + lb, 1ull)] = la;
  }
}

int vc_layout(gl_vcfrag* f, uint64_t n, uint32_t fid, uint32_t fnum) {
  const uint32_t side = (uint32_t) llround(std::sqrt((double) fnum));
  if (fnum == 0 || (uint64_t) side * side != fnum) {
    set_error("vertex-cut fragments need a perfect-square fnum, got %u", fnum);
    return GL_ERR_ARG;
  }
  GL_ARG(fid < fnum, "fid must be below fnum");
  GL_ARG(n >= 1, "n_vertices must be at least 1");
  f->fid = fid;
  f->fnum = fnum;
  f->side = side;
  f->n = n;
  f->mvc = (n + fnum - 1) / fnum;
  f->vchunk = f->mvc * side;
  const uint32_t lo = std::min(f->chunk_of_src(), f->chunk_of_dst()), hi = std::max(f->chunk_of_src(), f->chunk_of_dst());
  f->a_begin = f->chunk_begin(lo);
  f->a_end = f->chunk_end(lo);
  f->b_begin = lo == hi ? f->a_end : f->chunk_begin(hi);
  f->b_end = lo == hi ? f->a_end : f->chunk_end(hi);
  const uint64_t nl = (f->a_end - f->a_begin) + (f->b_end - f->b_begin);
  if (nl >= (1ull << 32)) {
    set_error("vertex-cut fragment %u has %llu local vertices (limit 2^32 - 1)", fid, (unsigned long long) nl);
    return GL_ERR_ARG;
  }
  f->nlocal = (uint32_t) nl;
  return GL_OK;
}

template <class Src>
int vc_build(gl_vcfrag* f, const Src& src, uint64_t m) {
  cudaStream_t s = nullptr;
  const uint32_t nl = f->nlocal;
  VcPart p{f->n, f->vchunk, f->chunk_of_src(), f->chunk_of_dst(), f->ranges()};
  DevBuf<unsigned long long> cnt, nblock;
  DevBuf<int> bad;
  GL_CUDA(cnt.alloc((size_t) nl + 1));
  GL_CUDA(nblock.alloc(1));
  GL_CUDA(bad.alloc(1));
  GL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long) * ((size_t) nl + 1), s));
  GL_CUDA(cudaMemsetAsync(nblock, 0, sizeof(unsigned long long), s));
  GL_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
  const int grid = num_sms() * 8;
  if (m) GL_LAUNCH(k_vc_count<Src>, grid, 256, s, src, m, p, cnt, nblock, bad);
  int h_bad = 0;
  unsigned long long h_nblock = 0;
  GL_CUDA(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s));
  GL_CUDA(cudaMemcpyAsync(&h_nblock, nblock, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  GL_CUDA(cudaStreamSynchronize(s));
  if (h_bad) {
    set_error("an edge endpoint lies outside [0, %llu)", (unsigned long long) f->n);
    return GL_ERR_ARG;
  }
  f->block_edges = h_nblock;
  const uint64_t entries = 2 * h_nblock;
  GL_CUDA(f->rp.alloc((size_t) nl + 1));
  {
    size_t tb = 0;
    DevBuf<char> tmp;
    const unsigned long long* in = cnt.get();
    unsigned long long* out = (unsigned long long*) f->rp.get();
    GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, (int64_t) nl + 1, s));
    GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
    GL_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, in, out, (int64_t) nl + 1, s));
  }
  GL_CUDA(f->col.alloc(entries + 16));
  if (entries) {
    GL_CUDA(cudaMemcpyAsync(cnt, f->rp, sizeof(uint64_t) * ((size_t) nl + 1), cudaMemcpyDeviceToDevice, s));
    GL_LAUNCH(k_vc_fill<Src>, grid, 256, s, src, m, p, cnt, f->col);
    GL_TRY(sort_csr_rows(s, f->rp, nl, entries, &f->col));
  }
  GL_CUDA(cudaStreamSynchronize(s));
  return GL_OK;
}

}  // namespace
}  // namespace gl

using namespace gl;

extern "C" {

int gl_vcfrag_create(gl_vcfrag_t** out, const gl_vcfrag_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->n_edges == 0 || (d->src && d->dst), "null edge arrays");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_vcfrag* f = new gl_vcfrag;
  int st = vc_layout(f, d->n_vertices, d->fid, d->fnum);
  if (st == GL_OK) {
    DevBuf<int64_t> s, t;
    const size_t m = d->n_edges;
    if (s.alloc(std::max<size_t>(m, 1)) != cudaSuccess || t.alloc(std::max<size_t>(m, 1)) != cudaSuccess) {
      set_error("gl_vcfrag_create: no device memory for %zu staged edges", m);
      st = GL_ERR_NOMEM;
    } else if (m && (cudaMemcpy(s, d->src, sizeof(int64_t) * m, cudaMemcpyHostToDevice) != cudaSuccess ||
                     cudaMemcpy(t, d->dst, sizeof(int64_t) * m, cudaMemcpyHostToDevice) != cudaSuccess)) {
      set_error("gl_vcfrag_create: edge upload failed");
      st = GL_ERR_CUDA;
    } else {
      st = vc_build(f, ListEdges{s, t}, m);
    }
  }
  if (st != GL_OK) {
    delete f;
    return st;
  }
  *out = f;
  return GL_OK;
}

int gl_vcfrag_build_rmat(gl_vcfrag_t** out, const gl_rmat_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->scale >= 1 && d->scale <= 30, "scale must be in [1,30]");
  GL_ARG(d->edgefactor >= 1, "edgefactor must be at least 1");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_vcfrag* f = new gl_vcfrag;
  int st = vc_layout(f, 1ull << d->scale, d->fid, d->fnum);
  if (st == GL_OK) st = vc_build(f, RmatEdges{d->scale, d->seed}, (uint64_t) d->edgefactor << d->scale);
  if (st != GL_OK) {
    delete f;
    return st;
  }
  *out = f;
  return GL_OK;
}

int gl_vcfrag_get_info(const gl_vcfrag_t* f, gl_vcfrag_info* o) {
  GL_ARG(f && o, "null argument");
  memset(o, 0, sizeof(*o));
  o->fid = f->fid;
  o->fnum = f->fnum;
  o->n_vertices = f->n;
  o->master_begin = f->master_begin(f->fid);
  o->master_end = f->master_end(f->fid);
  o->src_begin = f->chunk_begin(f->chunk_of_src());
  o->src_end = f->chunk_end(f->chunk_of_src());
  o->dst_begin = f->chunk_begin(f->chunk_of_dst());
  o->dst_end = f->chunk_end(f->chunk_of_dst());
  o->local_vnum = f->nlocal;
  o->block_edges = f->block_edges;
  o->entries = f->entries();
  o->device_bytes = sizeof(uint64_t) * ((uint64_t) f->nlocal + 1) + sizeof(uint32_t) * (f->entries() + 16);
  return GL_OK;
}

void gl_vcfrag_destroy(gl_vcfrag_t* f) { delete f; }

}  // extern "C"
