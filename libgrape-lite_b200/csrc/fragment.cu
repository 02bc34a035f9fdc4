// fragment.cu — device-side construction and storage of an edge-cut fragment.
//
// Replaces, for the GPU path, the chain
//   LoadGraph -> EVFragmentLoader -> ImmutableEdgecutFragment::Init -> buildCSR
//   -> HostFragment::__allocate_device_fragment__
// (grape/fragment/loader.h:46-53, immutable_edgecut_fragment.h:215-350,
//  csr_edgecut_fragment_base.h:417-734, grape/cuda/fragment/host_fragment.h:322-438)
// with: emit (row,neighbour) keys -> one 64-bit radix sort -> row pointers by
// binary search.  Layout invariants kept from the reference: rows sorted by
// neighbour lid; inner neighbours first, then outer neighbours in gid order
// (= grouped by owner fid); multi-edges and self loops kept; an undirected
// edge is stored in both endpoints' rows.
#include <cub/cub.cuh>

#include <algorithm>
#include <functional>

#include "dense.cuh"
#include "fragment.h"
#include "rmat.h"

namespace gl {

namespace {

constexpr uint32_t kOuterBit = 0x80000000u;

struct Part {
  uint64_t n, chunk, lo, hi;  // inner = [lo, hi)
  uint32_t fid, fnum;
};

__host__ __device__ inline uint32_t nkey(uint64_t x, uint64_t lo, uint64_t hi) {
  return (x >= lo && x < hi) ? (uint32_t) (x - lo) : (kOuterBit | (uint32_t) x);
}

// ---- chunk producers -------------------------------------------------------
__global__ void k_rmat_chunk(uint64_t first, uint32_t count, int scale,
                             uint64_t seed, int wmode, uint32_t* s, uint32_t* d,
                             float* w) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint64_t a, b;
  rmat_edge(first + i, scale, seed, &a, &b);
  s[i] = (uint32_t) a;
  d[i] = (uint32_t) b;
  if (w) w[i] = rmat_weight(first + i, seed, wmode);
}

// oid -> global index through the ascending oid list (binary search);
// unknown oids -> 0xFFFFFFFF (edge dropped)
__global__ void k_map_oids(const int64_t* in_s, const int64_t* in_d,
                           uint32_t count, const int64_t* oids, uint64_t n,
                           uint32_t* s, uint32_t* d) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  auto find = [&](int64_t o) -> uint32_t {
    if (!oids) return (o >= 0 && (uint64_t) o < n) ? (uint32_t) o : 0xFFFFFFFFu;
    uint64_t l = 0, r = n;
    while (l < r) {
      uint64_t m = (l + r) >> 1;
      if (oids[m] < o) l = m + 1; else r = m;
    }
    return (l < n && oids[l] == o) ? (uint32_t) l : 0xFFFFFFFFu;
  };
  s[i] = find(in_s[i]);
  d[i] = find(in_d[i]);
}

// ---- emission ---------------------------------------------------------------
// For edge (s,d):  oe-buffer gets (s-lo, d) when s is inner; and, undirected,
// (d-lo, s) when d is inner.  Directed: ie-buffer gets (d-lo, s) when d inner.
__global__ void k_count(const uint32_t* s, const uint32_t* d, uint32_t count,
                        Part p, int directed, uint32_t* c_oe, uint32_t* c_ie) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint32_t a = s[i], b = d[i];
  bool ok = a != 0xFFFFFFFFu && b != 0xFFFFFFFFu;
  bool ia = ok && a >= p.lo && a < p.hi, ib = ok && b >= p.lo && b < p.hi;
  if (directed) {
    c_oe[i] = ia;
    c_ie[i] = ib;
  } else {
    c_oe[i] = (uint32_t) ia + (uint32_t) ib;
  }
}

template <typename W>
__global__ void k_emit(const uint32_t* s, const uint32_t* d, const W* w,
                       uint32_t count, Part p, int directed,
                       const uint32_t* pos_oe, const uint32_t* pos_ie,
                       uint64_t base_oe, uint64_t base_ie, uint64_t* k_oe,
                       W* w_oe, uint64_t* k_ie, W* w_ie) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint32_t a = s[i], b = d[i];
  if (a == 0xFFFFFFFFu || b == 0xFFFFFFFFu) return;
  bool ia = a >= p.lo && a < p.hi, ib = b >= p.lo && b < p.hi;
  uint64_t q = base_oe + pos_oe[i];
  if (ia) {
    k_oe[q] = ((uint64_t) (a - p.lo) << 32) | nkey(b, p.lo, p.hi);
    if (w) w_oe[q] = w[i];
    ++q;
  }
  if (directed) {
    if (ib) {
      uint64_t r = base_ie + pos_ie[i];
      k_ie[r] = ((uint64_t) (b - p.lo) << 32) | nkey(a, p.lo, p.hi);
      if (w) w_ie[r] = w[i];
    }
  } else if (ib) {
    k_oe[q] = ((uint64_t) (b - p.lo) << 32) | nkey(a, p.lo, p.hi);
    if (w) w_oe[q] = w[i];
  }
}

__global__ void k_outer_flags(const uint64_t* keys, uint64_t m, uint32_t* out,
                              uint8_t* flag) {
  uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  uint32_t lo32 = (uint32_t) keys[i];
  flag[i] = (lo32 & kOuterBit) ? 1 : 0;
  out[i] = lo32 & ~kOuterBit;
}

__device__ inline uint64_t lower_bound_u64(const uint64_t* a, uint64_t n,
                                           uint64_t key) {
  uint64_t l = 0, r = n;
  while (l < r) {
    uint64_t m = (l + r) >> 1;
    if (a[m] < key) l = m + 1; else r = m;
  }
  return l;
}
__device__ inline uint32_t lower_bound_u32(const uint32_t* a, uint32_t n,
                                           uint32_t key) {
  uint32_t l = 0, r = n;
  while (l < r) {
    uint32_t m = (l + r) >> 1;
    if (a[m] < key) l = m + 1; else r = m;
  }
  return l;
}

__global__ void k_rowptr(const uint64_t* keys, uint64_t m, uint32_t rows,
                         uint64_t* rp, uint64_t* split) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > rows) return;
  rp[r] = lower_bound_u64(keys, m, (uint64_t) r << 32);
  if (r < rows)
    split[r] = lower_bound_u64(keys, m, ((uint64_t) r << 32) | kOuterBit);
}

__global__ void k_cols(const uint64_t* keys, uint64_t m, uint32_t ivnum,
                       const uint32_t* outer_sorted, uint32_t ovnum,
                       uint32_t* col) {
  uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  uint32_t lo32 = (uint32_t) keys[i];
  if (lo32 & kOuterBit) {
    col[i] = ivnum + lower_bound_u32(outer_sorted, ovnum, lo32 & ~kOuterBit);
  } else {
    col[i] = lo32;
  }
}

__global__ void k_ovgid(const uint32_t* outer_sorted, uint32_t ovnum,
                        uint64_t chunk, int fid_offset, uint32_t* ovgid) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ovnum) return;
  uint32_t g = outer_sorted[i];
  uint32_t f = (uint32_t) (g / chunk);
  ovgid[i] = (f << fid_offset) | (uint32_t) (g - (uint64_t) f * chunk);
}

__global__ void k_outer_range(const uint32_t* ovgid, uint32_t ovnum,
                              uint32_t ivnum, uint32_t fnum, int fid_offset,
                              uint32_t* range) {
  uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > fnum) return;
  uint32_t p = ovnum;
  if (f < fnum) p = lower_bound_u32(ovgid, ovnum, f << fid_offset);
  range[f] = ivnum + p;
}

__global__ void k_degree_stats(const uint64_t* rp, uint32_t rows,
                               unsigned long long* best, uint32_t* nz) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  bool has = false;
  unsigned long long v = 0;
  if (r < rows) {
    uint64_t dg = rp[r + 1] - rp[r];
    has = dg > 0;
    if (dg > 0xFFFFFFFFull) dg = 0xFFFFFFFFull;
    v = (dg << 32) | (0xFFFFFFFFu - r);
  }
  for (int o = 16; o; o >>= 1) {
    unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t > v ? t : v;
  }
  if ((threadIdx.x & 31) == 0 && v) atomicMax(best, v);
  uint32_t word = __ballot_sync(0xffffffffu, has);
  if ((threadIdx.x & 31) == 0 && (r >> 5) < ((rows + 31) >> 5)) nz[r >> 5] = word;
}

// reverse adjacency of outer vertices: (outer idx, inner row) from oe entries
__global__ void k_ovie_count(const uint32_t* col, uint64_t m, uint32_t ivnum,
                             uint8_t* flag) {
  uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  flag[i] = col[i] >= ivnum;
}
__global__ void k_ovie_keys(const uint64_t* rp, uint32_t rows,
                            const uint32_t* col, const uint64_t* split,
                            uint32_t ivnum, const uint64_t* pos_of_row,
                            uint64_t* keys) {
  // one thread per row: outer part of the row is [split[r], rp[r+1])
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  uint64_t o = pos_of_row[r];
  for (uint64_t e = split[r]; e < rp[r + 1]; ++e)
    keys[o++] = ((uint64_t) (col[e] - ivnum) << 32) | r;
}
__global__ void k_outer_deg(const uint64_t* rp, const uint64_t* split,
                            uint32_t rows, uint64_t* cnt) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  cnt[r] = rp[r + 1] - split[r];
}
__global__ void k_low32(const uint64_t* keys, uint64_t m, uint32_t* out) {
  uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) out[i] = (uint32_t) keys[i];
}
__global__ void k_split_from_cols(const uint64_t* rp, const uint32_t* col,
                                  uint32_t rows, uint32_t ivnum,
                                  uint64_t* split) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  uint64_t l = rp[r], h = rp[r + 1];
  while (l < h) {
    uint64_t m = (l + h) >> 1;
    if (col[m] < ivnum) l = m + 1; else h = m;
  }
  split[r] = l;
}

inline unsigned nblk(uint64_t n, unsigned t = 256) {
  return (unsigned) ((n + t - 1) / t);
}

// The builder's buffers take at least 16 bytes, so that an empty one is still a valid pointer.
template <typename T>
cudaError_t alloc16(DevBuf<T>& b, size_t n) {
  return b.alloc(n ? n : 16 / sizeof(T));
}

int sort_keys_u64(uint64_t*& keys, uint64_t*& alt, void*& vals, void*& vals_alt,
                  int vbytes, uint64_t m, int end_bit) {
  if (m == 0) return GL_OK;
  size_t tmp_bytes = 0;
  DevBuf<char> tmp;
  if (vbytes == 0) {
    cub::DoubleBuffer<uint64_t> kb(keys, alt);
    GL_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, kb, (int64_t) m, 0, end_bit));
    GL_CUDA(alloc16(tmp, tmp_bytes));
    GL_CUDA(cub::DeviceRadixSort::SortKeys(tmp.get(), tmp_bytes, kb, (int64_t) m, 0, end_bit));
    if (kb.Current() != keys) std::swap(keys, alt);
  } else if (vbytes == 4) {
    cub::DoubleBuffer<uint64_t> kb(keys, alt);
    cub::DoubleBuffer<uint32_t> vb((uint32_t*) vals, (uint32_t*) vals_alt);
    GL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, kb, vb, (int64_t) m, 0, end_bit));
    GL_CUDA(alloc16(tmp, tmp_bytes));
    GL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tmp_bytes, kb, vb, (int64_t) m, 0, end_bit));
    if (kb.Current() != keys) std::swap(keys, alt);
    if ((void*) vb.Current() != vals) std::swap(vals, vals_alt);
  } else {
    cub::DoubleBuffer<uint64_t> kb(keys, alt);
    cub::DoubleBuffer<uint64_t> vb((uint64_t*) vals, (uint64_t*) vals_alt);
    GL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, kb, vb, (int64_t) m, 0, end_bit));
    GL_CUDA(alloc16(tmp, tmp_bytes));
    GL_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tmp_bytes, kb, vb, (int64_t) m, 0, end_bit));
    if (kb.Current() != keys) std::swap(keys, alt);
    if ((void*) vb.Current() != vals) std::swap(vals, vals_alt);
  }
  GL_CUDA(cudaDeviceSynchronize());
  return GL_OK;
}

int bits_for(uint64_t x) {
  int b = 0;
  while (x) {
    ++b;
    x >>= 1;
  }
  return b ? b : 1;
}

// A producer fills device arrays (s, d, w) for edges [first, first+count).
struct Producer {
  virtual ~Producer() {}
  virtual uint64_t total() const = 0;
  virtual int fill(uint64_t first, uint32_t count, uint32_t* s, uint32_t* d,
                   void* w) = 0;
};

struct RmatProducer : Producer {
  gl_rmat_desc d;
  uint64_t total() const override { return (uint64_t) d.edgefactor << d.scale; }
  int fill(uint64_t first, uint32_t count, uint32_t* s, uint32_t* dd,
           void* w) override {
    k_rmat_chunk<<<nblk(count), 256>>>(first, count, d.scale, d.seed,
                                       d.weight_mode, s, dd, (float*) w);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
    return GL_OK;
  }
};

struct HostProducer : Producer {
  const gl_edges_desc* d;
  const int64_t* d_oids = nullptr;
  DevBuf<int64_t> ts, td;
  uint64_t total() const override { return d->n_edges; }
  int fill(uint64_t first, uint32_t count, uint32_t* s, uint32_t* dd,
           void* w) override {
    if (!ts) {
      GL_CUDA(alloc16(ts, (size_t) (1u << 24)));
      GL_CUDA(alloc16(td, (size_t) (1u << 24)));
    }
    GL_CUDA(cudaMemcpy(ts.get(), d->src + first, sizeof(int64_t) * count, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(td.get(), d->dst + first, sizeof(int64_t) * count, cudaMemcpyHostToDevice));
    k_map_oids<<<nblk(count), 256>>>(ts.get(), td.get(), count,
                                     d_oids, d->n_vertices, s, dd);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
    if (w && d->edata)
      GL_CUDA(cudaMemcpy(w, (const char*) d->edata + first * d->edata_bytes,
                         (size_t) d->edata_bytes * count, cudaMemcpyHostToDevice));
    return GL_OK;
  }
};

int finish_common(gl_frag* f);
int build_ovie(gl_frag* f);

// The builder proper.
int build_from_producer(gl_frag* f, Producer& prod, uint64_t n, int directed,
                        int edata_bytes) {
  const uint32_t CH = 1u << 24;
  Part p;
  p.n = n;
  p.fid = f->fid;
  p.fnum = f->fnum;
  p.chunk = (n + f->fnum - 1) / f->fnum;
  p.lo = std::min<uint64_t>(n, (uint64_t) f->fid * p.chunk);
  p.hi = std::min<uint64_t>(n, p.lo + p.chunk);
  GL_ARG(n < (1ull << 31), "n_vertices must be < 2^31");
  f->ivnum = (uint32_t) (p.hi - p.lo);
  f->part_chunk = p.chunk;
  f->total_vnum = n;
  f->directed = directed;
  f->edata_bytes = edata_bytes;
  id_parser_init(f->fnum, &f->fid_offset, &f->id_mask);
  GL_ARG(p.chunk <= (uint64_t) f->id_mask + 1, "fragment too large for 32-bit gid");

  const uint64_t E = prod.total();
  DevBuf<uint32_t> bs, bd, c_oe, c_ie;
  DevBuf<char> bw, scan_tmp;
  GL_CUDA(alloc16(bs, (size_t) CH));
  GL_CUDA(alloc16(bd, (size_t) CH));
  if (edata_bytes) GL_CUDA(alloc16(bw, (size_t) edata_bytes * CH));
  GL_CUDA(alloc16(c_oe, (size_t) (CH + 1)));
  GL_CUDA(alloc16(c_ie, (size_t) (CH + 1)));
  size_t scan_bytes = 0;
  GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, c_oe.get(),
                                        c_oe.get(), (int) (CH + 1)));
  GL_CUDA(alloc16(scan_tmp, scan_bytes));

  // pass 1: totals
  std::vector<uint64_t> base_oe, base_ie;
  uint64_t m_oe = 0, m_ie = 0;
  for (uint64_t first = 0; first < E; first += CH) {
    uint32_t cnt = (uint32_t) std::min<uint64_t>(CH, E - first);
    GL_TRY(prod.fill(first, cnt, bs.get(), bd.get(), nullptr));
    GL_CUDA(cudaMemsetAsync(c_oe.get(), 0, sizeof(uint32_t) * (cnt + 1)));
    GL_CUDA(cudaMemsetAsync(c_ie.get(), 0, sizeof(uint32_t) * (cnt + 1)));
    k_count<<<nblk(cnt), 256>>>(bs.get(), bd.get(), cnt, p,
                                directed, c_oe.get(), c_ie.get());
    GL_COUNT_LAUNCH();
    GL_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp.get(), scan_bytes, c_oe.get(),
                                          c_oe.get(), (int) (cnt + 1)));
    GL_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp.get(), scan_bytes, c_ie.get(),
                                          c_ie.get(), (int) (cnt + 1)));
    uint32_t t_oe = 0, t_ie = 0;
    GL_CUDA(cudaMemcpy(&t_oe, c_oe.get() + cnt, 4, cudaMemcpyDeviceToHost));
    GL_CUDA(cudaMemcpy(&t_ie, c_ie.get() + cnt, 4, cudaMemcpyDeviceToHost));
    base_oe.push_back(m_oe);
    base_ie.push_back(m_ie);
    m_oe += t_oe;
    m_ie += t_ie;
  }

  // pass 2: emit keys (+weights)
  DevBuf<uint64_t> k_oe, k_oe2, k_ie, k_ie2;
  DevBuf<char> w_oe, w_oe2, w_ie, w_ie2;
  GL_CUDA(alloc16(k_oe, m_oe));
  GL_CUDA(alloc16(k_oe2, m_oe));
  if (edata_bytes) {
    GL_CUDA(alloc16(w_oe, (size_t) edata_bytes * m_oe + 64));
    GL_CUDA(alloc16(w_oe2, (size_t) edata_bytes * m_oe + 64));
  }
  if (directed) {
    GL_CUDA(alloc16(k_ie, m_ie));
    GL_CUDA(alloc16(k_ie2, m_ie));
    if (edata_bytes) {
      GL_CUDA(alloc16(w_ie, (size_t) edata_bytes * m_ie + 64));
      GL_CUDA(alloc16(w_ie2, (size_t) edata_bytes * m_ie + 64));
    }
  }
  size_t ci = 0;
  for (uint64_t first = 0; first < E; first += CH, ++ci) {
    uint32_t cnt = (uint32_t) std::min<uint64_t>(CH, E - first);
    GL_TRY(prod.fill(first, cnt, bs.get(), bd.get(), bw.get()));
    GL_CUDA(cudaMemsetAsync(c_oe.get(), 0, sizeof(uint32_t) * (cnt + 1)));
    GL_CUDA(cudaMemsetAsync(c_ie.get(), 0, sizeof(uint32_t) * (cnt + 1)));
    k_count<<<nblk(cnt), 256>>>(bs.get(), bd.get(), cnt, p,
                                directed, c_oe.get(), c_ie.get());
    GL_COUNT_LAUNCH();
    GL_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp.get(), scan_bytes, c_oe.get(),
                                          c_oe.get(), (int) (cnt + 1)));
    GL_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp.get(), scan_bytes, c_ie.get(),
                                          c_ie.get(), (int) (cnt + 1)));
    if (edata_bytes == 8) {
      k_emit<double><<<nblk(cnt), 256>>>(
          bs.get(), bd.get(), (double*) bw.get(), cnt, p, directed,
          c_oe.get(), c_ie.get(), base_oe[ci], base_ie[ci],
          k_oe.get(), (double*) w_oe.get(), k_ie.get(), (double*) w_ie.get());
    } else {
      k_emit<float><<<nblk(cnt), 256>>>(
          bs.get(), bd.get(), (float*) bw.get(), cnt, p, directed,
          c_oe.get(), c_ie.get(), base_oe[ci], base_ie[ci],
          k_oe.get(), (float*) w_oe.get(), k_ie.get(), (float*) w_ie.get());
    }
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  GL_CUDA(cudaDeviceSynchronize());
  // free chunk scratch before the big sorts
  bs.reset();
  bd.reset();
  bw.reset();
  c_oe.reset();
  c_ie.reset();

  const int end_bit = 32 + bits_for(f->ivnum);
  {
    uint64_t *a = k_oe, *b = k_oe2;
    void *va = w_oe, *vb = w_oe2;
    GL_TRY(sort_keys_u64(a, b, va, vb, edata_bytes, m_oe, end_bit));
    if (a != k_oe.get()) std::swap(k_oe, k_oe2);
    if (va != w_oe.get()) std::swap(w_oe, w_oe2);
  }
  if (directed) {
    uint64_t *a = k_ie, *b = k_ie2;
    void *va = w_ie, *vb = w_ie2;
    GL_TRY(sort_keys_u64(a, b, va, vb, edata_bytes, m_ie, end_bit));
    if (a != k_ie.get()) std::swap(k_ie, k_ie2);
    if (va != w_ie.get()) std::swap(w_ie, w_ie2);
  }
  k_oe2.reset();
  w_oe2.reset();
  k_ie2.reset();
  w_ie2.reset();

  // outer vertex set = distinct neighbours with the outer bit (both CSRs)
  DevBuf<uint32_t> outer_sorted;
  uint32_t ovnum = 0;
  if (f->fnum > 1) {
    uint64_t m_all = m_oe + m_ie;
    DevBuf<uint32_t> cand, sel;
    DevBuf<uint8_t> flag;
    DevBuf<uint64_t> nsel;
    DevBuf<char> tmp;
    GL_CUDA(alloc16(cand, m_all));
    GL_CUDA(alloc16(flag, m_all));
    GL_CUDA(alloc16(sel, m_all));
    GL_CUDA(alloc16(nsel, 1));
    if (m_oe) k_outer_flags<<<nblk(m_oe), 256>>>(k_oe.get(), m_oe, cand.get(), flag.get());
    if (m_ie) k_outer_flags<<<nblk(m_ie), 256>>>(k_ie.get(), m_ie, cand.get() + m_oe, flag.get() + m_oe);
    GL_COUNT_LAUNCH();
    size_t tb = 0;
    GL_CUDA(cub::DeviceSelect::Flagged(nullptr, tb, cand.get(), flag.get(), sel.get(), nsel.get(), (int64_t) m_all));
    GL_CUDA(alloc16(tmp, tb));
    GL_CUDA(cub::DeviceSelect::Flagged(tmp.get(), tb, cand.get(), flag.get(), sel.get(), nsel.get(), (int64_t) m_all));
    uint64_t n_out = 0;
    GL_CUDA(cudaMemcpy(&n_out, nsel.get(), 8, cudaMemcpyDeviceToHost));
    flag.reset();
    tmp.reset();
    if (n_out) {
      // sort + unique
      size_t sb = 0;
      cub::DoubleBuffer<uint32_t> db(sel.get(), cand.get());
      GL_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sb, db, (int64_t) n_out, 0, bits_for(n)));
      DevBuf<char> st;
      GL_CUDA(alloc16(st, sb));
      GL_CUDA(cub::DeviceRadixSort::SortKeys(st.get(), sb, db, (int64_t) n_out, 0, bits_for(n)));
      uint32_t* sorted = db.Current();
      uint32_t* other = db.Alternate();
      size_t ub = 0;
      GL_CUDA(cub::DeviceSelect::Unique(nullptr, ub, sorted, other, nsel.get(), (int64_t) n_out));
      DevBuf<char> ut;
      GL_CUDA(alloc16(ut, ub));
      GL_CUDA(cub::DeviceSelect::Unique(ut.get(), ub, sorted, other, nsel.get(), (int64_t) n_out));
      uint64_t nu = 0;
      GL_CUDA(cudaMemcpy(&nu, nsel.get(), 8, cudaMemcpyDeviceToHost));
      ovnum = (uint32_t) nu;
      GL_CUDA(alloc16(outer_sorted, nu));
      GL_CUDA(cudaMemcpy(outer_sorted.get(), other, sizeof(uint32_t) * nu, cudaMemcpyDeviceToDevice));
    }
  }
  f->ovnum = ovnum;
  GL_ARG((uint64_t) f->ivnum + ovnum < (1ull << 32), "too many local vertices");

  auto finish_csr = [&](DevBuf<uint64_t>& keys, DevBuf<char>& w, uint64_t m, DevCsr& out) -> int {
    out.rows = f->ivnum;
    out.entries = m;
    GL_CUDA(cudaMalloc(&out.rp, sizeof(uint64_t) * ((size_t) f->ivnum + 1)));
    GL_CUDA(cudaMalloc(&out.split, sizeof(uint64_t) * std::max<size_t>(f->ivnum, 1)));
    GL_CUDA(cudaMalloc(&out.col, sizeof(uint32_t) * (m + 16)));
    k_rowptr<<<nblk((uint64_t) f->ivnum + 1), 256>>>(keys.get(), m, f->ivnum, out.rp, out.split);
    if (m) k_cols<<<nblk(m), 256>>>(keys.get(), m, f->ivnum, outer_sorted.get(), ovnum, out.col);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaDeviceSynchronize());
    out.w = w.release();
    f->device_bytes += sizeof(uint64_t) * (2 * (size_t) f->ivnum + 1) + sizeof(uint32_t) * m + (size_t) edata_bytes * m;
    keys.reset();
    return GL_OK;
  };
  GL_TRY(finish_csr(k_oe, w_oe, m_oe, f->oe));
  if (directed) {
    GL_TRY(finish_csr(k_ie, w_ie, m_ie, f->ie));
    f->ie_alias_oe = false;
  } else {
    f->ie = f->oe;
    f->ie_alias_oe = true;
  }
  if (ovnum) {
    GL_CUDA(cudaMalloc(&f->ovgid, sizeof(uint32_t) * ovnum));
    k_ovgid<<<nblk(ovnum), 256>>>(outer_sorted.get(), ovnum, p.chunk, f->fid_offset, f->ovgid);
    GL_COUNT_LAUNCH();
    f->device_bytes += sizeof(uint32_t) * ovnum;
  }
  return finish_common(f);
}

int finish_common(gl_frag* f) {
  // outer ranges per owner fid
  GL_CUDA(cudaMalloc(&f->outer_range, sizeof(uint32_t) * (f->fnum + 1)));
  k_outer_range<<<1, 256>>>(f->ovgid, f->ovnum, f->ivnum, f->fnum, f->fid_offset, f->outer_range);
  GL_COUNT_LAUNCH();
  f->h_outer_range.resize(f->fnum + 1);
  GL_CUDA(cudaMemcpy(f->h_outer_range.data(), f->outer_range, sizeof(uint32_t) * (f->fnum + 1), cudaMemcpyDeviceToHost));
  // degree stats + non-isolated bitmap
  size_t words = ((size_t) f->ivnum + 31) / 32;
  GL_CUDA(cudaMalloc(&f->nonzero_deg, sizeof(uint32_t) * std::max<size_t>(words, 1)));
  GL_CUDA(cudaMemset(f->nonzero_deg, 0, sizeof(uint32_t) * std::max<size_t>(words, 1)));
  DevBuf<unsigned long long> best;
  GL_CUDA(alloc16(best, 1));
  GL_CUDA(cudaMemset(best.get(), 0, 8));
  if (f->ivnum) {
    k_degree_stats<<<nblk(((uint64_t) f->ivnum + 31) / 32 * 32), 256>>>(f->oe.rp, f->ivnum, best.get(), f->nonzero_deg);
    GL_COUNT_LAUNCH();
  }
  unsigned long long hb = 0;
  GL_CUDA(cudaMemcpy(&hb, best.get(), 8, cudaMemcpyDeviceToHost));
  f->max_degree = (uint32_t) (hb >> 32);
  f->max_degree_lid = f->ivnum ? 0xFFFFFFFFu - (uint32_t) hb : 0;
  f->device_bytes += words * 4;
  if (f->ovnum) GL_TRY(build_ovie(f));
  // tile -> first row table of the dense sweeps
  f->oe_ntiles = (uint32_t) ((f->oe.entries + kDenseTile - 1) / kDenseTile);
  GL_CUDA(cudaMalloc(&f->oe_tile_row, sizeof(uint32_t) * ((size_t) f->oe_ntiles + 1)));
  k_dense_tile_rows<<<nblk((uint64_t) f->oe_ntiles + 1), 256>>>(f->oe.rp, f->ivnum, f->oe.entries, f->oe_ntiles, f->oe_tile_row);
  GL_COUNT_LAUNCH();
  f->device_bytes += sizeof(uint32_t) * ((size_t) f->oe_ntiles + 1);
  GL_CUDA(cudaDeviceSynchronize());
  return GL_OK;
}

int build_ovie(gl_frag* f) {
  // entries of oe whose neighbour is outer: count per row, scan, emit, sort
  const uint32_t rows = f->ivnum;
  DevBuf<uint64_t> cnt, pos;
  DevBuf<char> tmp;
  GL_CUDA(alloc16(cnt, ((size_t) rows + 1)));
  GL_CUDA(alloc16(pos, ((size_t) rows + 1)));
  GL_CUDA(cudaMemset(cnt.get(), 0, sizeof(uint64_t) * ((size_t) rows + 1)));
  k_outer_deg<<<nblk(rows), 256>>>(f->oe.rp, f->oe.split, rows, cnt.get());
  GL_COUNT_LAUNCH();
  size_t tb = 0;
  GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.get(), pos.get(), (int) (rows + 1)));
  GL_CUDA(alloc16(tmp, tb));
  GL_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, cnt.get(), pos.get(), (int) (rows + 1)));
  uint64_t m = 0;
  GL_CUDA(cudaMemcpy(&m, pos.get() + rows, 8, cudaMemcpyDeviceToHost));
  DevBuf<uint64_t> keys, keys2;
  GL_CUDA(alloc16(keys, m));
  GL_CUDA(alloc16(keys2, m));
  k_ovie_keys<<<nblk(rows), 256>>>(f->oe.rp, rows, f->oe.col, f->oe.split, f->ivnum, pos.get(), keys.get());
  GL_COUNT_LAUNCH();
  uint64_t *a = keys, *b = keys2;
  void *va = nullptr, *vb = nullptr;
  GL_TRY(sort_keys_u64(a, b, va, vb, 0, m, 32 + bits_for(f->ovnum)));
  if (a != keys.get()) std::swap(keys, keys2);
  DevCsr& o = f->ovie;
  o.rows = f->ovnum;
  o.entries = m;
  GL_CUDA(cudaMalloc(&o.rp, sizeof(uint64_t) * ((size_t) f->ovnum + 1)));
  GL_CUDA(cudaMalloc(&o.split, sizeof(uint64_t) * std::max<size_t>(f->ovnum, 1)));
  GL_CUDA(cudaMalloc(&o.col, sizeof(uint32_t) * (m + 16)));
  k_rowptr<<<nblk((uint64_t) f->ovnum + 1), 256>>>(keys.get(), m, f->ovnum, o.rp, o.split);
  if (m) k_low32<<<nblk(m), 256>>>(keys.get(), m, o.col);
  GL_COUNT_LAUNCH();
  GL_CUDA(cudaDeviceSynchronize());
  f->device_bytes += sizeof(uint64_t) * ((size_t) f->ovnum + 1) + sizeof(uint32_t) * m;
  return GL_OK;
}

}  // namespace

void frag_fill_view(const gl_frag* f, gl_frag_view* v) {
  memset(v, 0, sizeof(*v));
  v->fid = f->fid;
  v->fnum = f->fnum;
  v->ivnum = f->ivnum;
  v->ovnum = f->ovnum;
  v->total_vnum = f->total_vnum;
  v->directed = f->directed;
  v->edata_bytes = f->edata_bytes;
  v->fid_offset = f->fid_offset;
  v->id_mask = f->id_mask;
  v->oe_rp = f->oe.rp;
  v->oe_col = f->oe.col;
  v->oe_w = f->oe.w;
  v->oe_split = f->oe.split;
  v->ie_rp = f->ie.rp;
  v->ie_col = f->ie.col;
  v->ie_w = f->ie.w;
  v->ie_split = f->ie.split;
  v->ovie_rp = f->ovie.rp;
  v->ovie_col = f->ovie.col;
  v->ovgid = f->ovgid;
  v->outer_range = f->outer_range;
  v->inner_oids = f->inner_oids;
  v->oid_base = f->oid_base;
  v->oe_num = f->oe.entries;
  v->ie_num = f->ie.entries;
}

}  // namespace gl

using namespace gl;

extern "C" {

int gl_frag_build_rmat(gl_frag_t** out, const gl_rmat_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->scale >= 1 && d->scale <= 30, "scale must be in [1,30]");
  GL_ARG(d->fnum >= 1 && d->fid < d->fnum, "bad fid/fnum");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_frag* f = new gl_frag;
  f->fid = d->fid;
  f->fnum = d->fnum;
  f->load_strategy = GL_LOAD_ONLY_OUT;
  RmatProducer prod;
  prod.d = *d;
  uint64_t n = 1ull << d->scale;
  int st = build_from_producer(f, prod, n, 0, d->weight_mode ? 4 : 0);
  if (st != GL_OK) {
    gl_frag_destroy(f);
    return st;
  }
  uint64_t chunk = (n + d->fnum - 1) / d->fnum;
  f->oid_base = (int64_t) (chunk * d->fid);
  *out = f;
  return GL_OK;
}

int gl_rmat_edges_host(const gl_rmat_desc* d, uint64_t first, uint64_t count,
                       int64_t* src, int64_t* dst, float* w) {
  GL_ARG(d && src && dst, "null argument");
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t) count; ++i) {
    uint64_t a, b;
    rmat_edge(first + i, d->scale, d->seed, &a, &b);
    src[i] = (int64_t) a;
    dst[i] = (int64_t) b;
    if (w) w[i] = rmat_weight(first + i, d->seed, d->weight_mode);
  }
  return GL_OK;
}

int gl_frag_build_from_edges(gl_frag_t** out, const gl_edges_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->fnum >= 1 && d->fid < d->fnum, "bad fid/fnum");
  GL_ARG(d->edata_bytes == 0 || d->edata_bytes == 4 || d->edata_bytes == 8, "edata_bytes must be 0, 4 or 8");
  GL_ARG(d->n_edges == 0 || (d->src && d->dst), "null edge arrays");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_frag* f = new gl_frag;
  f->fid = d->fid;
  f->fnum = d->fnum;
  f->load_strategy = d->load_strategy;
  HostProducer prod;
  prod.d = d;
  DevBuf<int64_t> d_oids;
  if (d->oids) {
    if (d_oids.alloc(std::max<uint64_t>(d->n_vertices, 1)) != cudaSuccess ||
        cudaMemcpy(d_oids, d->oids, sizeof(int64_t) * d->n_vertices, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("oid upload failed");
      delete f;
      return GL_ERR_CUDA;
    }
    prod.d_oids = d_oids;
  }
  int st = build_from_producer(f, prod, d->n_vertices, d->directed ? 1 : 0,
                               d->edata ? d->edata_bytes : 0);
  if (st != GL_OK) {
    gl_frag_destroy(f);
    return st;
  }
  uint64_t chunk = (d->n_vertices + d->fnum - 1) / d->fnum;
  uint64_t lo = std::min<uint64_t>(d->n_vertices, chunk * d->fid);
  if (d->oids) {
    f->h_inner_oids.assign(d->oids + lo, d->oids + lo + f->ivnum);
    if (f->ivnum) {
      if (cudaMalloc(&f->inner_oids, sizeof(int64_t) * f->ivnum) != cudaSuccess ||
          cudaMemcpy(f->inner_oids, f->h_inner_oids.data(), sizeof(int64_t) * f->ivnum, cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("inner oid upload failed");
        gl_frag_destroy(f);
        return GL_ERR_CUDA;
      }
    }
  } else {
    f->oid_base = (int64_t) lo;
  }
  *out = f;
  return GL_OK;
}

int gl_frag_create(gl_frag_t** out, const gl_frag_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->fnum >= 1 && d->fid < d->fnum, "bad fid/fnum");
  GL_ARG(d->edata_bytes == 0 || d->edata_bytes == 4 || d->edata_bytes == 8, "edata_bytes must be 0, 4 or 8");
  GL_ARG(d->oe.row_ptr && d->oe.rows == d->ivnum, "oe must describe ivnum rows");
  GL_ARG(d->ovnum == 0 || d->ovgid, "ovgid required when ovnum > 0");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_frag* f = new gl_frag;
  f->fid = d->fid;
  f->fnum = d->fnum;
  f->directed = d->directed;
  f->load_strategy = d->load_strategy;
  f->ivnum = d->ivnum;
  f->ovnum = d->ovnum;
  f->total_vnum = d->total_vnum;
  f->edata_bytes = d->edata_bytes;
  f->oid_base = d->oid_base;
  id_parser_init(f->fnum, &f->fid_offset, &f->id_mask);
  auto fail = [&](int st) {
    gl_frag_destroy(f);
    return st;
  };
  auto upload = [&](const gl_csr_desc& c, DevCsr& o, bool has_w) -> int {
    uint64_t m = c.row_ptr[c.rows];
    o.rows = c.rows;
    o.entries = m;
    GL_CUDA(cudaMalloc(&o.rp, sizeof(uint64_t) * (c.rows + 1)));
    GL_CUDA(cudaMemcpy(o.rp, c.row_ptr, sizeof(uint64_t) * (c.rows + 1), cudaMemcpyHostToDevice));
    GL_CUDA(cudaMalloc(&o.col, sizeof(uint32_t) * (m + 16)));
    if (m) GL_CUDA(cudaMemcpy(o.col, c.col, sizeof(uint32_t) * m, cudaMemcpyHostToDevice));
    if (has_w && c.edata && m) {
      GL_CUDA(cudaMalloc(&o.w, (size_t) d->edata_bytes * m + 64));   // +64: bulk copies round up to 16 bytes
      GL_CUDA(cudaMemcpy(o.w, c.edata, (size_t) d->edata_bytes * m, cudaMemcpyHostToDevice));
    }
    GL_CUDA(cudaMalloc(&o.split, sizeof(uint64_t) * std::max<uint64_t>(c.rows, 1)));
    if (c.rows) {
      k_split_from_cols<<<nblk(c.rows), 256>>>(o.rp, o.col, (uint32_t) c.rows, d->ivnum, o.split);
      GL_COUNT_LAUNCH();
    }
    f->device_bytes += sizeof(uint64_t) * (2 * c.rows + 1) + (4 + (o.w ? d->edata_bytes : 0)) * m;
    return GL_OK;
  };
  int st = upload(d->oe, f->oe, d->edata_bytes != 0);
  if (st != GL_OK) return fail(st);
  if (d->directed && d->ie.row_ptr) {
    st = upload(d->ie, f->ie, d->edata_bytes != 0);
    if (st != GL_OK) return fail(st);
    f->ie_alias_oe = false;
  } else {
    f->ie = f->oe;
    f->ie_alias_oe = true;
  }
  if (d->ovnum) {
    if (cudaMalloc(&f->ovgid, sizeof(uint32_t) * d->ovnum) != cudaSuccess ||
        cudaMemcpy(f->ovgid, d->ovgid, sizeof(uint32_t) * d->ovnum, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("ovgid upload failed");
      return fail(GL_ERR_CUDA);
    }
  }
  if (d->inner_oids && d->ivnum) {
    f->h_inner_oids.assign(d->inner_oids, d->inner_oids + d->ivnum);
    // inner_oids is in lid order, whatever order the host assigned lids in (the reference's edge-file
    // loader numbers vertices by first appearance): oid -> lid then goes through a sorted side index
    const auto& io = f->h_inner_oids;
    if (std::adjacent_find(io.begin(), io.end(), std::greater_equal<int64_t>()) != io.end()) {
      f->h_oid_index.resize(d->ivnum);
      for (uint32_t l = 0; l < d->ivnum; ++l) f->h_oid_index[l] = {io[l], l};
      std::sort(f->h_oid_index.begin(), f->h_oid_index.end());
      auto dup = std::adjacent_find(f->h_oid_index.begin(), f->h_oid_index.end(),
                                    [](const std::pair<int64_t, uint32_t>& a, const std::pair<int64_t, uint32_t>& b) {
                                      return a.first == b.first;
                                    });
      if (dup != f->h_oid_index.end()) {
        set_error("inner oid %lld appears twice (lids %u and %u)", (long long) dup->first, dup->second,
                  (dup + 1)->second);
        return fail(GL_ERR_ARG);
      }
    }
    if (cudaMalloc(&f->inner_oids, sizeof(int64_t) * d->ivnum) != cudaSuccess ||
        cudaMemcpy(f->inner_oids, d->inner_oids, sizeof(int64_t) * d->ivnum, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("inner oid upload failed");
      return fail(GL_ERR_CUDA);
    }
  }
  st = finish_common(f);
  if (st != GL_OK) return fail(st);
  *out = f;
  return GL_OK;
}

int gl_frag_get_info(const gl_frag_t* f, gl_frag_info* o) {
  GL_ARG(f && o, "null argument");
  memset(o, 0, sizeof(*o));
  o->fid = f->fid;
  o->fnum = f->fnum;
  o->ivnum = f->ivnum;
  o->ovnum = f->ovnum;
  o->total_vnum = f->total_vnum;
  o->oe_num = f->oe.entries;
  o->ie_num = f->ie.entries;
  o->directed = f->directed;
  o->load_strategy = f->load_strategy;
  o->edata_bytes = f->edata_bytes;
  o->fid_offset = f->fid_offset;
  o->device_bytes = f->device_bytes;
  o->max_degree = f->max_degree;
  return GL_OK;
}

int gl_frag_view_get(const gl_frag_t* f, gl_frag_view* v) {
  GL_ARG(f && v, "null argument");
  // While the topology is offloaded (OffloadTopology, host_fragment.h:440-455) the view stays
  // usable for everything that is not adjacency: ids, gids of outer copies, ranges -- the
  // reference's lcc.h keeps calling DeviceObject() after it offloaded.  oe_col / oe_w are NULL.
  frag_fill_view(f, v);
  return GL_OK;
}

int gl_frag_copy_csr(const gl_frag_t* f, int which, uint64_t* rp, uint32_t* col,
                     void* w) {
  GL_ARG(f && which >= 0 && which <= 2, "bad argument");
  if (f->offloaded) {
    set_error("fragment topology is offloaded");
    return GL_ERR_STATE;
  }
  const DevCsr& c = which == 0 ? f->oe : (which == 1 ? f->ie : f->ovie);
  if (which == 2 && !c.rp) {
    if (rp) memset(rp, 0, sizeof(uint64_t) * ((size_t) f->ovnum + 1));
    return GL_OK;
  }
  if (rp) GL_CUDA(cudaMemcpy(rp, c.rp, sizeof(uint64_t) * (c.rows + 1), cudaMemcpyDeviceToHost));
  if (col && c.entries) GL_CUDA(cudaMemcpy(col, c.col, sizeof(uint32_t) * c.entries, cudaMemcpyDeviceToHost));
  if (w && c.w && c.entries) GL_CUDA(cudaMemcpy(w, c.w, (size_t) f->edata_bytes * c.entries, cudaMemcpyDeviceToHost));
  return GL_OK;
}

int gl_frag_copy_ovgid(const gl_frag_t* f, uint32_t* ovgid) {
  GL_ARG(f && (ovgid || !f->ovnum), "null argument");
  if (f->ovnum) GL_CUDA(cudaMemcpy(ovgid, f->ovgid, sizeof(uint32_t) * f->ovnum, cudaMemcpyDeviceToHost));
  return GL_OK;
}

int gl_frag_oid2lid(const gl_frag_t* f, int64_t oid, uint32_t* lid) {
  GL_ARG(f && lid, "null argument");
  if (!f->h_oid_index.empty()) {
    auto it = std::lower_bound(f->h_oid_index.begin(), f->h_oid_index.end(), std::make_pair(oid, 0u));
    if (it == f->h_oid_index.end() || it->first != oid) {
      set_error("oid %lld is not an inner vertex of fragment %u", (long long) oid, f->fid);
      return GL_ERR_ARG;
    }
    *lid = it->second;
    return GL_OK;
  }
  if (!f->h_inner_oids.empty()) {
    auto it = std::lower_bound(f->h_inner_oids.begin(), f->h_inner_oids.end(), oid);
    if (it == f->h_inner_oids.end() || *it != oid) {
      set_error("oid %lld is not an inner vertex of fragment %u", (long long) oid, f->fid);
      return GL_ERR_ARG;
    }
    *lid = (uint32_t) (it - f->h_inner_oids.begin());
    return GL_OK;
  }
  if (oid < f->oid_base || oid >= f->oid_base + (int64_t) f->ivnum) {
    set_error("oid %lld is not an inner vertex of fragment %u", (long long) oid, f->fid);
    return GL_ERR_ARG;
  }
  *lid = (uint32_t) (oid - f->oid_base);
  return GL_OK;
}

int gl_frag_max_degree_vertex(const gl_frag_t* f, uint32_t* lid, uint64_t* degree) {
  GL_ARG(f, "null argument");
  if (lid) *lid = f->max_degree_lid;
  if (degree) *degree = f->max_degree;
  return GL_OK;
}

// OffloadTopology / ReloadTopology (host_fragment.h:440-468): move the oe CSR
// to host memory and back (LCC frees the topology after building its DAG).
int gl_frag_offload(gl_frag_t* f) {
  GL_ARG(f, "null argument");
  if (f->offloaded) return GL_OK;
  f->sh_rp.resize(f->oe.rows + 1);
  f->sh_col.resize(f->oe.entries);
  GL_CUDA(cudaMemcpy(f->sh_rp.data(), f->oe.rp, sizeof(uint64_t) * (f->oe.rows + 1), cudaMemcpyDeviceToHost));
  if (f->oe.entries) GL_CUDA(cudaMemcpy(f->sh_col.data(), f->oe.col, sizeof(uint32_t) * f->oe.entries, cudaMemcpyDeviceToHost));
  if (f->oe.w) {
    f->sh_w.resize((size_t) f->edata_bytes * f->oe.entries);
    GL_CUDA(cudaMemcpy(f->sh_w.data(), f->oe.w, f->sh_w.size(), cudaMemcpyDeviceToHost));
  }
  cudaFree(f->oe.col);
  f->oe.col = nullptr;
  if (f->oe.w) cudaFree(f->oe.w);
  f->oe.w = nullptr;
  if (f->ie_alias_oe) f->ie = f->oe;
  f->offloaded = true;
  return GL_OK;
}

int gl_frag_reload(gl_frag_t* f) {
  GL_ARG(f, "null argument");
  if (!f->offloaded) return GL_OK;
  GL_CUDA(cudaMalloc(&f->oe.col, sizeof(uint32_t) * (f->oe.entries + 16)));
  if (f->oe.entries) GL_CUDA(cudaMemcpy(f->oe.col, f->sh_col.data(), sizeof(uint32_t) * f->oe.entries, cudaMemcpyHostToDevice));
  if (!f->sh_w.empty()) {
    GL_CUDA(cudaMalloc(&f->oe.w, f->sh_w.size() + 64));
    GL_CUDA(cudaMemcpy(f->oe.w, f->sh_w.data(), f->sh_w.size(), cudaMemcpyHostToDevice));
  }
  if (f->ie_alias_oe) f->ie = f->oe;
  f->sh_rp.clear();
  f->sh_col.clear();
  f->sh_w.clear();
  f->offloaded = false;
  return GL_OK;
}

void gl_frag_destroy(gl_frag_t* f) {
  if (!f) return;
  auto free_csr = [](DevCsr& c) {
    if (c.rp) cudaFree(c.rp);
    if (c.col) cudaFree(c.col);
    if (c.w) cudaFree(c.w);
    if (c.split) cudaFree(c.split);
    c = DevCsr();
  };
  if (!f->ie_alias_oe) free_csr(f->ie);
  free_csr(f->oe);
  free_csr(f->ovie);
  if (f->ovgid) cudaFree(f->ovgid);
  if (f->outer_range) cudaFree(f->outer_range);
  if (f->inner_oids) cudaFree(f->inner_oids);
  if (f->nonzero_deg) cudaFree(f->nonzero_deg);
  if (f->oe_tile_row) cudaFree(f->oe_tile_row);
  delete f;
}

}  // extern "C"
