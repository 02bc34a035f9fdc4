// hub_order.cu — degree-ordered ("hub-first") relabelling helpers.
//
// H100's L2 (50 MB) cannot hold the per-vertex state of a scale-24 graph next
// to the 2 GB edge stream, and an SM can only keep a bounded number of random
// sector misses in flight.  Ordering vertices by descending degree makes the
// state of the few thousand hubs — the target of most of the 5e8 random
// accesses of a sweep — contiguous, so those accesses hit L1/L2.  The apps
// use the order internally and translate at their result boundary; the
// fragment's public layout (lid = ascending oid) is unchanged.
#include <cub/cub.cuh>

#include "apps_common.cuh"

namespace gl {
namespace {
__global__ void k_degkey(const uint64_t* rp, uint32_t n, uint32_t* key, uint32_t* val) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint64_t dg = rp[i + 1] - rp[i];
    if (dg > 0xFFFFFFFFull) dg = 0xFFFFFFFFull;
    key[i] = 0xFFFFFFFFu - (uint32_t) dg;   // ascending key = descending degree (stable: ties by lid)
    val[i] = i;
  }
}
__global__ void k_invert(const uint32_t* order, uint32_t n, uint32_t* perm) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) perm[order[i]] = i;
}
__global__ void k_perm_deg(const uint64_t* rp, const uint32_t* order, uint32_t n, uint64_t* deg) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) deg[i] = rp[order[i] + 1] - rp[order[i]];
  if (i == n) deg[i] = 0;
}
// one warp per new row: copy the row of order[i], relabelling the neighbours
__global__ void __launch_bounds__(256)
k_perm_rows(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
            const uint32_t* __restrict__ order, const uint32_t* __restrict__ perm,
            uint32_t n, const uint64_t* __restrict__ rp_p, uint32_t* col_p,
            const uint32_t* __restrict__ w, uint32_t* w_p) {
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const uint32_t u = order[i];
    const uint64_t b = rp[u], e = rp[u + 1], o = rp_p[i];
    for (uint64_t p = b + lane_id(); p < e; p += 32) {
      const uint32_t c = col[p];
      col_p[o + (p - b)] = c < n ? perm[c] : c;
      if (w) w_p[o + (p - b)] = w[p];   // 4-byte edge data moves with its edge
    }
  }
}
}  // namespace

int build_hub_order(cudaStream_t s, const uint64_t* rp, uint32_t n, DevBuf<uint32_t>* perm_out, DevBuf<uint32_t>* order_out) {
  DevBuf<uint32_t> key, key2, val, val2, perm;
  DevBuf<char> tmp;
  GL_CUDA(key.alloc(std::max<uint32_t>(n, 1)));
  GL_CUDA(key2.alloc(std::max<uint32_t>(n, 1)));
  GL_CUDA(val.alloc(std::max<uint32_t>(n, 1)));
  GL_CUDA(val2.alloc(std::max<uint32_t>(n, 1)));
  if (n) GL_LAUNCH(k_degkey, (n + 255) / 256, 256, s, rp, n, key, val);
  size_t tb = 0;
  cub::DoubleBuffer<uint32_t> kb(key, key2), vb(val, val2);
  GL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, (int) n, 0, 32, s));
  GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
  if (n) GL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, kb, vb, (int) n, 0, 32, s));
  GL_CUDA(perm.alloc(std::max<uint32_t>(n, 1)));
  if (n) GL_LAUNCH(k_invert, (n + 255) / 256, 256, s, vb.Current(), n, perm);
  GL_CUDA(cudaStreamSynchronize(s));
  DevBuf<uint32_t>& order = vb.Current() == val.get() ? val : val2;
  // the temporaries are freed in allocation order
  key.reset();
  key2.reset();
  (&order == &val ? val2 : val).reset();
  tmp.reset();
  *perm_out = std::move(perm);
  if (order_out) *order_out = std::move(order);
  return GL_OK;
}

// rows reordered by `order`, neighbours relabelled by `perm`
int build_permuted_csr(cudaStream_t s, const uint64_t* rp, const uint32_t* col, uint64_t m, uint32_t n,
                       const uint32_t* order, const uint32_t* perm, DevBuf<uint64_t>* rp_out, DevBuf<uint32_t>* col_out,
                       const void* w4, DevBuf<uint32_t>* w4_out, bool sort_rows) {
  DevBuf<uint64_t> deg, rp_p;
  GL_CUDA(deg.alloc((size_t) n + 1));
  GL_CUDA(rp_p.alloc((size_t) n + 1));
  GL_LAUNCH(k_perm_deg, (n + 1 + 255) / 256, 256, s, rp, order, n, deg);
  size_t tb = 0;
  GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, deg.get(), rp_p.get(), (int) (n + 1), s));
  DevBuf<char> tmp;
  GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
  GL_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, deg.get(), rp_p.get(), (int) (n + 1), s));
  DevBuf<uint32_t> col_p, w_p;
  GL_CUDA(col_p.alloc(m + 16));
  if (w4) GL_CUDA(w_p.alloc(m + 16));
  if (n) GL_LAUNCH(k_perm_rows, num_sms() * 8, 256, s, rp, col, order, perm, n, rp_p, col_p, (const uint32_t*) w4, w_p);
  // rows sorted by the new ids = by descending degree of the neighbour: the
  // most promising parents come first in a pull scan, and the entries of a
  // row that fall into the same bitmap word are adjacent
  if (sort_rows) GL_TRY(sort_csr_rows(s, rp_p, n, m, &col_p, w4 ? &w_p : nullptr));
  GL_CUDA(cudaStreamSynchronize(s));
  deg.reset();
  tmp.reset();
  *rp_out = std::move(rp_p);
  *col_out = std::move(col_p);
  if (w4_out) *w4_out = std::move(w_p);
  return GL_OK;
}

template <typename V>
int sort_csr_rows(cudaStream_t s, const uint64_t* rp, uint32_t n, uint64_t m, DevBuf<uint32_t>* col, DevBuf<V>* val) {
  if (!n || !m) return GL_OK;
  DevBuf<uint32_t> sorted;
  DevBuf<V> val_sorted;
  GL_CUDA(sorted.alloc(m + 16));
  if (val) GL_CUDA(val_sorted.alloc(m + 16));
  size_t sb = 0;
  DevBuf<char> st;
  if (val) {
    GL_CUDA(cub::DeviceSegmentedSort::SortPairs(nullptr, sb, col->get(), sorted.get(), val->get(), val_sorted.get(),
                                                (int64_t) m, (int64_t) n, rp, rp + 1, s));
    GL_CUDA(st.alloc(std::max<size_t>(sb, 16)));
    GL_CUDA(cub::DeviceSegmentedSort::SortPairs(st, sb, col->get(), sorted.get(), val->get(), val_sorted.get(),
                                                (int64_t) m, (int64_t) n, rp, rp + 1, s));
  } else {
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, sb, col->get(), sorted.get(), (int64_t) m, (int64_t) n, rp, rp + 1, s));
    GL_CUDA(st.alloc(std::max<size_t>(sb, 16)));
    GL_CUDA(cub::DeviceSegmentedSort::SortKeys(st, sb, col->get(), sorted.get(), (int64_t) m, (int64_t) n, rp, rp + 1, s));
  }
  GL_CUDA(cudaStreamSynchronize(s));
  st.reset();
  *col = std::move(sorted);
  if (val) *val = std::move(val_sorted);
  return GL_OK;
}
template int sort_csr_rows(cudaStream_t, const uint64_t*, uint32_t, uint64_t, DevBuf<uint32_t>*, DevBuf<uint32_t>*);
template int sort_csr_rows(cudaStream_t, const uint64_t*, uint32_t, uint64_t, DevBuf<uint32_t>*, DevBuf<uint64_t>*);

}  // namespace gl
