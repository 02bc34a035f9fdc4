// primitives.cu — C-ABI engine primitives: fixed-function ForEachOutgoingEdge
// over a WorkSourceArray with the reference's load-balancing modes
// (grape/cuda/parallel/parallel_engine.h:987-1013, 1184-1394) and bitmap
// compaction (the ForEach+AppendWarp idiom, cuda/sssp/sssp.h:223-232).
#include <cub/cub.cuh>

#include "apps_common.cuh"

namespace gl {
namespace {

// Long-row cut of the cm / cmold queue scans: rows longer than this go to the hub phase (cta
// uses kHubDeg).  A row that long would serialise one CTA: measured 2x slower than the
// reference's cm.
constexpr uint32_t kHubDegCm = 8 * kHubDeg;

// Every op below may be handed a queue with repeated entries (see op_hub_overflow_inline).

struct OpLevel {
  static constexpr bool kHubOverflowInline = true;
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  uint32_t* level;
  uint32_t* out;
  uint32_t depth;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  GL_DEV void edge(uint32_t, Meta, uint32_t v, W, ScanAcc& acc) const {
    if (level[v] == kInfU32) {
      if (atomicCAS(level + v, kInfU32, depth) == kInfU32) {
        if (out) bit_set_atomic(out, v);
        acc.next_count++;
      }
    }
  }
};
struct OpMinU32 {
  static constexpr bool kHubOverflowInline = true;
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = true;
  uint32_t* state;
  uint32_t* out;
  int use_w;
  GL_DEV Meta assign(uint32_t u) const { return state[u]; }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W w, ScanAcc& acc) const {
    // saturating: an unreached source (kInfU32) never relaxes anything
    uint32_t nv = m;
    if (use_w) {
      nv = m + (uint32_t) w;
      if (nv < m) nv = kInfU32;
    }
    if (nv < atomicMin(state + v, nv)) {
      if (out) bit_set_atomic(out, v);
      acc.next_count++;
    }
  }
};
struct OpMinF32 {
  static constexpr bool kHubOverflowInline = true;
  using Meta = float;
  using W = float;
  static constexpr bool kWeighted = true;
  float* state;
  uint32_t* out;
  int use_w;
  GL_DEV Meta assign(uint32_t u) const { return state[u]; }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W w, ScanAcc& acc) const {
    float nv = use_w ? m + w : m;
    if (nv < atomic_min_f32_nonneg(state + v, nv)) {
      if (out) bit_set_atomic(out, v);
      acc.next_count++;
    }
  }
};
struct OpAddF64 {
  static constexpr bool kHubOverflowInline = true;
  using Meta = double;
  using W = float;
  static constexpr bool kWeighted = false;
  const double* src;
  double* dst;
  GL_DEV Meta assign(uint32_t u) const { return src[u]; }
  GL_DEV void edge(uint32_t, Meta m, uint32_t v, W, ScanAcc&) const {
    atomicAdd(dst + v, m);
  }
};
struct OpCount {
  static constexpr bool kHubOverflowInline = true;
  using Meta = uint32_t;
  using W = float;
  static constexpr bool kWeighted = false;
  unsigned long long* sink;
  GL_DEV Meta assign(uint32_t) const { return 0; }
  GL_DEV void edge(uint32_t, Meta, uint32_t v, W, ScanAcc& acc) const {
    acc.aux += (v == 0xFFFFFFFEu);  // keeps the column load alive
  }
};

struct PrimScratch {
  ScanCtrl* ctrl = nullptr;
  ScanCtrl* h_ctrl = nullptr;
  HubItem* hubs = nullptr;
  uint32_t hub_cap = 0;
  uint64_t* deg = nullptr;
  uint64_t* pfx = nullptr;
  uint32_t pfx_cap = 0;
  void* scan_tmp = nullptr;
  size_t scan_bytes = 0;
};
thread_local PrimScratch g_ps;

int ensure_scratch(const gl_frag* f, uint32_t n) {
  PrimScratch& ps = g_ps;
  if (!ps.ctrl) {
    GL_CUDA(cudaMalloc(&ps.ctrl, sizeof(ScanCtrl)));
    GL_CUDA(cudaMallocHost(&ps.h_ctrl, sizeof(ScanCtrl)));
  }
  uint64_t m = std::max<uint64_t>(f->oe.entries, 1);
  uint32_t need = (uint32_t) std::min<uint64_t>(m / kHubChunk + m / kHubDeg + 1024, 0x7FFFFFFFull);
  if (need > ps.hub_cap) {
    if (ps.hubs) cudaFree(ps.hubs);
    GL_CUDA(cudaMalloc(&ps.hubs, sizeof(HubItem) * (size_t) need));
    ps.hub_cap = need;
  }
  if (n + 1 > ps.pfx_cap) {
    if (ps.deg) cudaFree(ps.deg);
    if (ps.pfx) cudaFree(ps.pfx);
    if (ps.scan_tmp) cudaFree(ps.scan_tmp);
    GL_CUDA(cudaMalloc(&ps.deg, sizeof(uint64_t) * ((size_t) n + 1)));
    GL_CUDA(cudaMalloc(&ps.pfx, sizeof(uint64_t) * ((size_t) n + 1)));
    ps.scan_bytes = 0;
    GL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, ps.scan_bytes, ps.deg, ps.pfx, (int) (n + 1)));
    GL_CUDA(cudaMalloc(&ps.scan_tmp, ps.scan_bytes));
    ps.pfx_cap = n + 1;
  }
  return GL_OK;
}

template <class Op>
int scan_queue(const gl_frag* f, cudaStream_t s, const uint32_t* q, uint32_t n,
               const Op& op, int lb, uint64_t* scanned_host) {
  GL_TRY(ensure_scratch(f, n));
  PrimScratch& ps = g_ps;
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  EdgeRange er{f->oe.rp, f->oe.col, f->oe.w};
  GL_CUDA(cudaMemsetAsync(ps.ctrl, 0, sizeof(ScanCtrl), s));
  if (n) {
    switch (lb) {
      case GL_LB_NONE: {
        int g = std::min<int>(persistent_grid(k_queue_scan_none<Op>, di->sm_count), (int) ((n + kTB - 1) / kTB));
        GL_LAUNCH(k_queue_scan_none<Op>, g, kTB, s, ArraySrc{q}, n, er, op, ps.ctrl);
        break;
      }
      case GL_LB_WM: {
        int g = std::min<int>(persistent_grid(k_queue_scan_warp<Op>, di->sm_count), (int) ((n + kTB - 1) / kTB));
        GL_LAUNCH(k_queue_scan_warp<Op>, g, kTB, s, ArraySrc{q}, n, er, op, ps.ctrl);
        break;
      }
      case GL_LB_CM:
      case GL_LB_CMOLD:
      case GL_LB_CTA: {
        // CTA tiles; rows longer than hub_deg are cut into grid-wide kHubChunk-entry work items
        uint32_t hub_deg = lb == GL_LB_CTA ? kHubDeg : kHubDegCm;
        int g = std::min<int>(persistent_grid(k_queue_scan_cta<Op>, di->sm_count), (int) ((n + kTileV - 1) / kTileV));
        GL_LAUNCH(k_queue_scan_cta<Op>, g, kTB, s, ArraySrc{q}, n, er, op, ps.ctrl, ps.hubs, ps.hub_cap, hub_deg);
        int g2 = persistent_grid(k_hub_scan_tma<Op>, di->sm_count);
        GL_LAUNCH(k_hub_scan_tma<Op>, g2, kTB, s, er, op, ps.ctrl, ps.hubs, ps.hub_cap);
        break;
      }
      case GL_LB_STRICT: {
        GL_LAUNCH(k_queue_degrees<ArraySrc>, (n + 1 + 255) / 256, 256, s, ArraySrc{q}, n, f->oe.rp, ps.deg);
        GL_CUDA(cub::DeviceScan::ExclusiveSum(ps.scan_tmp, ps.scan_bytes, ps.deg, ps.pfx, (int) (n + 1), s));
        int g = persistent_grid(k_queue_scan_strict<Op>, di->sm_count);
        GL_LAUNCH(k_queue_scan_strict<Op>, g, kTB, s, ArraySrc{q}, n, ps.pfx, er, op, ps.ctrl);
        break;
      }
      default:
        set_error("unknown load-balancing mode %d", lb);
        return GL_ERR_ARG;
    }
  }
  if (scanned_host) {
    GL_CUDA(cudaMemcpyAsync(ps.h_ctrl, ps.ctrl, sizeof(ScanCtrl), cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    *scanned_host = ps.h_ctrl->scanned;
  }
  return GL_OK;
}

__global__ void k_compact(const uint32_t* bm, uint32_t nbits, uint32_t* q,
                          uint32_t* count) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t rounds = (nbits + stride - 1) / stride;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t r = 0; r < rounds; ++r, i += stride) {
    bool p = i < nbits && bit_test(bm, i);
    queue_append_warp(q, count, p, i);
  }
}

}  // namespace
}  // namespace gl

using namespace gl;

extern "C" {

int gl_edge_scan_queue(const gl_frag_t* f, void* stream, const uint32_t* queue,
                       uint32_t n, const gl_edge_op* op, int lb,
                       uint64_t* entries_scanned_host) {
  GL_ARG(f && op, "null argument");
  GL_ARG(n == 0 || queue, "null queue");
  if (f->offloaded) {
    set_error("fragment topology is offloaded");
    return GL_ERR_STATE;
  }
  if ((op->kind == GL_OP_MIN_RELAX_U32 || op->kind == GL_OP_MIN_RELAX_F32) && op->use_weight && f->oe.w &&
      f->edata_bytes != 4) {
    set_error("gl_edge_scan_queue: use_weight needs f32 edge data (this fragment has %d-byte edge data)",
              f->edata_bytes);
    return GL_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t) stream;
  switch (op->kind) {
    case GL_OP_BFS_LEVEL: {
      GL_ARG(op->state, "state required");
      OpLevel o{(uint32_t*) op->state, op->out_bitmap, op->depth};
      return scan_queue(f, s, queue, n, o, lb, entries_scanned_host);
    }
    case GL_OP_MIN_RELAX_U32: {
      GL_ARG(op->state, "state required");
      OpMinU32 o{(uint32_t*) op->state, op->out_bitmap, op->use_weight && f->oe.w != nullptr};
      return scan_queue(f, s, queue, n, o, lb, entries_scanned_host);
    }
    case GL_OP_MIN_RELAX_F32: {
      GL_ARG(op->state, "state required");
      OpMinF32 o{(float*) op->state, op->out_bitmap, op->use_weight && f->oe.w != nullptr};
      return scan_queue(f, s, queue, n, o, lb, entries_scanned_host);
    }
    case GL_OP_ADD_SCATTER_F64: {
      GL_ARG(op->state && op->state2, "state and state2 required");
      OpAddF64 o{(const double*) op->state, (double*) op->state2};
      return scan_queue(f, s, queue, n, o, lb, entries_scanned_host);
    }
    case GL_OP_COUNT: {
      OpCount o{nullptr};
      return scan_queue(f, s, queue, n, o, lb, entries_scanned_host);
    }
    default:
      set_error("unknown edge op %d", op->kind);
      return GL_ERR_ARG;
  }
}

int gl_compact_bitmap(void* stream, const uint32_t* bitmap, uint32_t n_bits,
                      uint32_t* queue_out, uint32_t* count_host) {
  GL_ARG(bitmap && queue_out && count_host, "null argument");
  cudaStream_t s = (cudaStream_t) stream;
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  DevBuf<uint32_t> d_count;
  GL_CUDA(d_count.alloc(1));
  GL_CUDA(cudaMemsetAsync(d_count, 0, 4, s));
  int g = std::max(1, std::min<int>(di->sm_count * 8, (int) ((n_bits + kTB - 1) / kTB)));
  k_compact<<<g, kTB, 0, s>>>(bitmap, n_bits, queue_out, d_count);
  GL_COUNT_LAUNCH();
  cudaError_t e = cudaMemcpyAsync(count_host, d_count, 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    set_error("gl_compact_bitmap: %s", cudaGetErrorString(e));
    return GL_ERR_CUDA;
  }
  return GL_OK;
}

}  // extern "C"

// ---- Face-2 containers (Queue / VertexArray) and PrepareToRunApp -------------------------------
struct gl_queue {
  uint32_t* data = nullptr;
  uint32_t* count = nullptr;
  uint32_t capacity = 0;
};

extern "C" {

int gl_queue_create(gl_queue_t** out, uint32_t capacity) {
  GL_ARG(out, "null argument");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_queue* q = new gl_queue;
  q->capacity = capacity;
  if (cudaMalloc(&q->data, sizeof(uint32_t) * std::max<uint32_t>(capacity, 1)) != cudaSuccess ||
      cudaMalloc(&q->count, sizeof(uint32_t)) != cudaSuccess || cudaMemset(q->count, 0, 4) != cudaSuccess) {
    gl_queue_destroy(q);
    set_error("gl_queue_create: device allocation failed");
    return GL_ERR_NOMEM;
  }
  *out = q;
  return GL_OK;
}
int gl_queue_clear(gl_queue_t* q, void* stream) {
  GL_ARG(q, "null argument");
  GL_CUDA(cudaMemsetAsync(q->count, 0, 4, (cudaStream_t) stream));
  return GL_OK;
}
int gl_queue_size(gl_queue_t* q, void* stream, uint32_t* size_host) {
  GL_ARG(q && size_host, "null argument");
  GL_CUDA(cudaMemcpyAsync(size_host, q->count, 4, cudaMemcpyDeviceToHost, (cudaStream_t) stream));
  GL_CUDA(cudaStreamSynchronize((cudaStream_t) stream));
  if (*size_host > q->capacity) *size_host = q->capacity;
  return GL_OK;
}
int gl_queue_data(gl_queue_t* q, uint32_t** data_dev, uint32_t** count_dev) {
  GL_ARG(q, "null argument");
  if (data_dev) *data_dev = q->data;
  if (count_dev) *count_dev = q->count;
  return GL_OK;
}
int gl_queue_fill_from_bitmap(gl_queue_t* q, void* stream, const uint32_t* bitmap, uint32_t n_bits) {
  GL_ARG(q && bitmap, "null argument");
  GL_ARG(n_bits <= q->capacity, "gl_queue_fill_from_bitmap: the queue is smaller than the bitmap");
  cudaStream_t s = (cudaStream_t) stream;
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  GL_CUDA(cudaMemsetAsync(q->count, 0, 4, s));
  if (n_bits) {
    int g = std::max(1, std::min<int>(di->sm_count * 8, (int) ((n_bits + kTB - 1) / kTB)));
    k_compact<<<g, kTB, 0, s>>>(bitmap, n_bits, q->data, q->count);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  return GL_OK;
}
void gl_queue_destroy(gl_queue_t* q) {
  if (!q) return;
  cudaFree(q->data);
  cudaFree(q->count);
  delete q;
}

int gl_varray_create(void** out, uint64_t count, int elem_bytes, int fill_byte) {
  GL_ARG(out && elem_bytes > 0, "bad argument");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  const size_t bytes = std::max<size_t>((size_t) count * (size_t) elem_bytes, 16);
  GL_CUDA(cudaMalloc(out, bytes));
  GL_CUDA(cudaMemset(*out, fill_byte, bytes));
  return GL_OK;
}
int gl_varray_h2d(void* v, const void* host, uint64_t count, int elem_bytes) {
  GL_ARG(v && host, "null argument");
  GL_CUDA(cudaMemcpy(v, host, (size_t) count * (size_t) elem_bytes, cudaMemcpyHostToDevice));
  return GL_OK;
}
int gl_varray_d2h(const void* v, void* host, uint64_t count, int elem_bytes) {
  GL_ARG(v && host, "null argument");
  GL_CUDA(cudaMemcpy(host, v, (size_t) count * (size_t) elem_bytes, cudaMemcpyDeviceToHost));
  return GL_OK;
}
int gl_varray_destroy(void* v) {
  if (v) GL_CUDA(cudaFree(v));
  return GL_OK;
}

int gl_frag_prepare(gl_frag_t* f, int message_strategy, int need_split_edges, int need_mirror_info) {
  GL_ARG(f, "null argument");
  GL_ARG(message_strategy >= 0 && message_strategy <= 3, "gl_frag_prepare: unknown message strategy");
  if (f->offloaded) {
    set_error("fragment topology is offloaded");
    return GL_ERR_STATE;
  }
  if (need_split_edges && (!f->oe.split || (f->directed && !f->ie_alias_oe && !f->ie.split))) {
    set_error("gl_frag_prepare: split positions are missing");
    return GL_ERR_STATE;
  }
  (void) need_mirror_info;   // mirror lists are exchanged by gl_mm_mirror_plan (needs the communicator)
  return GL_OK;
}

}  // extern "C"
