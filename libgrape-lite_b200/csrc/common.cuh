// common.cuh — shared host/device helpers of the PIE engine.
// sm_90a only (no multi-arch dispatch).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/grape_b200.h"

namespace gl {

// ---------------------------------------------------------------- errors ---
void set_error(const char* fmt, ...);
const char* last_error();

#define GL_CUDA(expr)                                                      \
  do {                                                                     \
    cudaError_t _e = (expr);                                               \
    if (_e != cudaSuccess) {                                               \
      ::gl::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,        \
                      cudaGetErrorString(_e));                             \
      return GL_ERR_CUDA;                                                  \
    }                                                                      \
  } while (0)

#define GL_TRY(expr)               \
  do {                             \
    int _s = (expr);               \
    if (_s != GL_OK) return _s;    \
  } while (0)

#define GL_ARG(cond, msg)                                      \
  do {                                                         \
    if (!(cond)) {                                             \
      ::gl::set_error("%s:%d: %s", __FILE__, __LINE__, msg);   \
      return GL_ERR_ARG;                                       \
    }                                                          \
  } while (0)

// Owning buffer of T: device memory (cudaMalloc), or pinned host memory
// (cudaMallocHost) when kPinned.  Move-only; freed on destruction, so a buffer
// is released on every return path.  alloc(n) takes exactly n * sizeof(T)
// bytes: pads stay with the caller, and the memory is plain cudaMalloc memory
// (CUDA IPC handles, free-memory accounting).  Converts to T* so that launches
// and copies take it like the raw pointer.
template <typename T, bool kPinned = false>
class Buf {
 public:
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept : p_(o.release()) {}
  Buf& operator=(Buf&& o) noexcept {
    reset(o.release());
    return *this;
  }
  ~Buf() { reset(); }

  cudaError_t alloc(size_t n) {
    reset();
    void* q = nullptr;
    cudaError_t e = kPinned ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
    p_ = (T*) q;
    return e;
  }
  T* get() const { return p_; }
  operator T*() const { return p_; }
  T* operator->() const { return p_; }
  T* release() {
    T* q = p_;
    p_ = nullptr;
    return q;
  }
  void reset(T* q = nullptr) {
    if (p_) {
      if (kPinned) cudaFreeHost(p_);
      else cudaFree(p_);
    }
    p_ = q;
  }

 private:
  T* p_ = nullptr;
};
template <typename T>
using DevBuf = Buf<T, false>;
template <typename T>
using PinnedBuf = Buf<T, true>;

// device properties (cached per process; one device per process/thread)
struct DeviceInfo {
  int device = -1;
  int sm_count = 0;
  int cc = 0;
  size_t l2_bytes = 0;
  size_t hbm_bytes = 0;
};
int device_info(DeviceInfo** out);
// SM count of the current device: grid size unit of the grid-stride helper kernels
int num_sms();

// L2 residency control (50 MB L2 on H100).  The randomly accessed per-vertex
// state of a sweep (PageRank contributions, SSSP distances, WCC labels: 64-128 MB
// at 2^24 vertices) competes with the streamed CSR (2-4 GB per sweep) for the L2;
// an access-policy window marks the state as PERSISTING and everything else the
// stream's kernels touch as STREAMING.  GL_L2_PERSIST=0 disables it (A/B).
int l2_persist_window(cudaStream_t s, const void* ptr, size_t bytes);
int l2_persist_clear(cudaStream_t s);

// Kernel launch counter (gpu_launches claim in bench.py)
extern thread_local uint64_t g_kernel_launches;
#define GL_COUNT_LAUNCH() (++::gl::g_kernel_launches)

constexpr uint32_t kInfU32 = 0xFFFFFFFFu;

// ------------------------------------------------------------- device ------
#ifdef __CUDACC__

#define GL_DEV __device__ __forceinline__

GL_DEV uint32_t lane_id() { return threadIdx.x & 31; }

// streaming 128-bit load that does not allocate in L1 (edge streams are read
// once; keep L1 for the frontier bitmap / per-vertex state)
GL_DEV uint4 ld_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
GL_DEV uint32_t ld_stream_u32(const uint32_t* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
GL_DEV float ld_stream_f32(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// Bitmap (replaces grape::cuda::dev::Bitset, grape/cuda/utils/bitset.h:32-103)
GL_DEV bool bit_test(const uint32_t* bm, uint32_t i) {
  return (bm[i >> 5] >> (i & 31)) & 1u;
}
// returns true when this call flipped the bit 0 -> 1
GL_DEV bool bit_set_atomic(uint32_t* bm, uint32_t i) {
  uint32_t m = 1u << (i & 31);
  uint32_t old = atomicOr(bm + (i >> 5), m);
  return !(old & m);
}

// float atomic min for non-negative values via integer ordering
// (replaces dev::atomicMinFloat, grape/cuda/utils/dev_utils.h:51-64).
GL_DEV float atomic_min_f32_nonneg(float* addr, float v) {
  return __uint_as_float(atomicMin((unsigned int*) addr, __float_as_uint(v)));
}
GL_DEV double atomic_min_f64_nonneg(double* addr, double v) {
  return __longlong_as_double((long long) atomicMin(
      (unsigned long long*) addr, (unsigned long long) __double_as_longlong(v)));
}

// warp-aggregated append (replaces dev::Queue::AppendWarp, queue.h:61-71)
GL_DEV void queue_append_warp(uint32_t* q, uint32_t* count, bool pred,
                              uint32_t value) {
  uint32_t mask = __ballot_sync(0xffffffffu, pred);
  if (mask == 0) return;
  uint32_t leader = __ffs(mask) - 1;
  uint32_t base = 0;
  if (lane_id() == leader) base = atomicAdd(count, __popc(mask));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (pred) q[base + __popc(mask & ((1u << lane_id()) - 1))] = value;
}

// ---- mbarrier + 1-D bulk async copy (TMA engine, SASS UBLKCP) -------------
GL_DEV uint32_t smem_u32(const void* p) {
  return (uint32_t) __cvta_generic_to_shared(p);
}
GL_DEV void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(count));
}
GL_DEV void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
GL_DEV void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
                   smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
GL_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
GL_DEV bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
GL_DEV void mbar_wait_parity(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned
GL_DEV void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes,
                        uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

#endif  // __CUDACC__

}  // namespace gl
