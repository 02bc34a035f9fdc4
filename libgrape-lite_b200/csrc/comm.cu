// comm.cu — landing-area allocation / CUDA-IPC mapping and the round protocol.
#include <cstring>
#include "comm.h"
#include "fragment.h"
#include "engine.cuh"
#include "apps_common.cuh"

#include <algorithm>
#include <cstdlib>

namespace gl {

namespace {
__global__ void k_publish_counts(uint32_t fnum, uint32_t fid,
                                 uint32_t* const* peer_count,
                                 uint32_t* send_count, uint32_t* h_out) {
  // one thread per destination: store my item count into the owner's header
  uint32_t d = threadIdx.x;
  uint32_t total = 0;
  if (d < fnum) {
    uint32_t c = send_count[d];
    if (d != fid) {
      *peer_count[d] = c;  // NVLink peer store
      total = c;
    }
    h_out[d] = c;
    send_count[d] = 0;  // ready for the next round
  }
  __threadfence_system();
}
// One block, one thread per peer: publish my contribution to every peer, wait
// for every peer's contribution of the same sequence number, reduce.
// With peer_count != nullptr it first publishes this round's item counts
// (FinishARound) and adds their total to i1, so that a round closes with ONE
// kernel and ONE stream synchronisation.
__global__ void k_peer_allreduce(uint32_t fnum, uint32_t fid, PeerSlot* const* my_slot_at_peer,
                                 const PeerSlot* local_slots, unsigned long long tag,
                                 long long i0, long long i1, double d0, int op,
                                 uint32_t* const* peer_count, uint32_t* send_count,
                                 uint32_t* h_counts, PeerSlot* h_out, long long i2 = 0,
                                 long long i3 = 0, const ScanCtrl* ctrl = nullptr,
                                 ScanCtrl* h_ctrl = nullptr) {
  __shared__ long long s_i0[GL_MAX_FNUM], s_i1[GL_MAX_FNUM], s_i2[GL_MAX_FNUM], s_i3[GL_MAX_FNUM];
  __shared__ double s_d0[GL_MAX_FNUM];
  __shared__ unsigned int s_total;
  const uint32_t p = threadIdx.x;
  if (p == 0) s_total = 0;
  __syncthreads();
  if (peer_count && p < fnum) {
    uint32_t c = send_count[p];
    if (p != fid) {
      *peer_count[p] = c;  // NVLink peer store
      atomicAdd(&s_total, c);
    }
    h_counts[p] = c;
    send_count[p] = 0;
  }
  __syncthreads();
  i1 += (long long) s_total;
  if (ctrl) {
    // vote taken from the engine's device counters
    const unsigned long long nc = ctrl->next_count, rc = ctrl->remote_count, ne = ctrl->next_edges;
    if (nc > 0) i0 = 1;
    i2 = (long long) (nc + rc);
    i3 = (long long) ne;
    if (p == 0 && h_ctrl) *h_ctrl = *ctrl;
  }
  if (p < fnum) {
    PeerSlot* dst = my_slot_at_peer[p];        // peer p's header, slot [me] (p == me: local)
    dst->i0 = i0;
    dst->i1 = i1;
    dst->i2 = i2;
    dst->i3 = i3;
    dst->d0 = d0;
    __threadfence_system();
    *(volatile unsigned long long*) &dst->tag = tag;
    // wait for peer p's contribution in MY header, slot [p]
    const volatile PeerSlot* src = local_slots + p;
    // bounded wait: a peer that failed on the host never arrives; report it
    // instead of spinning forever inside a kernel (GL_ERR_COMM on the host)
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    bool late = false;
    while (src->tag != tag) {
      __nanosleep(64);
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > 20000000000ull) {   // 20 s
        late = true;
        break;
      }
    }
    if (late) atomicExch(&s_total, 0xFFFFFFFFu);
    __threadfence_system();
    s_i0[p] = src->i0;
    s_i1[p] = src->i1;
    s_i2[p] = src->i2;
    s_i3[p] = src->i3;
    s_d0[p] = src->d0;
  }
  __syncthreads();
  if (p == 0) {
    long long a = s_i0[0], b = s_i1[0], e2 = s_i2[0], e3 = s_i3[0];
    double c = s_d0[0];
    for (uint32_t q = 1; q < fnum; ++q) {
      e2 += s_i2[q];
      e3 += s_i3[q];
      if (op == 0) { a += s_i0[q]; b += s_i1[q]; c += s_d0[q]; }
      else if (op == 1) { a = a < s_i0[q] ? a : s_i0[q]; b = b < s_i1[q] ? b : s_i1[q]; c = c < s_d0[q] ? c : s_d0[q]; }
      else { a = a > s_i0[q] ? a : s_i0[q]; b = b > s_i1[q] ? b : s_i1[q]; c = c > s_d0[q] ? c : s_d0[q]; }
    }
    h_out->i0 = a;
    h_out->i1 = b;
    h_out->i2 = e2;
    h_out->i3 = e3;
    h_out->d0 = c;
    h_out->tag = (s_total == 0xFFFFFFFFu) ? ~0ull : tag;   // ~0: a peer timed out
  }
  (void) fid;
}

// ---- dense mirror sync ------------------------------------------------------
// holder side of the plan: tell every owner which of its inner lids I hold
__global__ void k_mirror_request(const uint32_t* __restrict__ ovgid, uint32_t ivnum, uint32_t ovnum,
                                 const uint32_t* __restrict__ ghost_range, uint32_t fnum,
                                 uint32_t id_mask, char* const* msend) {
  for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < ovnum; o += gridDim.x * blockDim.x) {
    const uint32_t lid = ivnum + o;
    uint32_t f = 0;
    while (f + 1 < fnum && lid >= ghost_range[f + 1]) ++f;
    ((uint32_t*) msend[f])[lid - ghost_range[f]] = ovgid[o] & id_mask;
  }
}
__global__ void k_mirror_counts(const uint32_t* __restrict__ ghost_range, uint32_t fnum, uint32_t fid,
                                uint32_t* const* peer_count) {
  uint32_t f = threadIdx.x;
  if (f < fnum && f != fid) *peer_count[f] = ghost_range[f + 1] - ghost_range[f];
  __threadfence_system();
}
// owner side: pack the bits of my mirrored vertices, 32 per word, per holder
__global__ void k_mirror_pack_bits(const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ lids,
                                   const uint64_t* __restrict__ off, char* const* msend) {
  const uint32_t g = blockIdx.y;
  const uint64_t b = off[g], n = off[g + 1] - b;
  uint32_t* out = (uint32_t*) msend[g];
  const uint64_t npad = (n + 31) & ~31ull;
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < npad; k += (uint64_t) gridDim.x * blockDim.x) {
    bool bit = false;
    if (k < n) bit = bit_test(bitmap, lids[b + k]);
    uint32_t w = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) out[k >> 5] = w;
  }
}

// ---- word-parallel bit plan (MirrorBitsPlan) ---------------------------------
__global__ void k_mirror_check_sorted(const uint32_t* __restrict__ lids, const uint64_t* __restrict__ off,
                                      uint32_t fnum, uint32_t* bad) {
  const uint32_t g = blockIdx.y;
  const uint64_t b = off[g], n = off[g + 1] - b;
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k + 1 < n; k += (uint64_t) gridDim.x * blockDim.x)
    if (lids[b + k] >= lids[b + k + 1]) *bad = 1;
  (void) fnum;
}
__global__ void k_mirror_mask(const uint32_t* __restrict__ lids, const uint64_t* __restrict__ off,
                              uint32_t iv_words, uint32_t* mask) {
  const uint32_t g = blockIdx.y;
  const uint64_t b = off[g], n = off[g + 1] - b;
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x * blockDim.x) {
    const uint32_t l = lids[b + k];
    atomicOr(mask + (size_t) g * iv_words + (l >> 5), 1u << (l & 31));
  }
}
// one CTA per holder: pref[w] = mirrored vertices before word w
__global__ void __launch_bounds__(kTB) k_mirror_pref(const uint32_t* __restrict__ mask, uint32_t iv_words, uint32_t* pref) {
  __shared__ uint32_t s_warp[kTB / 32 + 1];
  const uint32_t g = blockIdx.x;
  uint32_t run = 0;
  for (uint32_t base = 0; base < iv_words; base += kTB) {
    const uint32_t w = base + threadIdx.x;
    const uint32_t c = w < iv_words ? __popc(mask[(size_t) g * iv_words + w]) : 0;
    uint32_t total;
    const uint32_t ex = block_excl_scan(c, s_warp, &total);
    if (w < iv_words) pref[(size_t) g * iv_words + w] = run + ex;
    run += total;
  }
}
// startw[woff[g] + j] = input word holding output bit 32 j of holder g
__global__ void k_mirror_startw(const uint32_t* __restrict__ mask, const uint32_t* __restrict__ pref,
                                uint32_t iv_words, const uint64_t* __restrict__ woff, uint32_t* startw) {
  const uint32_t g = blockIdx.y;
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < iv_words; w += gridDim.x * blockDim.x) {
    const uint32_t c = __popc(mask[(size_t) g * iv_words + w]);
    if (!c) continue;
    const uint32_t p0 = pref[(size_t) g * iv_words + w];
    // output bits [p0, p0 + c) live in this word; those that are multiples of 32 start an output word
    for (uint32_t j = (p0 + 31) >> 5; (j << 5) < p0 + c; ++j) startw[woff[g] + j] = w;
  }
}
__global__ void __launch_bounds__(256) k_mirror_pack_bits2(MirrorBitsPlan P, const uint32_t* __restrict__ bitmap,
                                                          char* const* msend) {
  mirror_pack_bits_phase(P, bitmap, msend, (uint64_t) blockIdx.x * blockDim.x + threadIdx.x,
                         (uint64_t) gridDim.x * blockDim.x);
}

// holder side: OR the received words into the ghost positions of my bitmap
// (one thread per 32 outer copies; the ghost range of an owner is contiguous
// but not word aligned, hence the two-part shifted OR)
__global__ void k_mirror_unpack_bits(uint32_t* bitmap, const uint32_t* __restrict__ ghost_range,
                                     const char* const* mrecv) {
  const uint32_t f = blockIdx.y;
  const uint32_t base = ghost_range[f], n = ghost_range[f + 1] - base;
  const uint32_t nw = (n + 31) >> 5;
  const uint32_t* in = (const uint32_t*) mrecv[f];
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nw; j += gridDim.x * blockDim.x) {
    const uint32_t w = __ldcg(in + j);   // written by the peer: bypass L1
    if (!w) continue;
    const uint32_t pos = base + (j << 5), sh = pos & 31;
    atomicOr(bitmap + (pos >> 5), w << sh);
    if (sh) atomicOr(bitmap + (pos >> 5) + 1, w >> (32 - sh));
  }
}
template <typename T>
__global__ void k_mirror_pack_vals(const T* __restrict__ values, const uint32_t* __restrict__ lids,
                                   const uint64_t* __restrict__ off, char* const* msend) {
  const uint32_t g = blockIdx.y;
  const uint64_t b = off[g], n = off[g + 1] - b;
  T* out = (T*) msend[g];
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x * blockDim.x)
    out[k] = values[lids[b + k]];
}
template <typename T>
__global__ void k_mirror_unpack_vals(T* values, const uint32_t* __restrict__ ghost_range,
                                     const char* const* mrecv) {
  const uint32_t f = blockIdx.y;
  const uint32_t base = ghost_range[f], n = ghost_range[f + 1] - base;
  const T* in = (const T*) mrecv[f];
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    values[base + k] = in[k];
}
// rows of w 8-byte words: one thread per word
__global__ void k_mirror_pack_rows(const uint64_t* __restrict__ values, uint32_t w, const uint32_t* __restrict__ lids,
                                   const uint64_t* __restrict__ off, char* const* msend) {
  const uint32_t g = blockIdx.y;
  const uint64_t b = off[g], n = (off[g + 1] - b) * w;
  uint64_t* out = (uint64_t*) msend[g];
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x * blockDim.x)
    out[k] = values[(uint64_t) lids[b + k / w] * w + k % w];
}
__global__ void k_mirror_unpack_rows(uint64_t* values, uint32_t w, const uint32_t* __restrict__ ghost_range,
                                     const char* const* mrecv) {
  const uint32_t f = blockIdx.y;
  const uint64_t base = (uint64_t) ghost_range[f] * w, n = (uint64_t) (ghost_range[f + 1] - ghost_range[f]) * w;
  const uint64_t* in = (const uint64_t*) mrecv[f];
  for (uint64_t k = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x * blockDim.x)
    values[base + k] = in[k];
}
}  // namespace

int MessageManager::PeerBarrier(cudaStream_t s) {
  long long a = 0, b = 0;
  double c = 0;
  return PeerAllReduce(s, &a, &b, &c, 0);
}

int MessageManager::PeerBarrierAsync(cudaStream_t s) {
  const unsigned long long tag = ++comm->seq_base;
  const int par = (int) (tag & 1);
  const PeerSlot* local = (const PeerSlot*) (comm->local_base + GL_COMM_SLOT_OFF) + (size_t) par * GL_MAX_FNUM;
  if (!d_scratch_result) GL_CUDA(d_scratch_result.alloc(1));
  GL_LAUNCH(k_peer_allreduce, 1, GL_MAX_FNUM, s, fnum, fid, d_peer_slot[par], local, tag, 0ll, 0ll, 0.0, 0,
            nullptr, nullptr, nullptr, d_scratch_result, 0ll, 0ll, nullptr, nullptr);
  return GL_OK;
}

int MessageManager::ExchangeBlobs(cudaStream_t s, const void* mine, size_t bytes, std::vector<char>* all) {
  all->assign(bytes * fnum, 0);
  if (fnum == 1) {
    memcpy(all->data(), mine, bytes);
    return GL_OK;
  }
  if (bytes > comm->landing_bytes) {
    set_error("ExchangeBlobs: %zu bytes exceed the landing slot", bytes);
    return GL_ERR_COMM;
  }
  GL_TRY(PeerBarrier(s));   // nobody still reads parity-0 slots of an earlier exchange
  for (uint32_t p = 0; p < fnum; ++p) {
    if (p == fid) continue;
    char* dst = comm->peer_base[p] + GL_COMM_HEADER + (size_t) fid * comm->landing_bytes;   // (parity 0, src = me)
    GL_CUDA(cudaMemcpyAsync(dst, mine, bytes, cudaMemcpyHostToDevice, s));
  }
  GL_CUDA(cudaStreamSynchronize(s));
  GL_TRY(PeerBarrier(s));
  for (uint32_t p = 0; p < fnum; ++p) {
    if (p == fid) {
      memcpy(all->data() + (size_t) p * bytes, mine, bytes);
      continue;
    }
    GL_CUDA(cudaMemcpyAsync(all->data() + (size_t) p * bytes,
                            comm->local_base + GL_COMM_HEADER + (size_t) p * comm->landing_bytes, bytes,
                            cudaMemcpyDeviceToHost, s));
  }
  GL_CUDA(cudaStreamSynchronize(s));
  GL_TRY(PeerBarrier(s));
  return GL_OK;
}

int MessageManager::BuildMirrorPlan(cudaStream_t s, const gl_frag_view& fv) {
  plan_built = true;
  plan_ivnum = fv.ivnum;
  if (fnum == 1) return GL_OK;
  comm->mirror_dirty = true;
  if (comm->mirror_bytes == 0) {
    set_error("communicator was created without a mirror-sync area (mirror_bytes = 0)");
    return GL_ERR_COMM;
  }
  // tables of mirror slots
  for (int par = 0; par < 2; ++par) {
    std::vector<char*> snd(fnum);
    std::vector<const char*> rcv(fnum);
    for (uint32_t p = 0; p < fnum; ++p) {
      snd[p] = comm->peer_base[p] + comm->mirror_off(par, fid);
      rcv[p] = comm->local_base + comm->mirror_off(par, p);
    }
    GL_CUDA(d_msend[par].alloc(fnum));
    GL_CUDA(d_mrecv[par].alloc(fnum));
    GL_CUDA(cudaMemcpy(d_msend[par], snd.data(), sizeof(char*) * fnum, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(d_mrecv[par], rcv.data(), sizeof(char*) * fnum, cudaMemcpyHostToDevice));
  }
  ghost_range.resize(fnum + 1);
  GL_CUDA(cudaMemcpy(ghost_range.data(), fv.outer_range, sizeof(uint32_t) * (fnum + 1), cudaMemcpyDeviceToHost));
  d_ghost_range = const_cast<uint32_t*>(fv.outer_range);
  for (uint32_t f = 0; f < fnum; ++f) {
    if ((size_t) (ghost_range[f + 1] - ghost_range[f]) * 8 > comm->mirror_bytes) {
      set_error("mirror-sync area too small: %u outer copies of fragment %u", ghost_range[f + 1] - ghost_range[f], f);
      return GL_ERR_COMM;
    }
  }
  GL_TRY(PeerBarrier(s));  // every rank's area is mapped and idle
  // 1. requests: my ghosts' owner-lids, in ghost order, into the owner's slot (parity 0)
  if (fv.ovnum) {
    k_mirror_request<<<num_sms() * 4, 256, 0, s>>>(fv.ovgid, fv.ivnum, fv.ovnum, d_ghost_range, fnum, id_mask, d_msend[0]);
    GL_COUNT_LAUNCH();
  }
  k_mirror_counts<<<1, GL_MAX_FNUM, 0, s>>>(d_ghost_range, fnum, fid, d_peer_count[0]);
  GL_COUNT_LAUNCH();
  GL_CUDA(cudaGetLastError());
  GL_TRY(PeerBarrier(s));
  // 2. owner: read how many lids every holder sent, copy the lists out
  std::vector<uint32_t> cnt(GL_MAX_FNUM);
  GL_CUDA(cudaMemcpy(cnt.data(), comm->local_base, sizeof(uint32_t) * GL_MAX_FNUM, cudaMemcpyDeviceToHost));
  mirror_off.assign(fnum + 1, 0);
  for (uint32_t g = 0; g < fnum; ++g) mirror_off[g + 1] = mirror_off[g] + (g == fid ? 0 : cnt[g]);
  mirror_total = mirror_off[fnum];
  GL_CUDA(d_mirror_lids.alloc(std::max<uint64_t>(mirror_total, 1)));
  GL_CUDA(d_mirror_off.alloc(fnum + 1));
  GL_CUDA(cudaMemcpy(d_mirror_off, mirror_off.data(), sizeof(uint64_t) * (fnum + 1), cudaMemcpyHostToDevice));
  for (uint32_t g = 0; g < fnum; ++g) {
    if (g == fid || cnt[g] == 0) continue;
    GL_CUDA(cudaMemcpyAsync(d_mirror_lids + mirror_off[g], comm->local_base + comm->mirror_off(0, g),
                            sizeof(uint32_t) * cnt[g], cudaMemcpyDeviceToDevice, s));
  }
  // the message-count cells were borrowed: clear them for the first round
  GL_CUDA(cudaMemsetAsync(comm->local_base, 0, sizeof(uint32_t) * 2 * GL_MAX_FNUM, s));
  GL_TRY(PeerBarrier(s));
  mirror_seq = 0;
  // word-parallel form for bit syncs (needs ascending lids per holder)
  mirror_sorted = false;
  if (mirror_total && fv.ivnum) {
    dim3 grid(num_sms() * 4, fnum);
    uint32_t bad = 1;
    {
      DevBuf<uint32_t> d_bad;
      GL_CUDA(d_bad.alloc(1));
      GL_CUDA(cudaMemsetAsync(d_bad, 0, 4, s));
      k_mirror_check_sorted<<<grid, 256, 0, s>>>(d_mirror_lids, d_mirror_off, fnum, d_bad);
      GL_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, s));
      GL_CUDA(cudaStreamSynchronize(s));
    }
    if (!bad) {
      iv_words = (uint32_t) ((fv.ivnum + 31) / 32);
      std::vector<uint64_t> woff(fnum + 1, 0);
      for (uint32_t g = 0; g < fnum; ++g) woff[g + 1] = woff[g] + (mirror_off[g + 1] - mirror_off[g] + 31) / 32;
      mirror_out_words = woff[fnum];
      GL_CUDA(d_mirror_mask.alloc((size_t) fnum * iv_words));
      GL_CUDA(d_mirror_pref.alloc((size_t) fnum * iv_words));
      GL_CUDA(d_mirror_startw.alloc(std::max<uint64_t>(mirror_out_words, 1)));
      GL_CUDA(d_mirror_woff.alloc(fnum + 1));
      GL_CUDA(cudaMemcpyAsync(d_mirror_woff, woff.data(), sizeof(uint64_t) * (fnum + 1), cudaMemcpyHostToDevice, s));
      GL_CUDA(cudaMemsetAsync(d_mirror_mask, 0, sizeof(uint32_t) * (size_t) fnum * iv_words, s));
      k_mirror_mask<<<grid, 256, 0, s>>>(d_mirror_lids, d_mirror_off, iv_words, d_mirror_mask);
      k_mirror_pref<<<fnum, kTB, 0, s>>>(d_mirror_mask, iv_words, d_mirror_pref);
      k_mirror_startw<<<grid, 256, 0, s>>>(d_mirror_mask, d_mirror_pref, iv_words, d_mirror_woff, d_mirror_startw);
      GL_CUDA(cudaGetLastError());
      GL_CUDA(cudaStreamSynchronize(s));
      mirror_sorted = true;
    }
  }
  return GL_OK;
}

MirrorBitsPlan MessageManager::bits_plan() const {
  MirrorBitsPlan P;
  P.fnum = fnum;
  P.iv_words = iv_words;
  P.mask = d_mirror_mask;
  P.pref = d_mirror_pref;
  P.startw = d_mirror_startw;
  P.woff = d_mirror_woff;
  P.off = d_mirror_off;
  return P;
}

int MessageManager::SyncBitsToGhosts(cudaStream_t s, uint32_t* bitmap) {
  if (fnum == 1) return GL_OK;
  comm->mirror_dirty = true;
  const int par = (int) (++mirror_seq & 1);
  if (mirror_total && mirror_sorted) {
    GL_LAUNCH(k_mirror_pack_bits2, num_sms() * 8, 256, s, bits_plan(), bitmap, d_msend[par]);
  } else if (mirror_total) {
    dim3 grid(num_sms() * 8, fnum);
    GL_LAUNCH(k_mirror_pack_bits, grid, 256, s, bitmap, d_mirror_lids, d_mirror_off, d_msend[par]);
  }
  GL_TRY(PeerBarrierAsync(s));
  if (ghost_range[fnum] > ghost_range[0]) {
    dim3 grid(num_sms() * 2, fnum);
    GL_LAUNCH(k_mirror_unpack_bits, grid, 256, s, bitmap, d_ghost_range, d_mrecv[par]);
  }
  return GL_OK;
}

int MessageManager::SyncValuesToGhosts(cudaStream_t s, void* values, int elem_bytes) {
  if (fnum == 1) return GL_OK;
  comm->mirror_dirty = true;
  const int par = (int) (++mirror_seq & 1);
  dim3 grid(num_sms() * 8, fnum);
  if (mirror_total) {
    if (elem_bytes == 4) k_mirror_pack_vals<uint32_t><<<grid, 256, 0, s>>>((const uint32_t*) values, d_mirror_lids, d_mirror_off, d_msend[par]);
    else k_mirror_pack_vals<uint64_t><<<grid, 256, 0, s>>>((const uint64_t*) values, d_mirror_lids, d_mirror_off, d_msend[par]);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  GL_TRY(PeerBarrierAsync(s));
  if (ghost_range[fnum] > ghost_range[0]) {
    if (elem_bytes == 4) k_mirror_unpack_vals<uint32_t><<<grid, 256, 0, s>>>((uint32_t*) values, d_ghost_range, d_mrecv[par]);
    else k_mirror_unpack_vals<uint64_t><<<grid, 256, 0, s>>>((uint64_t*) values, d_ghost_range, d_mrecv[par]);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  return GL_OK;
}

size_t MessageManager::MaxRowBytes() const {
  if (fnum == 1) return SIZE_MAX;
  uint32_t most = 0;
  for (uint32_t f = 0; f < fnum; ++f) most = std::max(most, ghost_range[f + 1] - ghost_range[f]);
  return most ? comm->mirror_bytes / most : SIZE_MAX;
}

int MessageManager::SyncRowsToGhosts(cudaStream_t s, void* values, int row_bytes) {
  if (fnum == 1) return GL_OK;
  if (row_bytes <= 0 || row_bytes % 8 || row_bytes > 256 || (size_t) row_bytes > MaxRowBytes()) {
    set_error("SyncRowsToGhosts: %d-byte rows do not fit the mirror-sync area (%zu bytes per peer)", row_bytes,
              comm->mirror_bytes);
    return GL_ERR_ARG;
  }
  const uint32_t w = (uint32_t) row_bytes / 8;
  comm->mirror_dirty = true;
  const int par = (int) (++mirror_seq & 1);
  dim3 grid(num_sms() * 8, fnum);
  if (mirror_total) {
    k_mirror_pack_rows<<<grid, 256, 0, s>>>((const uint64_t*) values, w, d_mirror_lids, d_mirror_off, d_msend[par]);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  GL_TRY(PeerBarrierAsync(s));
  if (ghost_range[fnum] > ghost_range[0]) {
    k_mirror_unpack_rows<<<grid, 256, 0, s>>>((uint64_t*) values, w, d_ghost_range, d_mrecv[par]);
    GL_COUNT_LAUNCH();
    GL_CUDA(cudaGetLastError());
  }
  return GL_OK;
}

int MessageManager::PeerAllReduce(cudaStream_t s, long long* i0, long long* i1, double* d0, int op) {
  const unsigned long long tag = ++comm->seq_base;
  const int par = (int) (tag & 1);
  const PeerSlot* local = (const PeerSlot*) (comm->local_base + GL_COMM_SLOT_OFF) + (size_t) par * GL_MAX_FNUM;
  k_peer_allreduce<<<1, GL_MAX_FNUM, 0, s>>>(fnum, fid, d_peer_slot[par], local, tag, *i0, *i1, *d0, op,
                                             nullptr, nullptr, nullptr, h_result);
  GL_COUNT_LAUNCH();
  GL_CUDA(cudaGetLastError());
  GL_CUDA(cudaStreamSynchronize(s));
  if (h_result->tag == ~0ull) {
    set_error("peer collective timed out (a fragment of the group did not arrive)");
    return GL_ERR_COMM;
  }
  *i0 = h_result->i0;
  *i1 = h_result->i1;
  *d0 = h_result->d0;
  return GL_OK;
}

int MessageManager::Init(gl_comm* c, const gl_frag_view& fv, uint32_t item_bytes_) {
  comm = c;
  fid = fv.fid;
  fnum = fv.fnum;
  fid_offset = fv.fid_offset;
  id_mask = fv.id_mask;
  item_bytes = item_bytes_;
  if (fnum == 1) return GL_OK;
  if (!c || !c->opened || c->fnum != fnum || c->fid != fid) {
    set_error("fragment has fnum=%u but no opened communicator was supplied", fnum);
    return GL_ERR_COMM;
  }
  GL_CUDA(d_send_count.alloc(fnum));
  GL_CUDA(cudaMemset(d_send_count, 0, sizeof(uint32_t) * fnum));
  GL_CUDA(d_zero_count.alloc(fnum));
  GL_CUDA(cudaMemset(d_zero_count, 0, sizeof(uint32_t) * fnum));
  GL_CUDA(h_send_count.alloc(fnum + 1));
  GL_CUDA(h_result.alloc(1));
  for (int par = 0; par < 2; ++par) {
    std::vector<char*> send(fnum);
    std::vector<const char*> recv(fnum);
    std::vector<uint32_t*> pc(fnum);
    for (uint32_t p = 0; p < fnum; ++p) {
      // my slot at peer p: (parity, src = me)
      send[p] = c->peer_base[p] + GL_COMM_HEADER +
                ((size_t) par * fnum + fid) * c->landing_bytes;
      pc[p] = (uint32_t*) (c->peer_base[p]) + (size_t) par * GL_MAX_FNUM + fid;
      // peer p's slot in my area
      recv[p] = c->local_base + GL_COMM_HEADER +
                ((size_t) par * fnum + p) * c->landing_bytes;
    }
    std::vector<PeerSlot*> ps(fnum);
    for (uint32_t p = 0; p < fnum; ++p)
      ps[p] = (PeerSlot*) (c->peer_base[p] + GL_COMM_SLOT_OFF) + (size_t) par * GL_MAX_FNUM + fid;
    GL_CUDA(d_peer_slot[par].alloc(fnum));
    GL_CUDA(cudaMemcpy(d_peer_slot[par], ps.data(), sizeof(PeerSlot*) * fnum, cudaMemcpyHostToDevice));
    GL_CUDA(d_send_slot[par].alloc(fnum));
    GL_CUDA(d_recv_slot[par].alloc(fnum));
    GL_CUDA(d_peer_count[par].alloc(fnum));
    GL_CUDA(cudaMemcpy(d_send_slot[par], send.data(), sizeof(char*) * fnum, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(d_recv_slot[par], recv.data(), sizeof(char*) * fnum, cudaMemcpyHostToDevice));
    GL_CUDA(cudaMemcpy(d_peer_count[par], pc.data(), sizeof(uint32_t*) * fnum, cudaMemcpyHostToDevice));
  }
  return GL_OK;
}

MsgView MessageManager::view() const {
  MsgView v;
  memset(&v, 0, sizeof(v));
  v.fid = fid;
  v.fnum = fnum;
  v.fid_offset = fid_offset;
  v.id_mask = id_mask;
  v.item_bytes = item_bytes;
  if (fnum > 1) {
    int par = round & 1, prev = (round + 1) & 1;
    v.capacity = (uint32_t) std::min<size_t>(comm->landing_bytes / item_bytes, 0xFFFFFFFFu);
    v.send_slot = d_send_slot[par];
    v.send_count = d_send_count;
    v.recv_slot = d_recv_slot[prev];
    // round 0 of a query receives nothing: the parity-1 count cells still hold a round of the
    // previous query on this manager
    v.recv_count = round == 0 ? d_zero_count.get()
                              : (const uint32_t*) comm->local_base + (size_t) prev * GL_MAX_FNUM;
  }
  return v;
}

int MessageManager::StartARound(cudaStream_t s) {
  stream_for_collectives = s;
  force_continue = false;
  return GL_OK;
}

// publish counts -> sync -> all-reduce (barrier + termination vote)
int MessageManager::FinishARound(cudaStream_t s) {
  if (decided_terminate) {
    decided_terminate = false;
    terminate = true;
    return GL_OK;
  }
  int64_t vote[2] = {force_continue ? 1 : 0, 0};
  if (fnum > 1) {
    int par = round & 1;
    if (use_peer_barrier) {
      // publish counts + barrier + termination vote: one kernel, one sync
      const unsigned long long tag = ++comm->seq_base;
      const int bp = (int) (tag & 1);
      const PeerSlot* local = (const PeerSlot*) (comm->local_base + GL_COMM_SLOT_OFF) + (size_t) bp * GL_MAX_FNUM;
      k_peer_allreduce<<<1, GL_MAX_FNUM, 0, s>>>(fnum, fid, d_peer_slot[bp], local, tag, (long long) vote[0], 0ll,
                                                 0.0, 0, d_peer_count[par], d_send_count, h_send_count, h_result,
                                                 stat_in[0], stat_in[1], vote_ctrl, vote_h_ctrl);
      vote_ctrl = nullptr;
      vote_h_ctrl = nullptr;
      GL_COUNT_LAUNCH();
      GL_CUDA(cudaGetLastError());
      GL_CUDA(cudaStreamSynchronize(s));
      if (h_result->tag == ~0ull) {
        set_error("round barrier timed out (a fragment of the group did not arrive)");
        return GL_ERR_COMM;
      }
      vote[0] = h_result->i0;
      vote[1] = h_result->i1;
      stat_out[0] = h_result->i2;
      stat_out[1] = h_result->i3;
      stat_in[0] = stat_in[1] = 0;
    } else {
      k_publish_counts<<<1, GL_MAX_FNUM, 0, s>>>(fnum, fid, d_peer_count[par], d_send_count, h_send_count);
      GL_COUNT_LAUNCH();
      GL_CUDA(cudaGetLastError());
      GL_CUDA(cudaStreamSynchronize(s));
    }
    uint64_t sent = 0;
    for (uint32_t p = 0; p < fnum; ++p)
      if (p != fid) {
        if (h_send_count[p] > comm->landing_bytes / item_bytes) {
          set_error("landing slot overflow: %u items to fragment %u", h_send_count[p], p);
          return GL_ERR_COMM;
        }
        sent += h_send_count[p];
      }
    bytes_sent += sent * item_bytes;
    if (!use_peer_barrier) {
      vote[1] = (int64_t) sent;
      GL_TRY(AllReduceI64(vote, 2, 0));
    }
  } else {
    GL_CUDA(cudaStreamSynchronize(s));
  }
  terminate = (vote[0] == 0 && vote[1] == 0);
  ++round;
  return GL_OK;
}

int MessageManager::AllReduceI64(int64_t* v, int n, int op) {
  if (fnum == 1) return GL_OK;
  if (!comm || !comm->allreduce) {
    set_error("communicator has no allreduce callback");
    return GL_ERR_COMM;
  }
  int st = comm->allreduce(comm->user, v, n, 0, op);
  if (st != 0) {
    set_error("allreduce callback failed (%d)", st);
    return GL_ERR_COMM;
  }
  return GL_OK;
}
int MessageManager::AllReduceF64(double* v, int n, int op) {
  if (fnum == 1) return GL_OK;
  if (use_peer_barrier && n == 1 && comm && comm->opened) {
    long long a = 0, b = 0;
    cudaStream_t s0 = stream_for_collectives;
    return PeerAllReduce(s0, &a, &b, v, op);
  }
  if (!comm || !comm->allreduce) {
    set_error("communicator has no allreduce callback");
    return GL_ERR_COMM;
  }
  int st = comm->allreduce(comm->user, v, n, 1, op);
  if (st != 0) {
    set_error("allreduce callback failed (%d)", st);
    return GL_ERR_COMM;
  }
  return GL_OK;
}

namespace {
// what a fragment tells its peers about its CSR part
struct PeerCsrExport {
  cudaIpcMemHandle_t h_rp, h_col, h_w;
  uint64_t rows, m;
};
}  // namespace

int PeerCsr::replicate(MessageManager& mm, cudaStream_t s, const gl_frag_view& fv, const uint64_t* rp,
                       const uint32_t* col, uint64_t m, const uint32_t* w) {
  if (!d_rp) {
    GL_CUDA(d_rp.alloc(fv.fnum));
    GL_CUDA(d_col.alloc(fv.fnum));
  }
  if (w && !d_w) GL_CUDA(d_w.alloc(fv.fnum));
  rep_rp.clear();
  rep_col.clear();
  rep_w.clear();
  rep_rp.resize(fv.fnum);
  rep_col.resize(fv.fnum);
  rep_w.resize(fv.fnum);
  std::vector<const uint64_t*> r_rp(fv.fnum);
  std::vector<const uint32_t*> r_col(fv.fnum), r_w(fv.fnum);
  r_rp[fv.fid] = rp;
  r_col[fv.fid] = col;
  r_w[fv.fid] = w;
  if (fv.fnum > 1) {
    PeerCsrExport mine;
    memset(&mine, 0, sizeof(mine));
    GL_CUDA(cudaIpcGetMemHandle(&mine.h_rp, (void*) rp));
    GL_CUDA(cudaIpcGetMemHandle(&mine.h_col, (void*) col));
    if (w) GL_CUDA(cudaIpcGetMemHandle(&mine.h_w, (void*) w));
    mine.rows = fv.ivnum;
    mine.m = m;
    std::vector<char> all;
    GL_TRY(mm.ExchangeBlobs(s, &mine, sizeof(mine), &all));
    for (uint32_t g = 0; g < fv.fnum; ++g) {
      if (g == fv.fid) continue;
      const PeerCsrExport& ex = *(const PeerCsrExport*) (all.data() + (size_t) g * sizeof(PeerCsrExport));
      GL_CUDA(rep_rp[g].alloc(ex.rows + 1));
      GL_CUDA(rep_col[g].alloc(std::max<uint64_t>(ex.m, 4)));
      r_rp[g] = rep_rp[g];
      r_col[g] = rep_col[g];
      void *p_rp = nullptr, *p_col = nullptr, *p_w = nullptr;
      GL_CUDA(cudaIpcOpenMemHandle(&p_rp, ex.h_rp, cudaIpcMemLazyEnablePeerAccess));
      GL_CUDA(cudaIpcOpenMemHandle(&p_col, ex.h_col, cudaIpcMemLazyEnablePeerAccess));
      GL_CUDA(cudaMemcpyAsync(rep_rp[g], p_rp, sizeof(uint64_t) * (ex.rows + 1), cudaMemcpyDeviceToDevice, s));
      if (ex.m) GL_CUDA(cudaMemcpyAsync(rep_col[g], p_col, sizeof(uint32_t) * ex.m, cudaMemcpyDeviceToDevice, s));
      if (w) {
        GL_CUDA(rep_w[g].alloc(std::max<uint64_t>(ex.m, 4)));
        r_w[g] = rep_w[g];
        GL_CUDA(cudaIpcOpenMemHandle(&p_w, ex.h_w, cudaIpcMemLazyEnablePeerAccess));
        if (ex.m) GL_CUDA(cudaMemcpyAsync(rep_w[g], p_w, sizeof(uint32_t) * ex.m, cudaMemcpyDeviceToDevice, s));
      }
      GL_CUDA(cudaStreamSynchronize(s));
      GL_CUDA(cudaIpcCloseMemHandle(p_rp));
      GL_CUDA(cudaIpcCloseMemHandle(p_col));
      if (p_w) GL_CUDA(cudaIpcCloseMemHandle(p_w));
    }
  }
  GL_CUDA(cudaMemcpyAsync(d_rp, r_rp.data(), sizeof(void*) * fv.fnum, cudaMemcpyHostToDevice, s));
  GL_CUDA(cudaMemcpyAsync(d_col, r_col.data(), sizeof(void*) * fv.fnum, cudaMemcpyHostToDevice, s));
  if (w) GL_CUDA(cudaMemcpyAsync(d_w, r_w.data(), sizeof(void*) * fv.fnum, cudaMemcpyHostToDevice, s));
  GL_CUDA(cudaStreamSynchronize(s));
  if (fv.fnum > 1) GL_TRY(mm.PeerBarrier(s));   // every peer has finished reading my arrays
  return GL_OK;
}

}  // namespace gl

using namespace gl;

extern "C" {

int gl_comm_create(gl_comm_t** out, const gl_comm_desc* d) {
  GL_ARG(out && d, "null argument");
  GL_ARG(d->fnum >= 1 && d->fnum <= GL_MAX_FNUM && d->fid < d->fnum, "bad fid/fnum");
  GL_ARG(d->fnum == 1 || d->allreduce, "allreduce callback required when fnum > 1");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  gl_comm* c = new gl_comm;
  c->fid = d->fid;
  c->fnum = d->fnum;
  c->allreduce = d->allreduce;
  c->user = d->user;
  c->landing_bytes = (d->landing_bytes + 255) & ~(size_t) 255;
  c->mirror_bytes = (d->mirror_bytes + 255) & ~(size_t) 255;
  cudaError_t e = cudaMalloc(&c->local_base, c->total_bytes());
  if (e != cudaSuccess) {
    set_error("landing area (%zu bytes): %s", c->total_bytes(), cudaGetErrorString(e));
    delete c;
    return GL_ERR_NOMEM;
  }
  cudaMemset(c->local_base, 0, GL_COMM_HEADER);
  c->peer_base.assign(c->fnum, nullptr);
  c->peer_base[c->fid] = c->local_base;
  if (c->fnum == 1) c->opened = true;
  *out = c;
  return GL_OK;
}

int gl_comm_export(gl_comm_t* c, void* handles_out, size_t bytes) {
  GL_ARG(c && handles_out && bytes >= GL_IPC_HANDLE_BYTES, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) <= GL_IPC_HANDLE_BYTES, "handle size");
  cudaIpcMemHandle_t h;
  GL_CUDA(cudaIpcGetMemHandle(&h, c->local_base));
  memset(handles_out, 0, GL_IPC_HANDLE_BYTES);
  memcpy(handles_out, &h, sizeof(h));
  return GL_OK;
}

int gl_comm_open(gl_comm_t* c, const void* all, size_t bytes) {
  GL_ARG(c && all && bytes >= (size_t) c->fnum * GL_IPC_HANDLE_BYTES, "bad argument");
  for (uint32_t p = 0; p < c->fnum; ++p) {
    if (p == c->fid) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*) all + (size_t) p * GL_IPC_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      set_error("cudaIpcOpenMemHandle(peer %u): %s", p, cudaGetErrorString(e));
      return GL_ERR_COMM;
    }
    c->peer_base[p] = (char*) ptr;
  }
  c->opened = true;
  return GL_OK;
}

int gl_comm_close_peers(gl_comm_t* c) {
  GL_ARG(c, "null argument");
  for (uint32_t p = 0; p < c->fnum; ++p)
    if (p != c->fid && c->peer_base[p]) {
      cudaIpcCloseMemHandle(c->peer_base[p]);
      c->peer_base[p] = nullptr;
    }
  c->opened = c->fnum == 1;
  return GL_OK;
}

void gl_comm_destroy(gl_comm_t* c) {
  if (!c) return;
  for (uint32_t p = 0; p < c->fnum; ++p)
    if (p != c->fid && c->peer_base[p]) cudaIpcCloseMemHandle(c->peer_base[p]);
  if (c->local_base) cudaFree(c->local_base);
  delete c;
}

}  // extern "C"

// ---- diagnostic: kernel-driven NVLink peer-store bandwidth --------------------
namespace gl {
namespace {
template <typename V>
__global__ void __launch_bounds__(256) k_peer_write(const V* __restrict__ src, V* const* dsts, uint32_t ndst, size_t n) {
  const size_t stride = (size_t) gridDim.x * blockDim.x;
  for (uint32_t d = 0; d < ndst; ++d) {
    V* dst = dsts[d];
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) __threadfence_system();
}
}  // namespace
}  // namespace gl

extern "C" int gl_comm_peer_write_us(gl_comm_t* c, size_t bytes, int vec16, int all_peers, int reps, double* us_out) {
  using namespace gl;
  GL_ARG(c && us_out && reps > 0, "gl_comm_peer_write_us: null argument");
  if (!c->opened || c->fnum < 2) {
    set_error("gl_comm_peer_write_us needs an opened communicator with fnum >= 2");
    return GL_ERR_STATE;
  }
  c->mirror_dirty = true;
  bytes &= ~(size_t) 15;
  if (bytes == 0 || bytes > c->mirror_bytes) {
    set_error("gl_comm_peer_write_us: bytes must be in (0, mirror_bytes]");
    return GL_ERR_ARG;
  }
  DevBuf<char> src;
  GL_CUDA(src.alloc(bytes));
  GL_CUDA(cudaMemset(src, 1, bytes));
  std::vector<char*> dsts;
  for (uint32_t k = 1; k < c->fnum; ++k) {
    const uint32_t p = (c->fid + k) % c->fnum;
    dsts.push_back(c->peer_base[p] + c->mirror_off(1, c->fid));   // my parity-1 mirror slot at peer p
    if (!all_peers) break;
  }
  DevBuf<char*> d_dsts;
  GL_CUDA(d_dsts.alloc(dsts.size()));
  GL_CUDA(cudaMemcpy(d_dsts, dsts.data(), sizeof(char*) * dsts.size(), cudaMemcpyHostToDevice));
  cudaEvent_t e0, e1;
  GL_CUDA(cudaEventCreate(&e0));
  GL_CUDA(cudaEventCreate(&e1));
  for (int r = -2; r < reps; ++r) {
    if (r == 0) GL_CUDA(cudaEventRecord(e0, 0));
    if (vec16) k_peer_write<uint4><<<num_sms() * 4, 256>>>((const uint4*) src.get(), (uint4* const*) d_dsts.get(), (uint32_t) dsts.size(), bytes / 16);
    else k_peer_write<uint32_t><<<num_sms() * 4, 256>>>((const uint32_t*) src.get(), (uint32_t* const*) d_dsts.get(), (uint32_t) dsts.size(), bytes / 4);
  }
  GL_CUDA(cudaEventRecord(e1, 0));
  GL_CUDA(cudaEventSynchronize(e1));
  float ms = 0;
  GL_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *us_out = (double) ms * 1e3 / reps;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return GL_OK;
}

// ---------------------------------------------------------------------------
// Face 2 of the boundary: gl_mm_* / gl_allreduce (include/grape_b200.h).
// A gl_mm is the library's MessageManager with byte-granular slots
// (item_bytes = 1): the shimmed grape::cuda::GPUMessageManager of
// compat/grape/cuda/b200_compat.h runs the reference's unchanged apps on it.
// ---------------------------------------------------------------------------
struct gl_mm {
  gl::MessageManager mm;
  gl_comm* comm = nullptr;
  bool owns_single = false;   // fnum == 1 and no communicator was given
  gl::DevBuf<gl::ScanCtrl> d_ctrl;
};

namespace gl {
namespace {
template <typename V>
struct GidVal {
  uint32_t gid;
  V val;
};
template <>
struct GidVal<double> {
  uint32_t gid, pad;
  double val;
};
// one launch over all sources; items are thrust::pair<vid_t, V>-shaped
template <typename V, int KIND>
__global__ void __launch_bounds__(256) k_mm_process(gl_mm_view mv, V* state, uint32_t* out_bitmap,
                                                     unsigned long long* n_items) {
  unsigned long long mine = 0;
  for (uint32_t src = 0; src < mv.fnum; ++src) {
    if (src == mv.fid) continue;
    uint32_t bytes = mv.recv_bytes[src];
    if (bytes > mv.capacity_bytes) bytes = mv.capacity_bytes;
    if (KIND == GL_MSG_SET_BIT) {
      const uint32_t n = bytes / 4;
      const uint32_t* g = (const uint32_t*) mv.recv_slot[src];
      for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t lid = __ldcg(g + i) & mv.id_mask;
        if (out_bitmap) atomicOr(out_bitmap + (lid >> 5), 1u << (lid & 31));
        ++mine;
      }
    } else {
      using It = GidVal<V>;
      const uint32_t n = bytes / (uint32_t) sizeof(It);
      const It* items = (const It*) mv.recv_slot[src];
      for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t lid = __ldcg(&items[i].gid) & mv.id_mask;
        const V v = __ldcg(&items[i].val);
        bool improved = false;
        if (KIND == GL_MSG_MIN_U32) improved = v < atomicMin((unsigned int*) (state + lid), (unsigned int) v);
        else if (KIND == GL_MSG_MIN_F32) improved = v < atomic_min_f32_nonneg((float*) (state + lid), (float) v);
        else if (KIND == GL_MSG_MIN_F64) improved = v < atomic_min_f64_nonneg((double*) (state + lid), (double) v);
        else atomicAdd(state + lid, v);
        if (improved && out_bitmap) atomicOr(out_bitmap + (lid >> 5), 1u << (lid & 31));
        ++mine;
      }
    }
  }
  mine = warp_sum(mine);
  if (lane_id() == 0 && mine && n_items) atomicAdd(n_items, mine);
}
}  // namespace
}  // namespace gl

namespace gl {
namespace {
template <int VB>
struct OuterItem;
template <>
struct OuterItem<0> { uint32_t gid; };
template <>
struct OuterItem<4> { uint32_t gid; uint32_t val; };
template <>
struct OuterItem<8> { uint32_t gid, pad; unsigned long long val; };

// one thread per outer copy; lanes of a warp bound for the same owner share a
// single byte reservation in that owner's landing slot
template <int VB>
__global__ void __launch_bounds__(256) k_mm_send_outer(gl_mm_view mv, uint32_t* remote, uint32_t ivnum, uint32_t ovnum,
                                                        const uint32_t* __restrict__ ovgid, const void* state,
                                                        int clear_bits) {
  using It = OuterItem<VB>;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t rounds = (ovnum + stride - 1) / stride;
  uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t r = 0; r < rounds; ++r, o += stride) {
    bool pred = false;
    uint32_t dst = 0;
    It it;
    memset(&it, 0, sizeof(it));
    if (o < ovnum) {
      const uint32_t v = ivnum + o;
      if (bit_test(remote, v)) {
        pred = true;
        it.gid = ovgid[o];
        dst = it.gid >> mv.fid_offset;
        if constexpr (VB == 4) it.val = ((const uint32_t*) state)[v];
        if constexpr (VB == 8) it.val = ((const unsigned long long*) state)[v];
      }
    }
    const uint32_t active = __ballot_sync(0xffffffffu, pred);
    if (pred) {
      const uint32_t peers = __match_any_sync(active, dst);
      const uint32_t leader = __ffs(peers) - 1;
      uint32_t base = 0;
      if (lane_id() == leader) base = atomicAdd(mv.send_bytes + dst, (uint32_t) (__popc(peers) * sizeof(It)));
      base = __shfl_sync(peers, base, leader);
      const uint32_t off = base + __popc(peers & ((1u << lane_id()) - 1)) * (uint32_t) sizeof(It);
      if (off + sizeof(It) <= mv.capacity_bytes) *(It*) (mv.send_slot[dst] + off) = it;
    }
  }
  (void) clear_bits;
}
__global__ void k_clear_bit_range(uint32_t* bm, uint32_t lo, uint32_t hi) {
  const uint32_t w_lo = lo >> 5, w_hi = (hi + 31) >> 5;
  for (uint32_t w = w_lo + blockIdx.x * blockDim.x + threadIdx.x; w < w_hi; w += gridDim.x * blockDim.x) {
    uint32_t keep = 0;
    const uint32_t b0 = w << 5;
    if (b0 < lo) keep |= (1u << (lo - b0)) - 1u;
    if (b0 + 32 > hi) keep |= hi > b0 ? ~((1u << (hi - b0)) - 1u) : 0xFFFFFFFFu;
    bm[w] &= keep;
  }
}
__global__ void k_bitmap_count(const uint32_t* bm, uint64_t nbits, unsigned long long* out) {
  const uint64_t words = (nbits + 31) / 32;
  unsigned long long c = 0;
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t) gridDim.x * blockDim.x) {
    uint32_t w = bm[i];
    if (i == words - 1 && (nbits & 31)) w &= (1u << (nbits & 31)) - 1u;
    c += __popc(w);
  }
  c = warp_sum(c);
  if (lane_id() == 0 && c) atomicAdd(out, c);
}
}  // namespace
}  // namespace gl

extern "C" {

int gl_bitmap_create(uint32_t** out, uint64_t nbits) {
  GL_ARG(out, "null argument");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  const size_t bytes = sizeof(uint32_t) * ((size_t) ((nbits + 31) / 32) + 1);
  GL_CUDA(cudaMalloc(out, bytes));
  GL_CUDA(cudaMemset(*out, 0, bytes));
  return GL_OK;
}
int gl_bitmap_clear(void* stream, uint32_t* bitmap, uint64_t nbits) {
  GL_ARG(bitmap, "null argument");
  GL_CUDA(cudaMemsetAsync(bitmap, 0, sizeof(uint32_t) * (size_t) ((nbits + 31) / 32), (cudaStream_t) stream));
  return GL_OK;
}
int gl_bitmap_count(void* stream, const uint32_t* bitmap, uint64_t nbits, uint64_t* count_host) {
  GL_ARG(bitmap && count_host, "null argument");
  cudaStream_t s = (cudaStream_t) stream;
  DevBuf<unsigned long long> d;
  GL_CUDA(d.alloc(1));
  GL_CUDA(cudaMemsetAsync(d, 0, 8, s));
  if (nbits) GL_LAUNCH(k_bitmap_count, num_sms() * 4, 256, s, bitmap, nbits, d);
  unsigned long long h = 0;
  GL_CUDA(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, s));
  GL_CUDA(cudaStreamSynchronize(s));
  *count_host = h;
  return GL_OK;
}
int gl_bitmap_destroy(uint32_t* bitmap) {
  if (bitmap) GL_CUDA(cudaFree(bitmap));
  return GL_OK;
}

int gl_mm_send_outer(gl_mm_t* m, void* stream, const gl_frag_t* frag, uint32_t* remote, const void* state,
                     int value_bytes, int clear_bits) {
  GL_ARG(m && frag && remote, "null argument");
  GL_ARG(value_bytes == 0 || ((value_bytes == 4 || value_bytes == 8) && state), "gl_mm_send_outer: value_bytes must be 0, 4 or 8");
  if (m->mm.fnum == 1 || frag->ovnum == 0) return GL_OK;
  cudaStream_t s = (cudaStream_t) stream;
  gl_mm_view mv;
  GL_TRY(gl_mm_view_get(m, &mv));
  const int grid = num_sms() * 4;
  if (value_bytes == 0) GL_LAUNCH(k_mm_send_outer<0>, grid, 256, s, mv, remote, frag->ivnum, frag->ovnum, frag->ovgid, state, 0);
  else if (value_bytes == 4) GL_LAUNCH(k_mm_send_outer<4>, grid, 256, s, mv, remote, frag->ivnum, frag->ovnum, frag->ovgid, state, 0);
  else GL_LAUNCH(k_mm_send_outer<8>, grid, 256, s, mv, remote, frag->ivnum, frag->ovnum, frag->ovgid, state, 0);
  if (clear_bits) GL_LAUNCH(k_clear_bit_range, num_sms(), 256, s, remote, frag->ivnum, frag->ivnum + frag->ovnum);
  return GL_OK;
}

int gl_mm_create(gl_mm_t** out, gl_comm_t* comm) {
  GL_ARG(out, "null argument");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  if (comm && !comm->opened) {
    set_error("gl_mm_create: the communicator is not opened (gl_comm_open)");
    return GL_ERR_STATE;
  }
  gl_mm* m = new gl_mm;
  m->comm = comm;
  gl_frag_view fv;
  memset(&fv, 0, sizeof(fv));
  fv.fid = comm ? comm->fid : 0;
  fv.fnum = comm ? comm->fnum : 1;
  id_parser_init(fv.fnum, &fv.fid_offset, &fv.id_mask);
  int st = m->mm.Init(comm, fv, 1);
  if (st != GL_OK) {
    delete m;
    return st;
  }
  if (m->d_ctrl.alloc(1) != cudaSuccess) {
    delete m;
    set_error("gl_mm_create: device allocation failed");
    return GL_ERR_NOMEM;
  }
  *out = m;
  return GL_OK;
}

int gl_mm_init_buffer(gl_mm_t* m, size_t send_bytes, size_t recv_bytes) {
  GL_ARG(m, "null argument");
  if (m->mm.fnum == 1) return GL_OK;
  const size_t need = send_bytes > recv_bytes ? send_bytes : recv_bytes;
  if (need > m->comm->landing_bytes) {
    set_error("gl_mm_init_buffer: %zu bytes per peer exceed the communicator's landing slot (%zu)", need,
              m->comm->landing_bytes);
    return GL_ERR_ARG;
  }
  return GL_OK;
}

int gl_mm_start(gl_mm_t* m) {
  GL_ARG(m, "null argument");
  m->mm.Start();
  return GL_OK;
}
int gl_mm_start_round(gl_mm_t* m, void* stream) {
  GL_ARG(m, "null argument");
  return m->mm.StartARound((cudaStream_t) stream);
}
int gl_mm_finish_round(gl_mm_t* m, void* stream) {
  GL_ARG(m, "null argument");
  return m->mm.FinishARound((cudaStream_t) stream);
}
int gl_mm_to_terminate(gl_mm_t* m, int* out) {
  GL_ARG(m && out, "null argument");
  *out = m->mm.ToTerminate() ? 1 : 0;
  return GL_OK;
}
int gl_mm_force_continue(gl_mm_t* m) {
  GL_ARG(m, "null argument");
  m->mm.ForceContinue();
  return GL_OK;
}
int gl_mm_view_get(gl_mm_t* m, gl_mm_view* out) {
  GL_ARG(m && out, "null argument");
  const MsgView v = m->mm.view();
  memset(out, 0, sizeof(*out));
  out->fid = v.fid;
  out->fnum = v.fnum;
  out->fid_offset = v.fid_offset;
  out->id_mask = v.id_mask;
  out->capacity_bytes = v.capacity;
  out->send_slot = v.send_slot;
  out->send_bytes = v.send_count;
  out->recv_slot = v.recv_slot;
  out->recv_bytes = v.recv_count;
  return GL_OK;
}
uint64_t gl_mm_bytes_sent(gl_mm_t* m) { return m ? m->mm.bytes_sent : 0; }
void gl_mm_destroy(gl_mm_t* m) {
  delete m;
}

int gl_mm_process(gl_mm_t* m, void* stream, const gl_msg_op* op, uint64_t* items_host) {
  GL_ARG(m && op, "null argument");
  GL_ARG(op->kind == GL_MSG_SET_BIT || op->state, "gl_mm_process: state array required");
  if (items_host) *items_host = 0;
  if (m->mm.fnum == 1) return GL_OK;
  cudaStream_t s = (cudaStream_t) stream;
  gl_mm_view mv;
  GL_TRY(gl_mm_view_get(m, &mv));
  unsigned long long* cnt = (unsigned long long*) m->d_ctrl.get();
  GL_CUDA(cudaMemsetAsync(cnt, 0, 8, s));
  const int grid = num_sms() * 4;
  switch (op->kind) {
    case GL_MSG_SET_BIT: GL_LAUNCH((k_mm_process<uint32_t, GL_MSG_SET_BIT>), grid, 256, s, mv, (uint32_t*) nullptr, op->out_bitmap, cnt); break;
    case GL_MSG_MIN_U32: GL_LAUNCH((k_mm_process<uint32_t, GL_MSG_MIN_U32>), grid, 256, s, mv, (uint32_t*) op->state, op->out_bitmap, cnt); break;
    case GL_MSG_MIN_F32: GL_LAUNCH((k_mm_process<float, GL_MSG_MIN_F32>), grid, 256, s, mv, (float*) op->state, op->out_bitmap, cnt); break;
    case GL_MSG_MIN_F64: GL_LAUNCH((k_mm_process<double, GL_MSG_MIN_F64>), grid, 256, s, mv, (double*) op->state, op->out_bitmap, cnt); break;
    case GL_MSG_ADD_F32: GL_LAUNCH((k_mm_process<float, GL_MSG_ADD_F32>), grid, 256, s, mv, (float*) op->state, op->out_bitmap, cnt); break;
    case GL_MSG_ADD_F64: GL_LAUNCH((k_mm_process<double, GL_MSG_ADD_F64>), grid, 256, s, mv, (double*) op->state, op->out_bitmap, cnt); break;
    default:
      set_error("gl_mm_process: unknown op kind %d", op->kind);
      return GL_ERR_ARG;
  }
  if (items_host) {
    unsigned long long h = 0;
    GL_CUDA(cudaMemcpyAsync(&h, cnt, 8, cudaMemcpyDeviceToHost, s));
    GL_CUDA(cudaStreamSynchronize(s));
    *items_host = h;
  }
  return GL_OK;
}

int gl_mm_mirror_plan(gl_mm_t* m, void* stream, const gl_frag_t* frag) {
  GL_ARG(m && frag, "null argument");
  gl_frag_view fv;
  frag_fill_view(frag, &fv);
  if (fv.fnum != m->mm.fnum || fv.fid != m->mm.fid) {
    set_error("gl_mm_mirror_plan: the fragment is not this rank's member of the group");
    return GL_ERR_ARG;
  }
  return m->mm.BuildMirrorPlan((cudaStream_t) stream, fv);
}
int gl_mm_sync_values_to_ghosts(gl_mm_t* m, void* stream, void* values, int elem_bytes) {
  GL_ARG(m && values && (elem_bytes == 4 || elem_bytes == 8), "gl_mm_sync_values_to_ghosts: bad argument");
  if (m->mm.fnum > 1 && !m->mm.plan_built) {
    set_error("gl_mm_sync_values_to_ghosts: call gl_mm_mirror_plan first");
    return GL_ERR_STATE;
  }
  return m->mm.SyncValuesToGhosts((cudaStream_t) stream, values, elem_bytes);
}
int gl_mm_sync_bits_to_ghosts(gl_mm_t* m, void* stream, uint32_t* bitmap) {
  GL_ARG(m && bitmap, "null argument");
  if (m->mm.fnum > 1 && !m->mm.plan_built) {
    set_error("gl_mm_sync_bits_to_ghosts: call gl_mm_mirror_plan first");
    return GL_ERR_STATE;
  }
  return m->mm.SyncBitsToGhosts((cudaStream_t) stream, bitmap);
}

int gl_allreduce(gl_mm_t* m, void* stream, void* inout_host, int dtype, int op) {
  GL_ARG(m && inout_host, "null argument");
  GL_ARG(op >= 0 && op <= 2 && (dtype == 0 || dtype == 1), "gl_allreduce: bad dtype/op");
  if (m->mm.fnum == 1) return GL_OK;
  // the unused lanes carry the operation's identity
  long long a = 0, b = 0;
  double c = 0;
  if (op == 1) { a = b = INT64_MAX; c = 1.7976931348623157e308; }
  if (op == 2) { a = b = INT64_MIN; c = -1.7976931348623157e308; }
  if (dtype == 0) a = *(long long*) inout_host; else c = *(double*) inout_host;
  GL_TRY(m->mm.PeerAllReduce((cudaStream_t) stream, &a, &b, &c, op));
  if (dtype == 0) *(long long*) inout_host = a; else *(double*) inout_host = c;
  return GL_OK;
}

}  // extern "C"
