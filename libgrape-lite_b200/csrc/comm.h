// comm.h — fragment-group communicator and the per-app message manager.
//
// Replaces grape::cuda::GPUMessageManager + dev::MessageManager +
// dev::InArchive/OutArchive (grape/cuda/parallel/gpu_message_manager.h:45-458,
// grape/cuda/serialization/in_archive.h:36-169, out_archive.h:32-178).
//
// Design: no host-side size exchange and no NCCL send/recv of byte
// archives.  Every rank owns ONE device allocation ("landing area") that its
// peers map through CUDA IPC; a producer kernel writes (lid_at_owner, value)
// items straight into the owner's landing slot over NVLink (peer stores) and
// then publishes the item count.  Slots are double-buffered by round parity so
// that round r+1 producers never overwrite round r items still being applied.
// The only host step per round is one tiny all-reduce that is both the
// barrier and the termination vote (gpu_message_manager.h:400-431 does an
// MPI_Allgather of sizes + MPI_Barrier for the same purpose).
#pragma once
#include <vector>

#include "common.cuh"

constexpr uint32_t GL_MAX_FNUM = 64;
// Header of a landing area: item counts + the peer-barrier slots.
//   [0, 512)      uint32 counts[2][GL_MAX_FNUM]
//   [1024, 7168)  PeerSlot slots[2][GL_MAX_FNUM]   (48 B each)
constexpr size_t GL_COMM_HEADER = 8192;
constexpr size_t GL_COMM_SLOT_OFF = 1024;
struct PeerSlot {            // one rank's contribution to a collective (48 B)
  unsigned long long tag;    // sequence number, written last (release)
  long long i0, i1, i2, i3;
  double d0;
};

struct gl_comm {
  uint32_t fid = 0, fnum = 1;
  gl_allreduce_fn allreduce = nullptr;
  void* user = nullptr;
  size_t landing_bytes = 0;  // per (parity, src) message slot
  size_t mirror_bytes = 0;   // per (parity, src) mirror-sync slot
  char* local_base = nullptr;
  std::vector<char*> peer_base;  // [fnum]; peer_base[fid] == local_base
  bool opened = false;
  unsigned long long seq_base = 0;  // last collective sequence number used on this communicator
  // something other than the fused BFS's frontier segments was written into the mirror slots
  // (value / bit syncs, mirror-plan requests): that app re-zeroes its segments before a query
  bool mirror_dirty = true;
  size_t total_bytes() const {
    return GL_COMM_HEADER + 2 * (size_t) fnum * (landing_bytes + mirror_bytes);
  }
  // byte offset of the mirror slot (parity, src) inside a landing area
  size_t mirror_off(int parity, uint32_t src) const {
    return GL_COMM_HEADER + 2 * (size_t) fnum * landing_bytes +
           ((size_t) parity * fnum + src) * mirror_bytes;
  }
};

namespace gl {

struct ScanCtrl;  // engine.cuh

// Device-side view handed to producer / consumer kernels.
struct MsgView {
  uint32_t fid, fnum;
  int fid_offset;
  uint32_t id_mask;
  uint32_t item_bytes;
  uint32_t capacity;        // items per slot
  char* const* send_slot;   // device table [fnum]: peer landing slot for (parity, me)
  uint32_t* send_count;     // device [fnum] local counters
  const char* const* recv_slot;  // device table [fnum]: my landing slot for (prev parity, src)
  const uint32_t* recv_count;    // device [fnum] (inside my header, prev parity)
};

// Owner-side plan of a BIT sync in word-parallel form.  The lids a holder
// mirrors are ascending, so "the bits of my bitmap at the mirrored lids, in the
// holder's ghost order" is a bit-compress (pext) of the bitmap under a per-holder
// mask: output word j of holder g starts at input word startw[woff[g]+j], after
// skipping (32 j - pref[g][that word]) selected bits.  One thread per OUTPUT
// word, coalesced peer stores, no index list traffic (the lid list costs 4 B per
// mirrored vertex per sync: 64 MB at 16 M mirrors).
struct MirrorBitsPlan {
  uint32_t fnum, iv_words;
  const uint32_t* mask;
  const uint32_t* pref;
  const uint32_t* startw;
  const uint64_t* woff;   // [fnum+1] output words
  const uint64_t* off;    // [fnum+1] mirrored vertices (= output bits)
};

struct MessageManager {
  gl_comm* comm = nullptr;
  uint32_t fid = 0, fnum = 1;
  int fid_offset = 31;
  uint32_t id_mask = 0x7fffffffu;
  uint32_t item_bytes = 8;
  int round = 0;
  bool force_continue = false;
  bool terminate = false;
  uint64_t bytes_sent = 0;
  // device tables
  DevBuf<char*> d_send_slot[2];          // [parity][fnum]
  DevBuf<const char*> d_recv_slot[2];    // [parity][fnum]
  DevBuf<uint32_t> d_send_count;         // [fnum]
  DevBuf<uint32_t> d_zero_count;         // [fnum] zeros: what round 0 of a query receives
  PinnedBuf<uint32_t> h_send_count;      // [fnum+1]
  DevBuf<uint32_t*> d_peer_count[2];     // [parity][fnum] address of my count cell at peer

  int Init(gl_comm* c, const gl_frag_view& fv, uint32_t item_bytes_);
  // GPUMessageManager::StartARound / FinishARound / ToTerminate / ForceContinue
  void Start() { round = 0; force_continue = false; terminate = false; bytes_sent = 0; }
  int StartARound(cudaStream_t s);
  int FinishARound(cudaStream_t s);
  bool ToTerminate() const { return terminate; }
  void ForceContinue() { force_continue = true; }
  // view for producers of the current round and consumers of the previous one
  MsgView view() const;
  // all-reduce helpers (cuda::Communicator::Sum/Min/Max, communicator.h:41-84)
  int AllReduceI64(int64_t* v, int n, int op);
  int AllReduceF64(double* v, int n, int op);
  // Device-side collective over NVLink peer memory: every rank stores its
  // contribution into every peer's header slot and spins until all peers'
  // slots carry this collective's sequence number.  Sum of (i0, i1, d0) in
  // fid order => bit-identical on all ranks.  Also a barrier: it is issued
  // after the round's peer stores on the same stream.
  int PeerAllReduce(cudaStream_t s, long long* i0, long long* i1, double* d0, int op);
  int PeerBarrier(cudaStream_t s);
  // barrier only: enqueued on the stream, no host synchronisation
  int PeerBarrierAsync(cudaStream_t s);
  // all-gather of one small host blob per rank through the landing area
  // (bytes <= landing_bytes; only between rounds, when no message slot of
  // parity 0 is in flight): all[p*bytes ..] = rank p's blob
  int ExchangeBlobs(cudaStream_t s, const void* mine, size_t bytes, std::vector<char>* all);
  // When set, FinishARound's kernel takes the vote straight from the engine's
  // device counters (force_continue |= next_count > 0, statistics = next_count
  // + remote_count, next_edges) and mirrors the control block to `vote_h_ctrl`,
  // so a round closes with ONE host synchronisation.
  const ScanCtrl* vote_ctrl = nullptr;
  ScanCtrl* vote_h_ctrl = nullptr;
  DevBuf<PeerSlot> d_scratch_result;
  // ---- dense mirror sync (owner's inner state -> the outer copies held by
  // other fragments); replaces BatchShuffleMessageManager::SyncInnerVertices.
  // BuildMirrorPlan is collective and must run once (Setup); afterwards every
  // Sync* call is collective too.
  int BuildMirrorPlan(cudaStream_t s, const gl_frag_view& fv);
  bool has_mirror_plan() const { return d_mirror_lids != nullptr || mirror_total == 0 && plan_built; }
  int SyncBitsToGhosts(cudaStream_t s, uint32_t* bitmap);   // ghost bits |= owner bits
  int SyncValuesToGhosts(cudaStream_t s, void* values, int elem_bytes);  // values[ghost] = owner value
  // the same for rows of row_bytes (a multiple of 8, up to 256): values[ghost * row_bytes ..] = owner's row;
  // GL_ERR_ARG when one peer's outer copies do not fit mirror_bytes (see MaxRowBytes)
  int SyncRowsToGhosts(cudaStream_t s, void* values, int row_bytes);
  // the largest row the mirror area holds for every peer's outer copies (after BuildMirrorPlan)
  size_t MaxRowBytes() const;
  bool plan_built = false;
  uint32_t plan_ivnum = 0;
  DevBuf<uint32_t> d_mirror_lids;          // my inner lids mirrored elsewhere, grouped by holder
  DevBuf<uint64_t> d_mirror_off;            // device [fnum+1]
  std::vector<uint64_t> mirror_off;         // host  [fnum+1]
  uint64_t mirror_total = 0;
  uint32_t* d_ghost_range = nullptr;        // device [fnum+1]: outer lids owned by each fid (outer_range)
  std::vector<uint32_t> ghost_range;
  DevBuf<char*> d_msend[2];         // [parity][fnum] mirror slot (parity, me) at peer
  DevBuf<const char*> d_mrecv[2];   // [parity][fnum] my mirror slot (parity, src)
  unsigned long long mirror_seq = 0;
  // word-parallel form of the plan for bit syncs (see MirrorBitsPlan below)
  bool mirror_sorted = false;
  uint32_t iv_words = 0;
  DevBuf<uint32_t> d_mirror_mask;     // [fnum][iv_words]
  DevBuf<uint32_t> d_mirror_pref;     // [fnum][iv_words]
  DevBuf<uint32_t> d_mirror_startw;   // [woff[fnum]]
  DevBuf<uint64_t> d_mirror_woff;     // [fnum+1] output words per holder (prefix)
  uint64_t mirror_out_words = 0;
  struct MirrorBitsPlan bits_plan() const;
  // extra statistics carried by the round vote (summed over fragments)
  long long stat_in[2] = {0, 0};
  long long stat_out[2] = {0, 0};
  bool use_peer_barrier = true;
  // set by an app whose PEval ran the whole query inside one kernel that already agreed on
  // termination over its in-kernel collectives (fused BFS): the next FinishARound is then a
  // local no-op on every rank instead of one more host-launched barrier + vote
  bool decided_terminate = false;
  cudaStream_t stream_for_collectives = nullptr;
  unsigned long long seq = 0;
  DevBuf<PeerSlot*> d_peer_slot[2];  // [parity][fnum] my slot at peer p
  PinnedBuf<PeerSlot> h_result;
};

#ifdef __CUDACC__
GL_DEV bool mirror_pack_bits_phase(const MirrorBitsPlan& P, const uint32_t* __restrict__ bitmap,
                                   char* const* msend, uint64_t gtid, uint64_t nthreads) {
  const uint64_t total = P.woff[P.fnum];
  const bool wrote = gtid < total;
  constexpr int kB = 4;   // output words in flight per thread (the loads of a word form a dependent chain)
  for (uint64_t i0 = gtid; i0 < total; i0 += (uint64_t) kB * nthreads) {
    uint32_t w[kB], g[kB], need[kB], skip[kB], sel[kB], val[kB];
    uint64_t j[kB];
    bool ok[kB];
#pragma unroll
    for (int q = 0; q < kB; ++q) {
      const uint64_t i = i0 + (uint64_t) q * nthreads;
      ok[q] = i < total;
      w[q] = ok[q] ? P.startw[i] : 0u;
      uint32_t gg = 0;
      while (ok[q] && gg + 1 < P.fnum && i >= P.woff[gg + 1]) ++gg;
      g[q] = gg;
      j[q] = ok[q] ? i - P.woff[gg] : 0;
    }
#pragma unroll
    for (int q = 0; q < kB; ++q) {
      const size_t at = (size_t) g[q] * P.iv_words + w[q];
      sel[q] = ok[q] ? P.mask[at] : 0u;
      skip[q] = ok[q] ? (uint32_t) (32 * j[q] - P.pref[at]) : 0u;
      val[q] = ok[q] ? bitmap[w[q]] : 0u;
      const uint64_t nbits = P.off[g[q] + 1] - P.off[g[q]];
      need[q] = ok[q] ? (uint32_t) ((nbits - 32 * j[q]) < 32 ? (nbits - 32 * j[q]) : 32) : 0u;
    }
#pragma unroll
    for (int q = 0; q < kB; ++q) {
      if (!ok[q]) continue;
      const uint32_t* mask = P.mask + (size_t) g[q] * P.iv_words;
      uint32_t out = 0, k = 0, ww = w[q], s_ = sel[q], v_ = val[q], sk = skip[q];
      if (sk == 0 && s_ == 0xFFFFFFFFu && need[q] == 32) {   // dense fast path
        out = v_;
      } else {
        for (;;) {
          while (sk && s_) {
            s_ &= s_ - 1;
            --sk;
          }
          while (s_ && k < need[q]) {
            const uint32_t b = __ffs(s_) - 1;
            out |= ((v_ >> b) & 1u) << k;
            ++k;
            s_ &= s_ - 1;
          }
          if (k >= need[q]) break;
          ++ww;
          s_ = mask[ww];
          v_ = bitmap[ww];
        }
      }
      ((uint32_t*) msend[g[q]])[j[q]] = out;
    }
  }
  return wrote;
}

// append one item to the slot of fragment `dst` (warp-aggregated per
// destination; replaces dev::InArchive::AddBytesWarpOpt, in_archive.h:51-67)
template <typename Item>
GL_DEV void msg_send(const MsgView& mv, bool pred, uint32_t dst, const Item& it) {
  // group lanes by destination
  uint32_t active = __ballot_sync(0xffffffffu, pred);
  if (!pred) return;
  uint32_t peers = __match_any_sync(active, dst);
  uint32_t leader = __ffs(peers) - 1;
  uint32_t base = 0;
  if (lane_id() == leader) base = atomicAdd(mv.send_count + dst, __popc(peers));
  base = __shfl_sync(peers, base, leader);
  uint32_t pos = base + __popc(peers & ((1u << lane_id()) - 1));
  if (pos < mv.capacity) ((Item*) mv.send_slot[dst])[pos] = it;
}
#endif

}  // namespace gl
