// app_base.h — PIE app scaffolding on top of the engine.
//
// Mirrors grape::cuda::GPUAppBase / GPUWorker / GPUMessageManager
// (grape/cuda/app/gpu_app_base.h:39-92, grape/cuda/worker/gpu_worker.h:44-107,
//  grape/cuda/parallel/gpu_message_manager.h:160-431): an app implements
// PEval / IncEval against a MessageManager; the worker loop runs PEval once
// and IncEval until every fragment is idle.
#pragma once
#include <vector>

#include "comm.h"
#include "engine.cuh"
#include "fragment.h"

namespace gl {

// Engine: per-app launch geometry + device control block + hub work list.
struct Engine {
  cudaStream_t stream = nullptr;
  int sm_count = 0;
  int grid = 0;            // persistent grid: SMs x resident CTAs
  DevBuf<ScanCtrl> ctrl;
  PinnedBuf<ScanCtrl> h_ctrl;  // host mirror
  DevBuf<HubItem> hubs;
  uint32_t hub_cap = 0;
  uint32_t hub_deg = kHubDeg;
  int init(const gl_frag* f);
  void destroy();
  int reset_ctrl();                 // async zero of the control block
  int fetch_ctrl();                 // D2H + sync; h_ctrl valid afterwards
};

// Every fragment's CSR part (row pointers over its inner vertices, m column entries) replicated on every
// fragment of the group: CUDA IPC export, one blob exchange, bulk peer copies, then a peer barrier so no
// fragment changes its arrays while a peer still reads them.  Collective when fnum > 1.  The device
// tables d_rp / d_col [fnum] point at the replicas and, at [fid], at this fragment's own arrays (which
// must be whole cudaMalloc allocations).  An optional per-entry weight array w travels the same way
// (d_w [fnum]; left unallocated when w is null).
struct PeerCsr {
  std::vector<DevBuf<uint64_t>> rep_rp;
  std::vector<DevBuf<uint32_t>> rep_col, rep_w;
  DevBuf<const uint64_t*> d_rp;
  DevBuf<const uint32_t*> d_col, d_w;
  int replicate(MessageManager& mm, cudaStream_t s, const gl_frag_view& fv, const uint64_t* rp,
                const uint32_t* col, uint64_t m, const uint32_t* w = nullptr);
};

struct StepRecorder {
  std::vector<cudaEvent_t> ev;
  std::vector<uint64_t> entries;
  std::vector<uint32_t> frontier;
  std::vector<uint8_t> mode;
  size_t used = 0;
  cudaEvent_t next();
  void reset() { used = 0; entries.clear(); frontier.clear(); mode.clear(); }
  void destroy();
};

}  // namespace gl

struct gl_vcfrag;

struct gl_app {
  int kind = 0;
  gl_frag* frag = nullptr;
  gl_comm* comm = nullptr;
  gl_app_config cfg;
  gl::Engine eng;
  gl::MessageManager mm;
  gl::StepRecorder rec;
  gl_frag_view fv;
  // accumulated over one Query()
  uint64_t q_entries = 0, q_frontier = 0, q_touched = 0;
  int rounds = 0;
  const gl_vm_t* vmap = nullptr;   // borrowed device vertex map (gl_app_set_vertex_map)

  virtual ~gl_app() {}
  virtual int Setup() = 0;                     // one-off allocations (GPUWorker::Init)
  virtual int Init() = 0;                      // context Init (per query state reset)
  virtual int PEval() = 0;
  virtual int IncEval() = 0;
  virtual int Result(void* host_out, size_t bytes) = 0;
  virtual size_t ResultElemBytes() const = 0;
  virtual size_t ResultCount() const { return frag ? frag->ivnum : 0; }   // elements gl_app_result writes
  virtual int ResultOids(int64_t* host_out, size_t count);               // gl_app_result_oids (worker.cu)
  virtual void FillStats(gl_query_stats*) {}   // apps that time supersteps on the device
  virtual void AfterRound() {}                 // runs after every FinishARound (global round statistics)
  virtual int SetSources(const int64_t*, uint64_t);                      // gl_app_set_sources (worker.cu)
  // Apps whose whole query is one launch record this event in-stream right after the query's last
  // device operation (kernel + control-block read-back); query_ms then ends there instead of at the
  // event the host records after it woke up from the stream synchronisation (host latency is part of
  // e2e, not of the device-timed value).  null: the worker loop's last event.
  cudaEvent_t query_end = nullptr;
  // record per-superstep stats (called by apps after fetch_ctrl)
  void note_step(uint64_t entries, uint32_t frontier, int mode) {
    rec.entries.push_back(entries);
    rec.frontier.push_back(frontier);
    rec.mode.push_back((uint8_t) mode);
    q_entries += entries;
    q_frontier += frontier;
  }
};

namespace gl {
// hub-first (descending degree) order of the inner vertices: perm[lid] = rank, order[rank] = lid
int build_hub_order(cudaStream_t s, const uint64_t* rp, uint32_t n, DevBuf<uint32_t>* perm_out, DevBuf<uint32_t>* order_out);
int build_permuted_csr(cudaStream_t s, const uint64_t* rp, const uint32_t* col, uint64_t m, uint32_t n,
                       const uint32_t* order, const uint32_t* perm, DevBuf<uint64_t>* rp_out, DevBuf<uint32_t>* col_out,
                       const void* w4 = nullptr, DevBuf<uint32_t>* w4_out = nullptr, bool sort_rows = true);
// every row [rp[i], rp[i+1]) of *col sorted ascending, the entries of *val (when non-null) moved with their
// keys (both arrays are replaced by sorted copies); V is uint32_t or uint64_t
template <typename V = uint32_t>
int sort_csr_rows(cudaStream_t s, const uint64_t* rp, uint32_t n, uint64_t m, DevBuf<uint32_t>* col,
                  DevBuf<V>* val = nullptr);
gl_app* make_bfs();
gl_app* make_sssp_f32();
gl_app* make_sssp_f64();
gl_app* make_wcc();
gl_app* make_pagerank();
gl_app* make_pagerank_directed();
gl_app* make_pagerank_local();
gl_app* make_cdlp();
gl_app* make_cdlp_directed();
gl_app* make_lcc();
gl_app* make_lcc_directed();
gl_app* make_wcc_opt();
gl_app* make_core_decomposition();
gl_app* make_kcore();
gl_app* make_kclique();
gl_app* make_bc();
gl_app* make_bc_sources();
gl_app* make_pagerank_vc(gl_vcfrag* f);
}  // namespace gl
