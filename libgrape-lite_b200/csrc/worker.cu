// worker.cu — engine bookkeeping and the PIE worker loop behind the C ABI.
// Replaces grape::cuda::GPUWorker::{Init,Query} (grape/cuda/worker/gpu_worker.h:44-107).
#include "apps_common.cuh"
#include "vcfrag.h"

namespace gl {

int Engine::init(const gl_frag* f) {
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  sm_count = di->sm_count;
  grid = sm_count * 8;
  GL_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  GL_CUDA(ctrl.alloc(1));
  GL_CUDA(cudaMemset(ctrl, 0, sizeof(ScanCtrl)));
  GL_CUDA(h_ctrl.alloc(1));
  memset(h_ctrl, 0, sizeof(ScanCtrl));
  // every hub row has > hub_deg entries, so (#pieces) <= M/kHubChunk + M/hub_deg
  uint64_t m = f ? std::max<uint64_t>(f->oe.entries, f->ie.entries) : 0;   // null: an app on a vertex-cut fragment
  uint64_t cap = m / kHubChunk + m / std::max<uint32_t>(hub_deg, 1) + 1024;
  hub_cap = (uint32_t) std::min<uint64_t>(cap, 0x7FFFFFFFull);
  GL_CUDA(hubs.alloc(hub_cap));
  return GL_OK;
}

void Engine::destroy() {
  if (stream) cudaStreamDestroy(stream);
  stream = nullptr;
}

int Engine::reset_ctrl() {
  GL_CUDA(cudaMemsetAsync(ctrl, 0, sizeof(ScanCtrl), stream));
  return GL_OK;
}

int Engine::fetch_ctrl() {
  GL_CUDA(cudaMemcpyAsync(h_ctrl, ctrl, sizeof(ScanCtrl), cudaMemcpyDeviceToHost, stream));
  GL_CUDA(cudaStreamSynchronize(stream));
  return GL_OK;
}

cudaEvent_t StepRecorder::next() {
  if (used == ev.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    ev.push_back(e);
  }
  return ev[used++];
}
void StepRecorder::destroy() {
  for (auto e : ev) cudaEventDestroy(e);
  ev.clear();
}

LabelMap label_map(const gl_app& a) {
  LabelMap lm;
  lm.fid_offset = a.fv.fid_offset;
  lm.id_mask = a.fv.id_mask;
  lm.fnum = a.fv.fnum;
  lm.chunk = a.frag->part_chunk;
  lm.inner_oids = a.fv.inner_oids;
  lm.oid_base = a.fv.oid_base;
  lm.vm_l2o = nullptr;
  lm.vm_off = nullptr;
  if (a.vmap) {
    gl_vm_view v;
    if (gl_vm_view_get(a.vmap, &v) == GL_OK && v.fnum == a.fv.fnum) {
      lm.vm_l2o = v.l2o;
      lm.vm_off = v.off;
    }
  }
  return lm;
}

}  // namespace gl

using namespace gl;

extern "C" {

int gl_app_set_vertex_map(gl_app_t* a, const gl_vm_t* vm) {
  GL_ARG(a, "null argument");
  GL_ARG(a->kind != GL_APP_PAGERANK_VC, "an app on a vertex-cut fragment reports oids itself: no vertex map");
  if (vm) {
    gl_vm_view v;
    GL_TRY(gl_vm_view_get(vm, &v));
    if (v.fnum != a->fv.fnum) {
      set_error("gl_app_set_vertex_map: the map describes %u fragments, the app's fragment group has %u", v.fnum, a->fv.fnum);
      return GL_ERR_ARG;
    }
  }
  a->vmap = vm;
  return GL_OK;
}

void gl_app_config_default(gl_app_config* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->lb = GL_LB_CM;
  c->source_oid = 0;
  c->pr_delta = 0.85;
  c->max_round = 10;
  c->direction_opt = 1;
  c->fuse_supersteps = 1;
}

int gl_app_create(gl_app_t** out, int kind, gl_frag_t* frag, gl_comm_t* comm,
                  const gl_app_config* cfg) {
  GL_ARG(out && frag, "null argument");
  if (frag->offloaded) {
    set_error("fragment topology is offloaded");
    return GL_ERR_STATE;
  }
  gl_app* a = nullptr;
  switch (kind) {
    case GL_APP_BFS: a = make_bfs(); break;
    case GL_APP_SSSP: a = (cfg && cfg->sssp_f64) ? make_sssp_f64() : make_sssp_f32(); break;
    case GL_APP_WCC: a = make_wcc(); break;
    case GL_APP_PAGERANK: a = make_pagerank(); break;
    case GL_APP_CDLP: a = make_cdlp(); break;
    case GL_APP_LCC: a = make_lcc(); break;
    case GL_APP_WCC_OPT: a = make_wcc_opt(); break;
    case GL_APP_CORE_DECOMPOSITION: a = make_core_decomposition(); break;
    case GL_APP_KCORE: a = make_kcore(); break;
    case GL_APP_KCLIQUE: a = make_kclique(); break;
    case GL_APP_BC: a = make_bc(); break;
    case GL_APP_BC_SOURCES: a = make_bc_sources(); break;
    case GL_APP_LCC_DIRECTED: a = make_lcc_directed(); break;
    case GL_APP_CDLP_DIRECTED: a = make_cdlp_directed(); break;
    case GL_APP_PAGERANK_DIRECTED: a = make_pagerank_directed(); break;
    case GL_APP_PAGERANK_LOCAL: a = make_pagerank_local(); break;
    case GL_APP_PAGERANK_VC:
      set_error("GL_APP_PAGERANK_VC runs on a vertex-cut fragment: use gl_vc_app_create");
      return GL_ERR_ARG;
    default:
      set_error("unknown app kind %d", kind);
      return GL_ERR_ARG;
  }
  if (!a) {
    set_error("app kind %d is not available in this build", kind);
    return GL_ERR_STATE;
  }
  a->kind = kind;
  a->frag = frag;
  a->comm = comm;
  if (cfg) a->cfg = *cfg; else gl_app_config_default(&a->cfg);
  frag_fill_view(frag, &a->fv);
  int st = a->eng.init(frag);
  if (st == GL_OK && frag->fnum > 1 && !comm) {
    set_error("fragment has fnum=%u: a communicator is required", frag->fnum);
    st = GL_ERR_COMM;
  }
  if (st == GL_OK) st = a->Setup();
  if (st != GL_OK) {
    gl_app_destroy(a);
    return st;
  }
  *out = a;
  return GL_OK;
}

int gl_vc_app_create(gl_app_t** out, int kind, gl_vcfrag_t* frag, gl_comm_t* comm, const gl_app_config* cfg) {
  GL_ARG(out && frag, "null argument");
  if (kind != GL_APP_PAGERANK_VC) {
    set_error("app kind %d does not run on a vertex-cut fragment (GL_APP_PAGERANK_VC only)", kind);
    return GL_ERR_ARG;
  }
  gl_app* a = make_pagerank_vc(frag);
  a->kind = kind;
  a->comm = comm;
  if (cfg) a->cfg = *cfg; else gl_app_config_default(&a->cfg);
  memset(&a->fv, 0, sizeof(a->fv));
  a->fv.fid = frag->fid;
  a->fv.fnum = frag->fnum;
  a->fv.fid_offset = 31;
  a->fv.id_mask = 0x7fffffffu;
  a->fv.total_vnum = frag->n;
  int st = a->eng.init(nullptr);
  if (st == GL_OK) st = a->Setup();
  if (st != GL_OK) {
    gl_app_destroy(a);
    return st;
  }
  *out = a;
  return GL_OK;
}

int gl_app_query(gl_app_t* a, gl_query_stats* stats) {
  GL_ARG(a, "null argument");
  const uint64_t launches0 = g_kernel_launches;
  a->rec.reset();
  a->query_end = nullptr;
  a->q_entries = a->q_frontier = a->q_touched = 0;
  a->rounds = 0;
  GL_TRY(a->Init());  // context Init (gpu_worker.h:61): resets per-query state
  a->mm.Start();
  cudaStream_t s = a->eng.stream;
  // run_cuda_app.h:117 puts an MPI_Barrier between Init and the timed Query.  Here the barrier is a
  // device-side one on the query's stream: the GPUs' start events are then aligned to a few
  // microseconds instead of the hosts' wake-up jitter (which the first in-kernel collective of a
  // fused query would otherwise absorb inside the timed region).
  if (a->fv.fnum > 1 && a->mm.use_peer_barrier && a->comm && a->comm->opened) GL_TRY(a->mm.PeerBarrierAsync(s));
  // --- the timed region of the reference: GPUWorker::Query (gpu_worker.h:69-107)
  GL_CUDA(cudaEventRecord(a->rec.next(), s));
  GL_TRY(a->mm.StartARound(s));
  GL_TRY(a->PEval());
  GL_TRY(a->mm.FinishARound(s));
  a->AfterRound();
  GL_CUDA(cudaEventRecord(a->rec.next(), s));
  a->rounds = 1;
  while (!a->mm.ToTerminate()) {
    GL_TRY(a->mm.StartARound(s));
    GL_TRY(a->IncEval());
    GL_TRY(a->mm.FinishARound(s));
    a->AfterRound();
    GL_CUDA(cudaEventRecord(a->rec.next(), s));
    ++a->rounds;
    if (a->rounds > 1000000) {
      set_error("superstep limit exceeded");
      return GL_ERR_STATE;
    }
  }
  GL_CUDA(cudaStreamSynchronize(s));
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->supersteps = a->rounds;
    float ms = 0;
    cudaEventElapsedTime(&ms, a->rec.ev[0], a->query_end ? a->query_end : a->rec.ev[a->rec.used - 1]);
    stats->query_ms = ms;
    if (getenv("GL_KTIME")) fprintf(stderr, "[gl-ktime] query %.1f us (start event -> end event)\n", ms * 1e3);
    stats->entries_scanned = a->q_entries;
    stats->frontier_vertices = a->q_frontier;
    stats->touched_vertices = a->q_touched;
    stats->kernel_launches = g_kernel_launches - launches0;
    stats->msg_bytes_sent = a->mm.bytes_sent;
    int n = (int) std::min<size_t>(a->rec.used - 1, GL_MAX_STEP_STATS);
    stats->n_steps = n;
    for (int i = 0; i < n; ++i) {
      float t = 0;
      cudaEventElapsedTime(&t, a->rec.ev[i], a->rec.ev[i + 1]);
      stats->step_ms[i] = t;
      // step i = round i; apps record one note per IncEval (round >= 1)
      if (i >= 1 && (size_t) (i - 1) < a->rec.entries.size()) {
        stats->step_entries[i] = a->rec.entries[i - 1];
        stats->step_frontier[i] = a->rec.frontier[i - 1];
        stats->step_mode[i] = a->rec.mode[i - 1];
      }
    }
    a->FillStats(stats);
  }
  return GL_OK;
}

int gl_app_result(gl_app_t* a, void* host_out, size_t bytes) {
  GL_ARG(a && host_out, "null argument");
  size_t need = a->ResultElemBytes() * a->ResultCount();
  if (bytes < need) {
    set_error("result buffer too small: %zu < %zu", bytes, need);
    return GL_ERR_ARG;
  }
  return a->Result(host_out, bytes);
}

int gl_app_set_sources(gl_app_t* a, const int64_t* oids, uint64_t n) {
  GL_ARG(a, "null argument");
  GL_ARG(oids || n == 0, "gl_app_set_sources: a NULL list must have n = 0");
  return a->SetSources(oids, n);
}

int gl_app_result_oids(gl_app_t* a, int64_t* host_out, size_t count) {
  GL_ARG(a && host_out, "null argument");
  return a->ResultOids(host_out, count);
}

}  // extern "C"

int gl_app::SetSources(const int64_t*, uint64_t) {
  set_error("gl_app_set_sources: app kind %d takes no source list (GL_APP_BC_SOURCES only)", kind);
  return GL_ERR_ARG;
}

int gl_app::ResultOids(int64_t* host_out, size_t count) {
  GL_ARG(count >= frag->ivnum, "bad argument");
  const gl_frag* f = frag;
  if (!f->h_inner_oids.empty()) {
    memcpy(host_out, f->h_inner_oids.data(), sizeof(int64_t) * f->ivnum);
  } else {
    for (uint32_t i = 0; i < f->ivnum; ++i) host_out[i] = f->oid_base + i;
  }
  return GL_OK;
}

extern "C" {

void gl_app_destroy(gl_app_t* a) {
  if (!a) return;
  if (a->eng.stream) l2_persist_clear(a->eng.stream);   // give the L2 set-aside back (common.cu)
  a->rec.destroy();
  a->eng.destroy();
  delete a;
}

}  // extern "C"
