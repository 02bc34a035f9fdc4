// ref_pagerank_vc_driver.cc — runs the UNMODIFIED reference CPU app PageRankVC
// (examples/analytical_apps/pagerank/pagerank_vc.h, what run_app --vc --application pagerank runs,
// run_app_vc.h) on ImmutableVertexcutFragment<uint64_t, EmptyType, EmptyType>.
// TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by pagerank_vc.mk next to ref_driver.
//
// The fragment is loaded the way run_app_vc.h loads it: LoadVertexcutGraph (VCFragmentLoader, the
// 2-D VCPartitioner) from an edge file and the vertex count.  Under the MPI shim GL_MPI_NP=N runs N
// fragments (N must be a perfect square).  Query(pr_d, pr_mr) is timed; each rank writes its master
// vertices to <out>.<fid>, one "oid value" line each, the value with 17 significant digits.
//
// usage: ref_pagerank_vc_driver (--efile FILE --vnum N | --rmat SCALE,EDGEFACTOR,SEED)
//                               [--pr_d D] [--pr_mr R] [--threads T] [--repeat K] [--out PREFIX]
// efile: "src dst" per line, vertices 0..N-1; --rmat writes the generator's edges (oracle/rmat_gen.h)
// to a temporary edge file first.
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <grape/grape.h>
#include <grape/fragment/immutable_vertexcut_fragment.h>
#include <grape/fragment/loader.h>

#include "../rmat_gen.h"
#include "pagerank/pagerank_vc.h"

using namespace grape;  // NOLINT

namespace {

int Run(const CommSpec& comm_spec, const std::string& efile, int64_t vnum, double pr_d, int pr_mr, int threads,
        int repeat, const std::string& out) {
  using FRAG_T = ImmutableVertexcutFragment<uint64_t, EmptyType, EmptyType>;
  auto t0 = std::chrono::steady_clock::now();
  LoadGraphSpec graph_spec = DefaultLoadGraphSpec();
  std::shared_ptr<FRAG_T> fragment = LoadVertexcutGraph<FRAG_T>(efile, vnum, comm_spec, graph_spec);
  const double load_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  ParallelEngineSpec spec = MultiProcessSpec(comm_spec, false);
  if (threads > 0) spec.thread_num = threads;
  std::vector<double> ms;
  for (int r = 0; r < repeat; ++r) {   // the worker is single-shot: a fresh app + worker per query
    using APP_T = PageRankVC<FRAG_T>;
    auto app = std::make_shared<APP_T>();
    auto worker = APP_T::CreateWorker(app, fragment);
    worker->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker->Query(pr_d, pr_mr);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    if (r + 1 == repeat && !out.empty()) {
      auto ctx = worker->GetContext();
      const std::string path = out + "." + std::to_string(comm_spec.fid());
      FILE* f = fopen(path.c_str(), "w");
      if (!f) return 2;
      for (auto v : fragment->MasterVertices())
        fprintf(f, "%llu %.17g\n", (unsigned long long) v.GetValue(), ctx->master_result[v]);
      fclose(f);
    }
    worker->Finalize();
  }
  if (comm_spec.worker_id() == 0) {
    printf("{\"app\": \"pagerank_vc\", \"fnum\": %u, \"threads\": %u, \"hardware_concurrency\": %u, "
           "\"load_s\": %.3f, \"vertices\": %lld, \"query_ms\": [",
           comm_spec.fnum(), spec.thread_num, std::thread::hardware_concurrency(), load_s, (long long) vnum);
    for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
    printf("]}\n");
    fflush(stdout);
  }
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string efile, rmat, out;
  int64_t vnum = -1;
  double pr_d = 0.85;
  int pr_mr = 10, threads = 0, repeat = 1;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--efile") efile = v;
    else if (a == "--vnum") vnum = atoll(v.c_str());
    else if (a == "--rmat") rmat = v;
    else if (a == "--pr_d") pr_d = atof(v.c_str());
    else if (a == "--pr_mr") pr_mr = atoi(v.c_str());
    else if (a == "--threads") threads = atoi(v.c_str());
    else if (a == "--repeat") repeat = atoi(v.c_str());
    else if (a == "--out") out = v;
    else { fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
  }
  std::string tmp;
  if (!rmat.empty()) {
    // before InitMPIComm: the shim forks the ranks there, so only one process writes the file
    int scale = 0, ef = 16;
    unsigned long long seed = 1;
    if (sscanf(rmat.c_str(), "%d,%d,%llu", &scale, &ef, &seed) < 1 || scale < 1 || scale > 30) {
      fprintf(stderr, "bad --rmat %s\n", rmat.c_str());
      return 2;
    }
    char path[] = "/tmp/ref_pagerank_vc_XXXXXX";
    int fd = mkstemp(path);
    FILE* f = fd >= 0 ? fdopen(fd, "w") : nullptr;
    if (!f) {
      fprintf(stderr, "cannot create a temporary edge file\n");
      return 2;
    }
    const int64_t m = (int64_t) ef << scale;
    for (int64_t i = 0; i < m; ++i) {
      uint64_t a, b;
      rmatdef::edge((uint64_t) i, scale, seed, &a, &b);
      fprintf(f, "%llu %llu\n", (unsigned long long) a, (unsigned long long) b);
    }
    fclose(f);
    tmp = efile = path;
    vnum = 1ll << scale;
  }
  if (efile.empty() || vnum < 1) {
    fprintf(stderr, "need --efile and --vnum, or --rmat\n");
    return 2;
  }
  InitMPIComm();
  int rc = 0;
  {
    CommSpec comm_spec;
    comm_spec.Init(MPI_COMM_WORLD);
    rc = Run(comm_spec, efile, vnum, pr_d, pr_mr, threads, repeat, out);
    MPI_Barrier(comm_spec.comm());
    if (!tmp.empty() && comm_spec.worker_id() == 0) unlink(tmp.c_str());
  }
  FinalizeMPIComm();
  return rc;
}
