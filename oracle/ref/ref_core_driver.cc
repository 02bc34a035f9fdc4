// ref_core_driver.cc — runs the UNMODIFIED reference CPU apps core_decomposition
// and kcore (examples/analytical_apps/{core_decomposition,kcore}/, the
// run_app --application choices of run_app.h:285-295) on an in-memory graph.
// TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by core.mk next to ref_driver.
//
// Loads the graph the way ref_driver does (BasicFragmentLoader, one fragment,
// undirected, run_app's map partitioner + hashmap idxer), times worker->Query(),
// and, because neither context's Output() writes per-vertex lines (both only
// LOG a sum), writes "oid partial_result" from the context itself.
//
// usage: ref_core_driver --app core_decomposition|kcore
//                        (--graph FILE.bin | --rmat SCALE,EDGEFACTOR,SEED)
//                        [--k K] [--threads T] [--repeat R] [--out FILE]
// graph file: ref_driver's "GRB1" format (oracle/refdriver.py write_graph).
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <grape/grape.h>
#include <grape/fragment/basic_fragment_loader.h>
#include <grape/fragment/immutable_edgecut_fragment.h>

#include "../rmat_gen.h"
#include "core_decomposition/core_decomposition.h"
#include "kcore/kcore.h"

using namespace grape;  // NOLINT

namespace {

struct Graph {
  int64_t n = 0, m = 0;
  std::vector<int64_t> oids, src, dst;
};

bool read_graph(const std::string& path, Graph& g) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  char magic[4];
  int32_t weighted = 0, has_oids = 0;
  bool ok = fread(magic, 1, 4, f) == 4 && memcmp(magic, "GRB1", 4) == 0;
  ok = ok && fread(&g.n, 8, 1, f) == 1 && fread(&g.m, 8, 1, f) == 1;
  ok = ok && fread(&weighted, 4, 1, f) == 1 && fread(&has_oids, 4, 1, f) == 1;
  if (ok && has_oids) {
    g.oids.resize(g.n);
    ok = fread(g.oids.data(), 8, g.n, f) == (size_t) g.n;
  }
  if (ok) {
    g.src.resize(g.m);
    g.dst.resize(g.m);
    ok = fread(g.src.data(), 8, g.m, f) == (size_t) g.m && fread(g.dst.data(), 8, g.m, f) == (size_t) g.m;
  }
  fclose(f);   // weights, if any, are not used by these apps
  return ok;
}

template <template <class> class APP_T, typename... Args>
int Run(const CommSpec& comm_spec, const Graph& g, const std::string& name, int threads, int repeat,
        const std::string& out, Args... args) {
  using FRAG_T = ImmutableEdgecutFragment<int64_t, uint32_t, EmptyType, EmptyType, LoadStrategy::kOnlyOut>;
  auto t0 = std::chrono::steady_clock::now();
  LoadGraphSpec graph_spec = DefaultLoadGraphSpec();
  graph_spec.set_directed(false);
  graph_spec.set_rebalance(false, 0);
  graph_spec.partitioner_type = PartitionerType::kMapPartitioner;   // flags.cc:60-63
  graph_spec.idxer_type = IdxerType::kHashMapIdxer;
  std::shared_ptr<FRAG_T> fragment(nullptr);
  {
    BasicFragmentLoader<FRAG_T> loader(comm_spec, graph_spec);
    EmptyType e;
    for (int64_t i = 0; i < g.n; ++i) loader.AddVertex(g.oids.empty() ? i : g.oids[i], e);
    loader.ConstructVertices();
    for (int64_t i = 0; i < g.m; ++i) loader.AddEdge(g.src[i], g.dst[i], e);
    loader.ConstructFragment(fragment);
  }
  const double load_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  ParallelEngineSpec spec = MultiProcessSpec(comm_spec, false);
  if (threads > 0) spec.thread_num = threads;
  std::vector<double> ms;
  for (int r = 0; r < repeat; ++r) {   // the worker is single-shot: a fresh app + worker per query
    auto app = std::make_shared<APP_T<FRAG_T>>();
    auto worker = APP_T<FRAG_T>::CreateWorker(app, fragment);
    worker->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker->Query(args...);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    if (r + 1 == repeat && !out.empty()) {
      auto ctx = worker->GetContext();
      FILE* f = fopen(out.c_str(), "w");
      if (!f) return 2;
      for (auto v : fragment->InnerVertices())
        fprintf(f, "%lld %d\n", (long long) fragment->GetId(v), (int) ctx->partial_result[v]);
      fclose(f);
    }
    worker->Finalize();
  }
  printf("{\"app\": \"%s\", \"threads\": %u, \"hardware_concurrency\": %u, \"load_s\": %.3f, \"vertices\": %lld, "
         "\"edges\": %lld, \"query_ms\": [",
         name.c_str(), spec.thread_num, std::thread::hardware_concurrency(), load_s, (long long) g.n, (long long) g.m);
  for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
  printf("]}\n");
  fflush(stdout);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string app, graph, rmat, out;
  int k = 0, threads = 0, repeat = 1;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--app") app = v;
    else if (a == "--graph") graph = v;
    else if (a == "--rmat") rmat = v;
    else if (a == "--k") k = atoi(v.c_str());
    else if (a == "--threads") threads = atoi(v.c_str());
    else if (a == "--repeat") repeat = atoi(v.c_str());
    else if (a == "--out") out = v;
    else { fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
  }
  Graph g;
  if (!rmat.empty()) {
    int scale = 0, ef = 16;
    unsigned long long seed = 1;
    if (sscanf(rmat.c_str(), "%d,%d,%llu", &scale, &ef, &seed) < 1 || scale < 1 || scale > 30) {
      fprintf(stderr, "bad --rmat %s\n", rmat.c_str());
      return 2;
    }
    g.n = 1ll << scale;
    g.m = (int64_t) ef << scale;
    g.src.resize(g.m);
    g.dst.resize(g.m);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < g.m; ++i) {
      uint64_t a, b;
      rmatdef::edge((uint64_t) i, scale, seed, &a, &b);
      g.src[i] = (int64_t) a;
      g.dst[i] = (int64_t) b;
    }
  } else if (!read_graph(graph, g)) {
    fprintf(stderr, "cannot read graph %s\n", graph.c_str());
    return 2;
  }
  InitMPIComm();
  int rc = 0;
  {
    CommSpec comm_spec;
    comm_spec.Init(MPI_COMM_WORLD);
    if (app == "core_decomposition") rc = Run<CoreDecomposition>(comm_spec, g, app, threads, repeat, out);
    else if (app == "kcore") rc = Run<KCore, int>(comm_spec, g, app, threads, repeat, out, k);
    else { fprintf(stderr, "unknown app %s\n", app.c_str()); rc = 2; }
  }
  FinalizeMPIComm();
  return rc;
}
