// ref_kclique_driver.cc — runs the UNMODIFIED reference CPU app kclique
// (examples/analytical_apps/kclique/, run_app --application kclique --kclique_k K)
// on an in-memory graph.  TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by
// kclique.mk next to ref_core_driver.
//
// Loads the graph the way ref_core_driver does (BasicFragmentLoader, one
// fragment, undirected, run_app's map partitioner + hashmap idxer), times
// worker->Query(k) and prints the context's clique_num (what its Output()
// writes) in the JSON line.  --simple 1 first maps every edge to (min, max),
// drops self loops and duplicates: the reference's count is a clique count on
// a simple graph only.
//
// usage: ref_kclique_driver (--graph FILE.bin | --rmat SCALE,EDGEFACTOR,SEED)
//                           --k K [--simple 0|1] [--threads T] [--repeat R]
// graph file: ref_driver's "GRB1" format (oracle/refdriver.py write_graph).
#include <unistd.h>

#include <algorithm>
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
#include "kclique/kclique.h"

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
  fclose(f);   // weights, if any, are not used by this app
  return ok;
}

// (min, max) per edge, self loops and repeated pairs removed
void simplify(Graph& g) {
  std::vector<std::pair<int64_t, int64_t>> e;
  e.reserve(g.m);
  for (int64_t i = 0; i < g.m; ++i)
    if (g.src[i] != g.dst[i]) e.emplace_back(std::min(g.src[i], g.dst[i]), std::max(g.src[i], g.dst[i]));
  std::sort(e.begin(), e.end());
  e.erase(std::unique(e.begin(), e.end()), e.end());
  g.m = (int64_t) e.size();
  g.src.resize(g.m);
  g.dst.resize(g.m);
  for (int64_t i = 0; i < g.m; ++i) {
    g.src[i] = e[i].first;
    g.dst[i] = e[i].second;
  }
}

int Run(const CommSpec& comm_spec, const Graph& g, int k, int threads, int repeat) {
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
  size_t clique_num = 0;
  for (int r = 0; r < repeat; ++r) {   // the worker is single-shot: a fresh app + worker per query
    auto app = std::make_shared<KClique<FRAG_T>>();
    auto worker = KClique<FRAG_T>::CreateWorker(app, fragment);
    worker->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker->Query(k);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    clique_num = worker->GetContext()->clique_num;
    worker->Finalize();
  }
  printf("{\"app\": \"kclique\", \"k\": %d, \"clique_num\": %llu, \"threads\": %u, \"hardware_concurrency\": %u, "
         "\"load_s\": %.3f, \"vertices\": %lld, \"edges\": %lld, \"query_ms\": [",
         k, (unsigned long long) clique_num, spec.thread_num, std::thread::hardware_concurrency(), load_s,
         (long long) g.n, (long long) g.m);
  for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
  printf("]}\n");
  fflush(stdout);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string graph, rmat;
  int k = 0, threads = 0, repeat = 1, simple = 0;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--graph") graph = v;
    else if (a == "--rmat") rmat = v;
    else if (a == "--k") k = atoi(v.c_str());
    else if (a == "--simple") simple = atoi(v.c_str());
    else if (a == "--threads") threads = atoi(v.c_str());
    else if (a == "--repeat") repeat = atoi(v.c_str());
    else { fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
  }
  if (k < 3) {   // the app indexes past its per-level vectors for k < 3
    fprintf(stderr, "--k must be >= 3\n");
    return 2;
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
  if (simple) simplify(g);
  InitMPIComm();
  int rc = 0;
  {
    CommSpec comm_spec;
    comm_spec.Init(MPI_COMM_WORLD);
    rc = Run(comm_spec, g, k, threads, repeat);
  }
  FinalizeMPIComm();
  return rc;
}
