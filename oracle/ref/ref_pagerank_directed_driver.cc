// ref_pagerank_directed_driver.cc — runs the UNMODIFIED reference CPU app PageRankDirected
// (examples/analytical_apps/pagerank/pagerank_directed.h, the run_app_opt --application pagerank
// --directed choice of run_app_opt.h:371-382) on an in-memory graph.
// TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by pagerank_directed.mk next to ref_driver.
//
// Loads the graph as one kBothOutIn fragment through the reference's BasicFragmentLoader, with the
// segment partitioner and sorted-array idxer ref_driver --opt 1 uses (run_app_opt picks hash + pthash for
// this app; on one fragment that changes only the lid order, i.e. the f64 summation order), runs
// PageRankDirected with --pr_d / --mr, times Query(), and writes the context's Output() text
// ("oid value" per inner vertex).
//
// usage: ref_pagerank_directed_driver (--graph FILE.bin | --rmat SCALE,EDGEFACTOR,SEED)
//                                     [--pr_d D] [--mr R] [--threads T] [--repeat K] [--out FILE]
// graph file: ref_driver's "GRB1" format (oracle/refdriver.py write_graph); --rmat edges are directed.
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <grape/grape.h>
#include <grape/fragment/basic_fragment_loader.h>
#include <grape/fragment/immutable_edgecut_fragment.h>

#include "../rmat_gen.h"
#include "pagerank/pagerank_directed.h"

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

int Run(const CommSpec& comm_spec, const Graph& g, double pr_d, int mr, int threads, int repeat,
        const std::string& out) {
  using FRAG_T = ImmutableEdgecutFragment<int64_t, uint32_t, EmptyType, EmptyType, LoadStrategy::kBothOutIn>;
  auto t0 = std::chrono::steady_clock::now();
  LoadGraphSpec graph_spec = DefaultLoadGraphSpec();
  graph_spec.set_directed(true);
  graph_spec.set_rebalance(false, 0);
  graph_spec.partitioner_type = PartitionerType::kSegmentedPartitioner;
  graph_spec.idxer_type = IdxerType::kSortedArrayIdxer;
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
    using APP_T = PageRankDirected<FRAG_T>;
    auto app = std::make_shared<APP_T>();
    auto worker = APP_T::CreateWorker(app, fragment);
    worker->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker->Query(pr_d, mr);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    if (r + 1 == repeat && !out.empty()) {
      std::ofstream os(out);
      worker->Output(os);
    }
    worker->Finalize();
  }
  printf("{\"app\": \"pagerank_directed\", \"threads\": %u, \"hardware_concurrency\": %u, \"load_s\": %.3f, "
         "\"vertices\": %lld, \"edges\": %lld, \"query_ms\": [",
         spec.thread_num, std::thread::hardware_concurrency(), load_s, (long long) g.n, (long long) g.m);
  for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
  printf("]}\n");
  fflush(stdout);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string graph, rmat, out;
  double pr_d = 0.85;
  int mr = 10, threads = 0, repeat = 1;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--graph") graph = v;
    else if (a == "--rmat") rmat = v;
    else if (a == "--pr_d") pr_d = atof(v.c_str());
    else if (a == "--mr") mr = atoi(v.c_str());
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
    rc = Run(comm_spec, g, pr_d, mr, threads, repeat, out);
  }
  FinalizeMPIComm();
  return rc;
}
