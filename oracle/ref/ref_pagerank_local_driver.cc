// ref_pagerank_local_driver.cc — runs the UNMODIFIED reference CPU app PageRankLocal
// (examples/analytical_apps/pagerank/pagerank_local.h, run_app --application pagerank_local) on an
// in-memory graph.
// TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by pagerank_local.mk next to ref_driver.
//
// Loads the graph as a kOnlyOut fragment (the app's load strategy) through the reference's
// BasicFragmentLoader with the segment partitioner and sorted-array idxer ref_driver uses, undirected
// or directed (--directed), runs PageRankLocal with --pr_d / --mr, times Query(), and has each rank
// write its inner vertices to <out>.<fid>, one "oid value" line each, the value with 17 significant
// digits (the context's Output() prints 16).  Under the MPI shim GL_MPI_NP=N runs N fragments; rank r
// feeds the loader the vertices and edges whose index is r mod N.  Rank 0 prints one JSON line with the
// query times and its fragment's avg_degree, the value that selects the app's branch.
//
// usage: ref_pagerank_local_driver (--graph FILE.bin | --rmat SCALE,EDGEFACTOR,SEED) [--directed 0|1]
//                                  [--pr_d D] [--mr R] [--threads T] [--repeat K] [--out PREFIX]
// graph file: ref_driver's "GRB1" format (oracle/refdriver.py write_graph); --rmat edges as generated.
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
#include "pagerank/pagerank_local.h"

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

int Run(const CommSpec& comm_spec, const Graph& g, bool directed, double pr_d, int mr, int threads, int repeat,
        const std::string& out) {
  using FRAG_T = ImmutableEdgecutFragment<int64_t, uint32_t, EmptyType, EmptyType, LoadStrategy::kOnlyOut>;
  const int64_t me = comm_spec.worker_id(), nw = comm_spec.worker_num();
  auto t0 = std::chrono::steady_clock::now();
  LoadGraphSpec graph_spec = DefaultLoadGraphSpec();
  graph_spec.set_directed(directed);
  graph_spec.set_rebalance(false, 0);
  graph_spec.partitioner_type = PartitionerType::kSegmentedPartitioner;
  graph_spec.idxer_type = IdxerType::kSortedArrayIdxer;
  std::shared_ptr<FRAG_T> fragment(nullptr);
  {
    BasicFragmentLoader<FRAG_T> loader(comm_spec, graph_spec);
    EmptyType e;
    for (int64_t i = me; i < g.n; i += nw) loader.AddVertex(g.oids.empty() ? i : g.oids[i], e);
    loader.ConstructVertices();
    for (int64_t i = me; i < g.m; i += nw) loader.AddEdge(g.src[i], g.dst[i], e);
    loader.ConstructFragment(fragment);
  }
  const double load_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  ParallelEngineSpec spec = MultiProcessSpec(comm_spec, false);
  if (threads > 0) spec.thread_num = threads;
  std::vector<double> ms;
  double avg_degree = 0;
  for (int r = 0; r < repeat; ++r) {   // the worker is single-shot: a fresh app + worker per query
    using APP_T = PageRankLocal<FRAG_T>;
    auto app = std::make_shared<APP_T>();
    auto worker = APP_T::CreateWorker(app, fragment);
    worker->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker->Query(pr_d, mr);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    auto ctx = worker->GetContext();
    avg_degree = ctx->avg_degree;
    if (r + 1 == repeat && !out.empty()) {
      const std::string path = out + "." + std::to_string(comm_spec.fid());
      FILE* f = fopen(path.c_str(), "w");
      if (!f) return 2;
      for (auto v : fragment->InnerVertices())
        fprintf(f, "%lld %.17g\n", (long long) fragment->GetId(v), ctx->result[v]);
      fclose(f);
    }
    worker->Finalize();
  }
  if (me == 0) {
    printf("{\"app\": \"pagerank_local\", \"fnum\": %u, \"directed\": %d, \"threads\": %u, "
           "\"hardware_concurrency\": %u, \"load_s\": %.3f, \"vertices\": %lld, \"edges\": %lld, "
           "\"avg_degree\": %.17g, \"query_ms\": [",
           comm_spec.fnum(), directed ? 1 : 0, spec.thread_num, std::thread::hardware_concurrency(), load_s,
           (long long) g.n, (long long) g.m, avg_degree);
    for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
    printf("]}\n");
    fflush(stdout);
  }
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string graph, rmat, out;
  double pr_d = 0.85;
  int mr = 10, threads = 0, repeat = 1, directed = 0;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--graph") graph = v;
    else if (a == "--rmat") rmat = v;
    else if (a == "--directed") directed = atoi(v.c_str());
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
    rc = Run(comm_spec, g, directed != 0, pr_d, mr, threads, repeat, out);
  }
  FinalizeMPIComm();
  return rc;
}
