// ref_bc_driver.cc — runs the UNMODIFIED reference CPU app bc (StagedBCBFS then
// StagedBC on one shared BCContext, examples/analytical_apps/bc/, the
// run_app --application bc choice of run_app.h:280-284) on an in-memory graph.
// TEST / MEASUREMENT INFRASTRUCTURE ONLY; built by bc.mk next to ref_driver.
//
// Loads the graph the way ref_core_driver does (BasicFragmentLoader, one
// fragment, undirected, run_app's map partitioner + hashmap idxer), runs the
// two workers as DoDualQuery does (run_app.h:68-82), times both Query() calls,
// and writes the context's Output() line "oid c sigma depth" at full precision:
// c as %a (the f32 value, exactly), sigma as %.17g.
//
// usage: ref_bc_driver (--graph FILE.bin | --rmat SCALE,EDGEFACTOR,SEED)
//                      [--source OID | --source maxdeg] [--threads T] [--repeat R] [--out FILE]
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
#include "bc/staged_bc.h"
#include "bc/staged_bc_bfs.h"

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

int Run(const CommSpec& comm_spec, const Graph& g, int64_t source, int threads, int repeat, const std::string& out) {
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
  for (int r = 0; r < repeat; ++r) {   // the workers are single-shot: fresh apps + workers per query
    using App1 = StagedBCBFS<FRAG_T>;
    using App2 = StagedBC<FRAG_T>;
    auto app1 = std::make_shared<App1>();
    auto app2 = std::make_shared<App2>();
    auto worker1 = App1::CreateWorker(app1, fragment);
    worker1->Init(comm_spec, spec);
    auto worker2 = std::make_shared<typename App2::worker_t>(app2, fragment, worker1->GetContext());
    worker2->Init(comm_spec, spec);
    MPI_Barrier(comm_spec.comm());
    auto q0 = std::chrono::steady_clock::now();
    worker1->Query(source);
    worker2->Query(source);
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - q0).count());
    if (r + 1 == repeat && !out.empty()) {
      auto ctx = worker1->GetContext();
      FILE* f = fopen(out.c_str(), "w");
      if (!f) return 2;
      for (auto v : fragment->InnerVertices())
        fprintf(f, "%lld %a %.17g %lld\n", (long long) fragment->GetId(v), (double) ctx->centrality_value[v],
                ctx->path_num[v], (long long) ctx->partial_result[v]);
      fclose(f);
    }
    worker1->Finalize();
    worker2->Finalize();
  }
  printf("{\"app\": \"bc\", \"source\": %lld, \"threads\": %u, \"hardware_concurrency\": %u, \"load_s\": %.3f, "
         "\"vertices\": %lld, \"edges\": %lld, \"query_ms\": [",
         (long long) source, spec.thread_num, std::thread::hardware_concurrency(), load_s, (long long) g.n,
         (long long) g.m);
  for (size_t i = 0; i < ms.size(); ++i) printf("%s%.4f", i ? ", " : "", ms[i]);
  printf("]}\n");
  fflush(stdout);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  std::string graph, rmat, out, source = "0";
  int threads = 0, repeat = 1;
  for (int i = 1; i + 1 < argc; i += 2) {
    std::string a = argv[i], v = argv[i + 1];
    if (a == "--graph") graph = v;
    else if (a == "--rmat") rmat = v;
    else if (a == "--source") source = v;
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
  int64_t src_oid = 0;
  if (source == "maxdeg") {
    // degree = CSR entries of the undirected graph (a self loop counts twice), ties -> smallest id
    std::vector<uint32_t> deg((size_t) g.n, 0);
    for (int64_t i = 0; i < g.m; ++i) {
      ++deg[(size_t) g.src[i]];
      ++deg[(size_t) g.dst[i]];
    }
    int64_t best = 0;
    for (int64_t v = 1; v < g.n; ++v)
      if (deg[(size_t) v] > deg[(size_t) best]) best = v;
    src_oid = g.oids.empty() ? best : g.oids[(size_t) best];
  } else {
    src_oid = atoll(source.c_str());
  }
  InitMPIComm();
  int rc = 0;
  {
    CommSpec comm_spec;
    comm_spec.Init(MPI_COMM_WORLD);
    rc = Run(comm_spec, g, src_oid, threads, repeat, out);
  }
  FinalizeMPIComm();
  return rc;
}
