// app_lcc.cu — local clustering coefficient by oriented triangle counting.
//
// Semantics of examples/analytical_apps/lcc/lcc.h:48-233 + lcc_context.h:52-66
// (GPU apps: cuda/lcc/lcc_preprocess.h:96-188 + lcc_opt.h:183-316):
//   degree(v) = CSR entries of v's row (multi-edges count);
//   N+(v) = { u in N(v) : deg u < deg v, or deg u == deg v and gid(v) > gid(u) }
//   for every v, every u in N+(v) (with multiplicity), every w in N+(u) (with
//   multiplicity): if w is a member of N+(v) then tri[u], tri[v], tri[w] += 1;
//   lcc(v) = 2*tri / (d*(d-1)), 0 when d < 2.
// Integer counting => bit-exact; the final division is fp64 as in the reference.
//
// Re-design: the degree-ordered DAG is built on the device (the reference
// builds it on the CPU with one std::vector per vertex and ships it through
// MPI, lcc_preprocess.h), then one warp per oriented edge (v,u) intersects
// N+(u) against the sorted N+(v) by binary search; counts use 64-bit atomics.
//
// fnum > 1 (lcc.h:96-140 ships the filtered neighbour lists of every inner
// vertex to the fragments mirroring it, through MPI byte archives): here
//   1. degrees of the outer copies come from the dense mirror sync;
//   2. each fragment builds its part of the DAG with GLOBAL ids (rows sorted
//      by gid) and exports the two arrays through CUDA IPC;
//   3. every fragment replicates its peers' parts with bulk NVLink copies
//      (the whole DAG is 4 B per oriented edge — 1 GB at scale 24);
//   4. a triangle is counted once, by the owner of its highest-ranked vertex;
//      counts that land on outer copies go to their owners as (lid, count)
//      items and are added in the next round (the reference's
//      SyncStateOnOuterVertex + sum, lcc.h:178-196).
#include "dag_common.cuh"

namespace gl {
namespace {

// v -> u is kept when u ranks below v
struct LccKeep {
  GL_DEV bool operator()(const uint32_t*, uint64_t, uint64_t, uint32_t, uint32_t, uint32_t dv, uint32_t du,
                         uint32_t gv, uint32_t gu) const {
    return du < dv || (du == dv && gv > gu);
  }
};

struct LccApp : TriangleApp<false> {
  // PEval: degrees + degree-ordered DAG (lcc.h:48-74 and stage 0, :84-132)
  int PEval() override {
    cudaStream_t s = eng.stream;
    const GidOf gid{fv.ivnum, fv.fid, fv.fid_offset, fv.ovgid};
    // 1. degrees: own rows, then the owners' values for the outer copies
    if (fv.ivnum) GL_LAUNCH(k_row_length<uint32_t>, (fv.ivnum + 255) / 256, 256, s, fv.oe_rp, fv.ivnum, deg.get());
    if (fv.fnum > 1) GL_TRY(mm.SyncValuesToGhosts(s, deg, 4));
    // 2. my part of the DAG, global ids; several fragments: rows sorted by gid (outer gids do not follow
    //    lid order)
    GL_LAUNCH(k_dag_count<LccKeep>, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, LccKeep{}, cnt,
              nullptr);
    GL_TRY(scan_and_resize());
    if (fv.ivnum && om) {
      GL_LAUNCH(k_dag_fill<LccKeep>, eng.sm_count * 8, 256, s, fv.oe_rp, fv.oe_col, deg, gid, fv.ivnum, LccKeep{}, orp,
                okey, olid, osrc);
      if (fv.fnum > 1) GL_TRY(sort_csr_rows(s, orp, fv.ivnum, om, &okey, &olid));
    }
    // 3. replicate the peers' parts (bulk NVLink copies)
    GL_TRY(peers.replicate(mm, s, fv, orp, okey, om));
    mm.ForceContinue();
    return GL_OK;
  }

  int Result(void* host_out, size_t) override { return WriteResult(host_out, deg, 2.0); }
};

}  // namespace

gl_app* make_lcc() { return new LccApp; }

}  // namespace gl
