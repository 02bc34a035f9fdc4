/* grape_b200.h — C ABI of the H100-native PIE graph engine.
 *
 * The reference (alibaba/libgrape-lite @ e7c4465) exposes NO C ABI: its GPU
 * path is header-only C++ compiled into each app.  This header is the thin
 * boundary the reference's C++ host would bind instead of grape/cuda/ **:
 * every entry point cites the reference interface it replaces
 * (paths relative to the reference root).  Plain pointers and sizes only.
 *
 * Conventions
 *   - every function returns gl_status (0 = ok, <0 = error);
 *     gl_last_error() returns a thread-local message.  The C++ shim turns a
 *     non-zero status into LOG(FATAL), preserving the reference's
 *     abort-on-error behaviour (grape/cuda/utils/cuda_utils.h:60-108).
 *   - one host thread per device (mirrors one MPI rank per GPU,
 *     examples/analytical_apps/run_cuda_app.h:207-214); handles are not
 *     thread-safe.  The library uses the CUDA *current device* of the caller.
 *   - host pointers passed in descriptors are BORROWED for the call.
 *   - there is no CPU fallback: every call fails with GL_ERR_CUDA when no
 *     CUDA device is usable.
 */
#ifndef GRAPE_B200_H_
#define GRAPE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GL_ABI_VERSION 2

typedef enum {
  GL_OK = 0,
  GL_ERR_CUDA = -1,   /* CUDA runtime error / no device            */
  GL_ERR_ARG = -2,    /* invalid argument                          */
  GL_ERR_NOMEM = -3,  /* host or device allocation failed          */
  GL_ERR_STATE = -4,  /* call not valid in the handle's state      */
  GL_ERR_COMM = -5    /* peer / collective failure                 */
} gl_status;

const char* gl_last_error(void);
int gl_abi_version(void);
/* Device facts used for grid sizing: sm_count, cc major*10+minor, L2 bytes. */
int gl_device_info(int* sm_count, int* cc, size_t* l2_bytes, size_t* hbm_bytes);

/* ------------------------------------------------------------------ *
 * Load balancing of ForEachEdge (grape/cuda/parallel/parallel_engine.h:51,
 * ParseLoadBalancing :53-70; flag --lb, examples/analytical_apps/flags.cc).
 * ------------------------------------------------------------------ */
typedef enum {
  GL_LB_NONE = 0,   /* thread per vertex            (LBNONE   :621-646) */
  GL_LB_CM = 1,     /* CTA-cooperative mapping      (LBCM     :716-771) */
  GL_LB_WM = 2,     /* warp-cooperative mapping     (LBWARP   :773-845) */
  GL_LB_CTA = 3,    /* 3-tier CTA/warp/thread       (LBCTA    :847-879) */
  GL_LB_STRICT = 4, /* exact edge-balanced          (LBSTRICT :881-979) */
  GL_LB_CMOLD = 5   /* alias of CM (LBCMOld :648-714)                   */
} gl_lb;

/* grape::LoadStrategy (grape/types.h) */
typedef enum { GL_LOAD_ONLY_OUT = 0, GL_LOAD_BOTH_OUT_IN = 1 } gl_load_strategy;

/* ------------------------------------------------------------------ *
 * Fragment: replaces grape::cuda::HostFragment / dev::DeviceFragment
 * (grape/cuda/fragment/host_fragment.h:100-120,322-438,
 *  grape/cuda/fragment/device_fragment.h:36-450).
 * Storage is SoA: 64-bit row pointers, 32-bit neighbour lids, separate
 * weight array; rows sorted by neighbour lid, inner neighbours first
 * (grape/graph/immutable_csr.h:104-131).
 * ------------------------------------------------------------------ */
typedef struct gl_frag gl_frag_t;

/* One CSR as the host's ImmutableEdgecutFragment holds it
 * (grape/fragment/csr_edgecut_fragment_base.h: oe_/ie_ + offsets). */
typedef struct {
  const uint64_t* row_ptr; /* rows+1 entries                                 */
  const uint32_t* col;     /* neighbour lid                                  */
  const void* edata;       /* NULL | float[] | double[] (see edata_bytes)    */
  uint64_t rows;           /* number of rows described                       */
} gl_csr_desc;

typedef struct {
  uint32_t fid, fnum;
  int directed;
  int load_strategy;   /* gl_load_strategy                                   */
  uint32_t ivnum;      /* inner vertices: lids [0, ivnum)                     */
  uint32_t ovnum;      /* outer vertices: lids [ivnum, ivnum+ovnum)           */
  uint64_t total_vnum; /* GetTotalVerticesNum()                               */
  int edata_bytes;     /* 0 (EmptyType), 4 (float) or 8 (double)              */
  gl_csr_desc oe;      /* rows = ivnum (inner rows; outer rows are empty)     */
  gl_csr_desc ie;      /* directed: rows = ivnum; undirected: ignored         */
  gl_csr_desc ov_ie;   /* not read: gl_frag_create always derives the reverse
                          adjacency of the OUTER vertices from oe (what the
                          reference keeps in ie_ rows ivnum..tvnum for kOnlyOut
                          undirected, csr_edgecut_fragment_base.h:475-492);
                          gl_frag_copy_csr(which = 2) reads it back           */
  const uint32_t* ovgid;     /* gid of each outer vertex, ascending (IdParser
                                format, grape/fragment/id_parser.h:28-55)     */
  const int64_t* inner_oids; /* oid of each inner vertex in lid order, any
                                order, no oid twice (GL_ERR_ARG); NULL ->
                                oid = oid_base + lid                          */
  int64_t oid_base;
} gl_frag_desc;

/* replaces HostFragment::__allocate_device_fragment__ (host_fragment.h:322-438).
 * Preconditions the library relies on (the reference's loaders satisfy them):
 *  - rows sorted by neighbour lid, inner neighbours first; ovgid ascending;
 *  - a DIRECTED fragment passes its in-edges in d->ie (without them BFS only pushes, PageRank pull
 *    falls back to push and WCC / wcc_opt are refused).
 * Any partition and any lid order are accepted.  Ties follow gid order: CDLP / WCC take the smallest
 * GID as label and LCC orients equal degrees by gid (as the reference's lcc.h does; on repeated edges
 * that decides the count).  The reference's vfile loader puts ascending oid blocks on the fids and
 * assigns lids in oid order, so there the smallest gid is the smallest oid; its efile loader hashes
 * oids to fids (oid % fnum) and assigns lids in order of first appearance, so there it is not.  With
 * fnum > 1 attach a gl_vm_t (gl_app_set_vertex_map) to get WCC / CDLP labels back as oids (without one
 * they are raw gids). */
int gl_frag_create(gl_frag_t** out, const gl_frag_desc* d);
/* HostFragment::PrepareToRunApp (host_fragment.h:122-215): split positions, outer ranges, the
 * reverse adjacency of the outer copies and the destination-fragment information are part of the
 * device layout from gl_frag_create on, so this only validates the request: need_mirror_info needs a
 * communicator with a mirror area at sync time, need_build_device_vm is served by gl_vm_create. */
int gl_frag_prepare(gl_frag_t*, int message_strategy, int need_split_edges, int need_mirror_info);

/* Edge-list front end: replaces LoadGraph -> EVFragmentLoader ->
 * ImmutableEdgecutFragment::Init -> buildCSR -> upload
 * (grape/fragment/loader.h:46-53, immutable_edgecut_fragment.h:215-350,
 * csr_edgecut_fragment_base.h:417-734) with a device-side build (radix sort).
 * Partitioner: contiguous blocks of ceil(n/fnum) ascending oids
 * (grape/vertex_map/partitioner.h:115-126 SegmentedPartitioner); lid = rank
 * of the oid inside the block, so gid order == oid order.
 * Vertices are oids 0..n-1 (oids==NULL) or the given ascending oid list.
 * Every rank passes the edges it holds; edges with no inner endpoint are
 * ignored, edges naming unknown oids are dropped. */
typedef struct {
  uint64_t n_vertices;
  const int64_t* oids;  /* NULL or ascending list of n_vertices oids          */
  uint64_t n_edges;
  const int64_t* src;   /* host pointers                                      */
  const int64_t* dst;
  const void* edata;    /* NULL | float[] | double[]                          */
  int edata_bytes;      /* 0 | 4 | 8 ; device copy keeps this width           */
  int directed;
  int load_strategy;
  uint32_t fid, fnum;
} gl_edges_desc;
int gl_frag_build_from_edges(gl_frag_t** out, const gl_edges_desc* d);

/* Synthetic Graph500 R-MAT fragment built entirely on the device
 * (SURVEY.md §8(d): A,B,C,D = .57,.19,.19,.05; ids scrambled by a fixed
 * bijection; self loops and duplicates kept; undirected).  weight_mode:
 * 0 none, 1 integer-valued 1..255 stored as f32, 2 real (0,1] stored as f32. */
typedef struct {
  int scale;
  int edgefactor;
  uint64_t seed;
  int weight_mode;
  uint32_t fid, fnum;
} gl_rmat_desc;
int gl_frag_build_rmat(gl_frag_t** out, const gl_rmat_desc* d);
/* Host copy of the same generator (inputs for the CPU oracle / reference);
 * w may be NULL. Generates edges [first, first+count). */
int gl_rmat_edges_host(const gl_rmat_desc* d, uint64_t first, uint64_t count,
                       int64_t* src, int64_t* dst, float* w);

typedef struct {
  uint32_t fid, fnum, ivnum, ovnum;
  uint64_t total_vnum;
  uint64_t oe_num, ie_num; /* CSR entries held (GetOutgoingEdgeNum etc.)      */
  int directed, load_strategy, edata_bytes;
  int fid_offset;          /* IdParser::fid_offset_                           */
  uint64_t device_bytes;   /* HBM held by the fragment                        */
  uint32_t max_degree;
} gl_frag_info;
int gl_frag_get_info(const gl_frag_t*, gl_frag_info* out);

/* Device view (POD of device pointers): replaces HostFragment::DeviceObject()
 * (host_fragment.h:277-320).  Invalidated by destroy; while the topology is
 * offloaded oe_col / oe_w (and their ie aliases) are NULL, the id fields stay valid. */
typedef struct {
  uint32_t fid, fnum, ivnum, ovnum;
  uint64_t total_vnum;
  int directed, edata_bytes, fid_offset;
  uint32_t id_mask;
  const uint64_t* oe_rp;    /* [ivnum+1] */
  const uint32_t* oe_col;
  const void* oe_w;
  const uint64_t* oe_split; /* [ivnum] first outer-neighbour position of the row
                               (oespliters_, immutable_edgecut_fragment.h:744-772) */
  const uint64_t* ie_rp;    /* directed: [ivnum+1]; undirected: == oe_rp      */
  const uint32_t* ie_col;
  const void* ie_w;
  const uint64_t* ie_split;
  const uint64_t* ovie_rp;  /* [ovnum+1] reverse adjacency of outer vertices   */
  const uint32_t* ovie_col; /* inner lids                                     */
  const uint32_t* ovgid;    /* [ovnum]                                        */
  const uint32_t* outer_range; /* [fnum+1] outer lids owned by each fid
                                  (outer_vertices_of_frag_)                   */
  const int64_t* inner_oids;   /* may be NULL (oid = oid_base + lid)          */
  int64_t oid_base;
  uint64_t oe_num, ie_num;     /* CSR entries behind oe_col / ie_col          */
} gl_frag_view;
int gl_frag_view_get(const gl_frag_t*, gl_frag_view* out);

/* D2H copies of the stored CSR (layout parity tests; Serialize analogue,
 * grape/graph/immutable_csr.h:307-363).  which: 0 = oe, 1 = ie, 2 = ov_ie.
 * Any of the output pointers may be NULL. w is written with edata_bytes width. */
int gl_frag_copy_csr(const gl_frag_t*, int which, uint64_t* row_ptr,
                     uint32_t* col, void* w);
int gl_frag_copy_ovgid(const gl_frag_t*, uint32_t* ovgid);
/* GetInnerVertex(oid) -> lid (host; host_fragment / fragment_base API).
 * Returns GL_OK and *lid, or GL_ERR_ARG when the oid is not an inner vertex. */
int gl_frag_oid2lid(const gl_frag_t*, int64_t oid, uint32_t* lid);
/* max-out-degree inner vertex (ties -> smallest lid) and its degree */
int gl_frag_max_degree_vertex(const gl_frag_t*, uint32_t* lid, uint64_t* degree);
/* Binary cache of a fragment: ImmutableEdgecutFragment::Serialize / Deserialize
 * (grape/fragment/immutable_edgecut_fragment.h:508-584, immutable_csr.h:307-363;
 * the reference writes <prefix>/frag_<fid>.s).  Header + raw SoA arrays; a load
 * is fread + H2D, nothing is re-sorted. */
int gl_frag_save(const gl_frag_t*, const char* path);
int gl_frag_load(gl_frag_t** out, const char* path);
/* OffloadTopology / ReloadTopology (host_fragment.h:440-468) */
int gl_frag_offload(gl_frag_t*);
int gl_frag_reload(gl_frag_t*);
void gl_frag_destroy(gl_frag_t*);

/* ------------------------------------------------------------------ *
 * Device vertex map (oid <-> gid): replaces grape::cuda::DeviceVertexMap
 * (grape/cuda/vertex_map/device_vertex_map.h:94-172; built when an app sets
 * need_build_device_vm, host_fragment.h:205-215).  One device array of oids
 * per group (fragment f at off[f]) + binary search instead of the reference's
 * chained hash maps.  oids[f] = host array of fragment f's inner oids in lid
 * order (VertexMap::GetOid(fid, lid)).
 * ------------------------------------------------------------------ */
typedef struct gl_vm gl_vm_t;
typedef struct {
  uint32_t fnum;
  int fid_offset;
  uint32_t id_mask;
  const int64_t* l2o;          /* device [off[fnum]]: oid of (f, lid) at off[f] + lid   */
  const uint64_t* off;         /* device [fnum+1]                                        */
  const int64_t* sorted_oid;   /* device, NULL when every slice of l2o is ascending      */
  const uint32_t* sorted_lid;  /* device, lid of sorted_oid[i]                           */
} gl_vm_view;
int gl_vm_create(gl_vm_t** out, uint32_t fnum, const uint64_t* ivnums, const int64_t* const* oids);
int gl_vm_view_get(const gl_vm_t*, gl_vm_view* out);          /* DeviceObject()          */
/* batch lookups on device arrays: dev::DeviceVertexMap::GetGid / GetOid (:36-80);
 * unknown oid -> gid 0xFFFFFFFF, invalid gid -> oid -1 */
int gl_vm_oid2gid(const gl_vm_t*, void* stream, const int64_t* d_oids, uint64_t n, uint32_t* d_gids);
int gl_vm_gid2oid(const gl_vm_t*, void* stream, const uint32_t* d_gids, uint64_t n, int64_t* d_oids);
void gl_vm_destroy(gl_vm_t*);

/* ------------------------------------------------------------------ *
 * Fragment group communicator: replaces GPUMessageManager's NCCL/MPI
 * bootstrap (grape/cuda/parallel/gpu_message_manager.h:160-194) and
 * cuda::Communicator (grape/cuda/communication/communicator.h:41-95).
 * The data plane is NVLink peer memory: each rank exports its landing
 * buffers as CUDA IPC handles (gl_comm_export), the launcher exchanges the
 * 64-byte handles (any out-of-band channel: torch.distributed, a file) and
 * every rank maps its peers (gl_comm_open).  Scalar collectives and the
 * per-superstep barrier go through a caller-supplied callback so the
 * library needs no MPI/NCCL link dependency.
 * ------------------------------------------------------------------ */
typedef struct gl_comm gl_comm_t;
/* sum/min/max all-reduce of n int64 / double values in place (host memory). */
typedef int (*gl_allreduce_fn)(void* user, void* inout, int n, int is_double,
                               int op /*0 sum,1 min,2 max*/);
typedef struct {
  uint32_t fid, fnum;
  gl_allreduce_fn allreduce; /* required when fnum > 1 */
  void* user;
  size_t landing_bytes;      /* per-peer landing buffer capacity (bytes)      */
  size_t mirror_bytes;       /* per-peer capacity of the dense mirror-sync area
                                (inner state -> outer copies, the reference's
                                BatchShuffleMessageManager::SyncInnerVertices,
                                grape/cuda/parallel/batch_shuffle_message_manager.h:142-220);
                                0 = 8 bytes per inner vertex of the largest fragment
                                is NOT assumed: pass it explicitly.
                                GL_APP_PAGERANK_VC on F > 1 vertex-cut fragments
                                needs mirror_bytes >= 8 * ceil(n_vertices / F)
                                (gl_comm_create rounds it up to a multiple of 256) */
} gl_comm_desc;
#define GL_IPC_HANDLE_BYTES 64
int gl_comm_create(gl_comm_t** out, const gl_comm_desc* d);
/* writes fnum_slots*GL_IPC_HANDLE_BYTES bytes: handle of this rank's landing
 * area (one allocation, sliced per source rank) + control block */
int gl_comm_export(gl_comm_t*, void* handles_out, size_t bytes);
/* all_handles: fnum consecutive exports, ordered by fid */
int gl_comm_open(gl_comm_t*, const void* all_handles, size_t bytes);
/* Unmaps the peers' landing areas (keeps the local one).  Teardown order for a
 * group: every rank closes its peers, the group meets in a barrier, then each
 * rank destroys its communicator -- nobody frees memory a peer still maps. */
int gl_comm_close_peers(gl_comm_t*);
void gl_comm_destroy(gl_comm_t*);
/* Diagnostic: average time (us) of one kernel that stores `bytes` from local
 * memory into the next peer's (all_peers = 0) or every peer's (1) mirror slot
 * with 16-byte (vec16 = 1) or 4-byte stores, followed by a fence.sys per CTA.
 * Sizes the multi-GPU design decisions in DESIGN.md section 5. */
int gl_comm_peer_write_us(gl_comm_t*, size_t bytes, int vec16, int all_peers, int reps, double* us_out);

/* ------------------------------------------------------------------ *
 * Message manager (SURVEY 8b, Face 2): the halo exchange that the shimmed
 * grape::cuda::GPUMessageManager / dev::MessageManager sit on
 * (grape/cuda/parallel/gpu_message_manager.h:45-458,
 *  grape/cuda/serialization/in_archive.h:36-169, out_archive.h:32-178,
 *  grape/cuda/parallel/message_kernels.h:28-127).
 * A producer kernel appends bytes for fragment d at
 *   send_slot[d] + atomicAdd(&send_bytes[d], sizeof(item))
 * -- send_slot[d] is fragment d's landing slot for this rank, mapped over
 * NVLink / CUDA IPC: the store IS the transfer (no staging archive, no NCCL
 * send/recv, no host size exchange).  gl_mm_finish_round publishes the byte
 * counts, runs the device-side barrier + termination vote and flips the
 * double buffer; what was sent in round r is readable through recv_slot /
 * recv_bytes during round r+1 only (the reference's rule: messages are
 * visible in the next IncEval); round 0 after gl_mm_start receives nothing.
 * Termination = no fragment sent a byte and
 * none called force_continue (gpu_message_manager.h:413-430).
 * ------------------------------------------------------------------ */
typedef struct gl_mm gl_mm_t;
typedef struct {
  uint32_t fid, fnum;
  int fid_offset;            /* gid = fid << fid_offset | lid (IdParser)        */
  uint32_t id_mask;
  uint32_t capacity_bytes;   /* per landing slot                               */
  char* const* send_slot;    /* device table [fnum]: my slot at fragment d     */
  uint32_t* send_bytes;      /* device [fnum]: bytes appended this round       */
  const char* const* recv_slot;   /* device table [fnum]: what fragment s sent me last round */
  const uint32_t* recv_bytes;     /* device [fnum]                              */
} gl_mm_view;
/* GPUMessageManager::Init (:160-194) on an OPENED communicator; fnum == 1: comm may be NULL */
int gl_mm_create(gl_mm_t** out, gl_comm_t* comm);
/* InitBuffer (:196-204): checks the per-peer capacities against the communicator's landing slots */
int gl_mm_init_buffer(gl_mm_t*, size_t send_bytes_per_peer, size_t recv_bytes_per_peer);
int gl_mm_start(gl_mm_t*);                         /* Start (:219) + round counter reset */
int gl_mm_start_round(gl_mm_t*, void* stream);     /* StartARound (:225-231)             */
int gl_mm_finish_round(gl_mm_t*, void* stream);    /* FinishARound (:237-303) + syncLengths (:400-431); synchronises the stream */
int gl_mm_to_terminate(gl_mm_t*, int* out);        /* ToTerminate (:321)                 */
int gl_mm_force_continue(gl_mm_t*);                /* ForceContinue (:338)               */
int gl_mm_view_get(gl_mm_t*, gl_mm_view* out);     /* DeviceObject (:342-344): valid for the current round */
uint64_t gl_mm_bytes_sent(gl_mm_t*);               /* GetMsgSize, accumulated over the query */
void gl_mm_destroy(gl_mm_t*);

/* Fixed-function consumers of ParallelProcess (:362-393): the received bytes
 * are (uint32 gid, value) pairs -- thrust::pair<vid_t, MESSAGE_T> -- or bare
 * uint32 gids (GL_MSG_SET_BIT); lid = gid & id_mask. */
typedef enum {
  GL_MSG_SET_BIT = 0,   /* bare gid: out_bitmap |= bit(lid)                     */
  GL_MSG_MIN_U32 = 1,   /* if (v < atomicMin(state[lid], v)) out_bitmap |= bit   */
  GL_MSG_MIN_F32 = 2,
  GL_MSG_MIN_F64 = 3,
  GL_MSG_ADD_F32 = 4,   /* atomicAdd(state[lid], v)                              */
  GL_MSG_ADD_F64 = 5
} gl_msg_op_kind;
typedef struct {
  int kind;               /* gl_msg_op_kind                                     */
  void* state;            /* device array indexed by lid                        */
  uint32_t* out_bitmap;   /* may be NULL                                        */
} gl_msg_op;
int gl_mm_process(gl_mm_t*, void* stream, const gl_msg_op* op, uint64_t* items_host /* may be NULL */);

/* Fixed-function producer: the "ForEach over outer vertices +
 * SyncStateOnOuterVertex[WarpOpt]" idiom (e.g. cuda/sssp/sssp.h:295-304).  For
 * every set bit v of `remote` inside the fragment's outer range, appends
 * (gid(v)[, state[v]]) to the owner's landing slot (value_bytes: 0 = bare gid,
 * 4 or 8 = thrust::pair<vid_t, value> layout) and clears the bit when
 * clear_bits != 0. */
int gl_mm_send_outer(gl_mm_t*, void* stream, const gl_frag_t* frag, uint32_t* remote_bitmap,
                     const void* state, int value_bytes, int clear_bits);

/* Dense mirror sync: owner state -> the outer copies other fragments hold
 * (BatchShuffleMessageManager::SyncInnerVertices,
 * grape/cuda/parallel/batch_shuffle_message_manager.h:142-220; mirror lists =
 * edgecut_fragment_base.h:569-603).  The communicator must have been created
 * with mirror_bytes >= 8 * (largest inner vertex count of the group).
 * gl_mm_mirror_plan is collective and runs once per (mm, fragment); every
 * sync is collective: owners pack their mirrored values straight into the
 * holders' mirror slots (peer stores), a device-side barrier follows, holders
 * copy the slots into their outer range.  values: device array over ALL local
 * vertices (inner then outer), elem_bytes 4 or 8; bitmap: one bit per local
 * vertex (ghost bits |= owner bits). */
int gl_mm_mirror_plan(gl_mm_t*, void* stream, const gl_frag_t* frag);
int gl_mm_sync_values_to_ghosts(gl_mm_t*, void* stream, void* values, int elem_bytes);
int gl_mm_sync_bits_to_ghosts(gl_mm_t*, void* stream, uint32_t* bitmap);

/* cuda::Communicator::Sum/Min/Max on one host scalar
 * (grape/cuda/communication/communicator.h:41-84,160-172): device-side peer
 * all-reduce, bit-identical on every rank (fixed fid order).
 * dtype: 0 int64, 1 double; op: 0 sum, 1 min, 2 max.  Synchronises `stream`.
 * The result is the left fold in fid order (sum: ((v0 + v1) + v2) ...); min / max
 * keep the running value only when it compares strictly less / greater, so of
 * values that compare equal (-0.0 and +0.0) the one of the highest fid wins. */
int gl_allreduce(gl_mm_t*, void* stream, void* inout_host, int dtype, int op);

/* ------------------------------------------------------------------ *
 * PIE apps (PEval / IncEval / Output): replaces GPUWorker::{Init,Query}
 * (grape/cuda/worker/gpu_worker.h:44-107) running the six GPU apps of
 * examples/analytical_apps/cuda/{bfs,sssp,wcc,pagerank,cdlp,lcc}.
 * ------------------------------------------------------------------ */
typedef enum {
  GL_APP_BFS = 0,      /* cuda/bfs/bfs.h        result: int64 depth            */
  GL_APP_SSSP = 1,     /* cuda/sssp/sssp.h      result: double (f32/f64 math)  */
  GL_APP_WCC = 2,      /* cuda/wcc/wcc.h        result: int64 oid of min-gid   */
  GL_APP_PAGERANK = 3, /* cuda/pagerank/pagerank.h result: double; on a directed
                          fragment it follows pagerank_parallel.h (a vertex without
                          out-edges keeps base each round); the Graphalytics
                          directed PageRank is GL_APP_PAGERANK_DIRECTED         */
  GL_APP_CDLP = 4,     /* cuda/cdlp/cdlp.h      result: int64 label            */
  GL_APP_LCC = 5,      /* cuda/lcc/lcc_opt.h    result: double                 */
  GL_APP_WCC_OPT = 6,  /* cuda/wcc/wcc_opt.h (union-find) result: as GL_APP_WCC  */
  /* undirected fragments only (GL_ERR_ARG otherwise); degree = CSR entries
   * (a multi-edge counts once per copy, a self loop twice) */
  GL_APP_CORE_DECOMPOSITION = 7, /* core_decomposition/core_decomposition.h
                                    result: int64 core number (isolated: 0)     */
  GL_APP_KCORE = 8,    /* kcore/kcore.h  result: int64 entries whose other
                          endpoint survives the k-core peel (k = max_round);
                          v is in the k-core iff value >= k                   */
  GL_APP_KCLIQUE = 9,  /* kclique/kclique.h (--kclique_k = max_round), see below */
  GL_APP_BC = 10,      /* bc/staged_bc_bfs.h + bc/staged_bc.h (--bc_source =
                          source_oid)  result: gl_bc_value, see below          */
  GL_APP_LCC_DIRECTED = 11,  /* lcc/lcc_directed.h (LCCDirected)  result: double,
                                see below                                        */
  GL_APP_PAGERANK_VC = 12,  /* pagerank/pagerank_vc.h (PageRankVC, run_app --vc) on a
                               gl_vcfrag_t: created by gl_vc_app_create only;
                               result: double per master vertex, see below      */
  GL_APP_CDLP_DIRECTED = 13, /* cuda/cdlp/cdlp.h on kBothOutIn (--directed)
                               result: int64 label, see below                   */
  GL_APP_PAGERANK_DIRECTED = 14, /* pagerank/pagerank_directed.h (PageRankDirected,
                                   run_app_opt --application pagerank --directed)
                                   result: double, see below                    */
  GL_APP_BC_SOURCES = 15, /* bc (--bc_source) summed over a list of sources set by
                             gl_app_set_sources  result: double, see below      */
  GL_APP_PAGERANK_LOCAL = 16 /* pagerank/pagerank_local.h (PageRankLocal, run_app
                                --application pagerank_local): un-normalised
                                PageRank  result: double, see below             */
} gl_app_kind;

/* ------------------------------------------------------------------ *
 * Vertex-cut fragment: replaces ImmutableVertexcutFragment with the 2-D
 * VCPartitioner (grape/fragment/immutable_vertexcut_fragment.h,
 * grape/vertex_map/partitioner.h).  Vertices are the oids 0..n-1, F = fnum
 * must be a perfect square, s = sqrt(F):
 *   mvc = ceil(n / F), vchunk = mvc * s;
 *   edge (a, b) belongs to fragment (a / vchunk) * s + b / vchunk;
 *   the masters of fragment f are [f * mvc, min((f + 1) * mvc, n)) (tail
 *   fragments may have none);
 *   the source range of f is chunk f / s, the destination range chunk f % s
 *   (chunk c = [c * vchunk, min((c + 1) * vchunk, n))); the masters lie in the
 *   source range.  The local vertices are the union of the two ranges, lower
 *   chunk first, each in oid order (one range on a diagonal block).
 * The device holds a local CSR over the local vertices: every block edge
 * (a, b) puts b in a's row and a in b's row (a self loop twice in its row,
 * duplicates kept), 64-bit row pointers, 32-bit local column ids, rows sorted.
 * ------------------------------------------------------------------ */
typedef struct gl_vcfrag gl_vcfrag_t;
typedef struct {
  uint64_t n_vertices;
  uint64_t n_edges;
  const int64_t* src;  /* host pointers; any superset of this fid's block (e.g.
                          the whole edge list): edges of other blocks are ignored */
  const int64_t* dst;
  uint32_t fid, fnum;
} gl_vcfrag_desc;
/* GL_ERR_ARG: fnum not a perfect square, fid >= fnum, an endpoint of ANY edge
 * outside [0, n), or 2^32 or more local vertices. */
int gl_vcfrag_create(gl_vcfrag_t** out, const gl_vcfrag_desc* d);
/* The device R-MAT generator of gl_frag_build_rmat (ids in [0, 2^scale)); every
 * generated edge is used once, as generated (the app treats each edge both ways).
 * weight_mode is ignored. */
int gl_vcfrag_build_rmat(gl_vcfrag_t** out, const gl_rmat_desc* d);
typedef struct {
  uint32_t fid, fnum;
  uint64_t n_vertices;
  uint64_t master_begin, master_end;  /* oids [begin, end)                            */
  uint64_t src_begin, src_end;        /* source range (chunk fid / s)                  */
  uint64_t dst_begin, dst_end;        /* destination range (chunk fid % s)             */
  uint64_t local_vnum;                /* |source range U destination range|            */
  uint64_t block_edges;               /* edges of this fragment's block                 */
  uint64_t entries;                   /* local CSR entries = 2 * block_edges            */
  uint64_t device_bytes;              /* HBM held by the fragment                      */
} gl_vcfrag_info;
int gl_vcfrag_get_info(const gl_vcfrag_t*, gl_vcfrag_info* out);
void gl_vcfrag_destroy(gl_vcfrag_t*);

/* GL_APP_PAGERANK_VC: PageRankVC on a vertex-cut fragment.  Uses pr_delta (d) and max_round (R);
 * every other gl_app_config field is ignored.  gl_app_create refuses kind 12 and gl_vc_app_create
 * every other kind (GL_ERR_ARG); gl_app_set_vertex_map is refused (GL_ERR_ARG).  The result is one
 * double per master vertex in oid order (gl_app_result_oids gives the master oids).  With F > 1 the
 * app needs an opened communicator with mirror_bytes >= 8 * mvc (GL_ERR_ARG otherwise); F = 1 does
 * no communication and comm may be NULL.
 * Semantics (n vertices, deg(v) = edge endpoints equal to v: a self loop counts twice, every duplicate
 * counts; v is dangling when deg(v) = 0; D = dangling vertices of the whole graph):
 *   R <= 0: nothing runs, every result is 0.0, supersteps = 1.
 *   PEval: p = 1/n; mr[v] = p if v is dangling, else p / deg(v); dangling_sum = p * D; curr = mr
 *          on every local copy.
 *   IncEval step k = 1..R: base = (1 - d)/n + d * dangling_sum / n, then dangling_sum = base * D;
 *          next[v] = sum of curr[u] over the local CSR entries (v, u); sum(v) = the partial next[v]
 *          of every fragment holding v, folded in fid order; k < R: mr[v] = (base + d * sum) / deg(v)
 *          (base when dangling) and curr = mr on every copy; k = R: result[v] = sum * d + base.
 *   Everything is f64 and every sum has a fixed order (a row's entries in fixed per-lane strides and
 *   shuffle tree, long rows in fixed 4096-entry chunks folded in order), so the same input gives
 *   bit-identical output on every run.  It equals GL_APP_PAGERANK (push or pull, same d and R) on
 *   the undirected edge-cut fragment of the same edges up to f64 summation order.
 * Stats: supersteps = R + 1; step k = round k (1..R), mode 2, step_frontier = local vertices,
 *   step_entries = local CSR entries (2 x block edges, a host count); touched_vertices = masters x R.
 *   msg_bytes_sent (F > 1) = (R + 1) x G + R x S where G = 8 |masters(g)| summed over the other
 *   fragments g whose masters lie in this fragment's local range (the gather of PEval's degrees and
 *   of every round's sums) and S = 8 |own masters| x (the other fragments holding them) (the scatter
 *   of PEval and of rounds 1..R-1).  R <= 0: 0. */

/* GL_APP_LCC_DIRECTED: the local clustering coefficient of a directed graph (the reference's
 * run_app_opt --application lcc --directed), one double per inner vertex in lid order.  It needs a
 * directed fragment with its in-edges (gl_frag_desc.ie / kBothOutIn): an undirected fragment (use
 * GL_APP_LCC there) and a directed one without ie are refused at gl_app_create with GL_ERR_ARG.  Edge
 * data is ignored.  For an inner vertex v, over its out-row and in-row together, oe(v) + ie(v), with
 * multiplicity:
 *   N(v) = the distinct neighbours in the union (v itself when v has a self loop);
 *   d(v) = |N(v)|, the deduplicated degree;
 *   w(v,u) = the CSR entries of u in oe(v) + ie(v) = #(v->u) + #(u->v) (symmetric);
 *   tri(v) = the sum of w(u,x) over unordered pairs {u, x} of N(v) \ {v}, u != x, u and x adjacent;
 *   lcc(v) = double(tri(v)) / double(int64(d) * (d - 1)); 0.0 when d < 2.
 * Each triangle is counted once along a degree orientation (|oe| + |ie| entries); the reference breaks
 * degree ties by IdHasher(gid), this app by gid.  Every weight is symmetric, so any strict total order
 * gives the same tri.  Two deliberate differences from the reference:
 *   - weights are exact: the reference keeps w in a uint8_t, so a pair joined by 256 entries weighs 0
 *     there (and 300 entries weigh 44); here w is exact below 2^32 entries per pair;
 *   - tri is counted in 64 bits: the reference's LCCDirected32, which it picks for graphs of at most
 *     2^32 edges, can wrap on hubs.
 * Where every pair has fewer than 256 entries and the counts fit 32 bits, the result equals the
 * reference's bit for bit. */

/* GL_APP_CDLP_DIRECTED: label propagation over the in- and out-neighbours of a directed graph (the
 * reference's run_cuda_app --application cdlp --directed, the LDBC Graphalytics directed CDLP), one
 * int64 label per inner vertex in lid order, as for GL_APP_CDLP: labels are kept as gids and mapped
 * to oids on output, and gl_app_set_vertex_map works the same way.  It needs a directed fragment with
 * its in-edges (gl_frag_desc.ie / kBothOutIn): an undirected fragment (use GL_APP_CDLP there) and a
 * directed one without ie are refused at gl_app_create with GL_ERR_ARG.  Uses max_round only; every
 * other gl_app_config field is ignored; edge data is ignored.
 *   Labels start as the vertex's own id; each of max_round rounds updates all vertices at once.
 *   The candidates of inner vertex v are the labels of ie(v) plus the labels of oe(v), with
 *   multiplicity: a reciprocal pair u <-> v counts twice, a self loop twice (once in oe, once in ie),
 *   every repeated edge once per copy.
 *   The new label is the label with the highest count; ties go to the smallest label.
 *   A vertex with |ie(v)| + |oe(v)| = 0 keeps its label; one with only in-edges updates (GL_APP_CDLP
 *   keeps the label of a vertex without out-edges).  max_round = 0 returns the identity labelling.
 * Ties are broken on the smallest gid, as GL_APP_CDLP does: under the segment partitioner that is the
 * reference's smallest-oid rule; on hash or map partitions gid order is not oid order (see DESIGN.md).
 * Directed CDLP on edge list E equals GL_APP_CDLP on the undirected fragment built from E, whose row
 * of u is oe(u) + ie(u) as a multiset.  GL_APP_CDLP on a directed fragment is unchanged (out-edges
 * only). */

/* GL_APP_PAGERANK_DIRECTED: the directed PageRank of LDBC Graphalytics (the reference's PageRankDirected,
 * run_app_opt --application pagerank --directed), one double per inner vertex in lid order.  It needs a
 * directed fragment with its in-edges (gl_frag_desc.ie / kBothOutIn): an undirected fragment (use
 * GL_APP_PAGERANK there) and a directed one without ie are refused at gl_app_create with GL_ERR_ARG.
 * Uses pr_delta (d) and max_round (R); every other gl_app_config field, pr_pull included, is ignored;
 * edge data is ignored.  N = vertices of the whole group; deg(v) = the entries of v's out-row
 * (duplicates count, a self loop counts once); v is dangling when deg(v) = 0; D = the dangling vertices
 * of the group.
 *   R <= 0: nothing runs; every result is 0.0 (the reference's zero-initialised result); supersteps = 1.
 *   PEval: p = 1/N; x[v] = p / deg(v), or p when v is dangling; S = p * D.
 *   Round k = 1..R: base = (1 - d)/N + d * S/N;
 *          c(v) = d * (sum of x[w] over the entries w of ie(v)) + base;
 *          x[v] = c(v) when v is dangling, else c(v) / deg(v);
 *          k < R: S = the sum of c(v) over the dangling vertices of the group.
 *   Output: x[v] * deg(v) for a non-dangling v (the reference's multiply-back, (c / deg) * deg, not c);
 *          x[v] for a dangling v.
 * A vertex without out-edges keeps what arrives over its in-edges, and the mass the dangling vertices
 * hold is spread evenly over every vertex in the next round, so for R >= 1 the results of the group
 * sum to 1 up to rounding.  GL_APP_PAGERANK on a directed fragment does not have this property: it
 * resets such a vertex to base every round.
 * Everything is f64, and every sum has a fixed order: an in-row in the row tiers of GL_APP_PAGERANK_VC
 * (a thread up to 32 entries, a warp up to 4096, longer rows in 4096-entry chunks folded in order), S
 * from per-CTA partials folded in CTA order and, on several fragments, in fid order.  The same input
 * on the same fragments gives bit-identical output on every run.
 * Stats: supersteps = R + 1; step k = round k (1..R), mode 2, step_frontier = ivnum, step_entries = the
 *   fragment's ie entries (a host count); touched_vertices = ivnum x R.  msg_bytes_sent (F > 1) =
 *   R x 8 M + (R - 1) x 8 (F - 1), where M = the outer copies of this fragment's inner vertices held
 *   by the other fragments (the dense mirror sync of x after PEval and after rounds 1..R-1) and 8 (F - 1)
 *   is the value S this fragment sends to its peers in each all-reduce after rounds 1..R-1.
 *   R <= 0: 0. */

/* GL_APP_PAGERANK_LOCAL: the original, un-normalised PageRank (the reference's PageRankLocal, run_app
 * --application pagerank_local), one double per inner vertex in lid order.  The ranks sum to about N
 * rather than 1, and no dangling mass is redistributed.  Undirected and directed fragments are both
 * accepted; on a directed one the sum runs over the out-row (the reference's kOnlyOut), so ie is not
 * needed.  Uses pr_delta (d) and max_round (R); every other gl_app_config field, pr_pull included, is
 * ignored; edge data is ignored.  deg(v) = the entries of v's out-row (a multi-edge counts once per
 * copy, a self loop as often as the fragment stores it: twice on an undirected fragment, once on a
 * directed one).
 *   R <= 0 is refused at gl_app_create with GL_ERR_ARG (the reference never terminates there).
 *   PEval: x(v) = 1 / deg(v), or 1 when deg(v) = 0.
 *   Round k = 1..R: c(v) = (1 - d) + d * (sum of x(u) over the entries u of v's out-row);
 *          k < R: x(v) = c(v) / deg(v), or c(v) when deg(v) = 0.
 *   Output: c(v) of round R (not divided).
 * On an undirected fragment with no zero-degree vertex the result equals N x GL_APP_PAGERANK (same d and
 * R) in real arithmetic; with zero-degree vertices the two are not related by a scale factor.  The
 * reference's single-fragment run on a graph whose average out-row length exceeds 10 never divides by
 * the degree after PEval (its values grow every round); this app follows the definition above on any
 * number of fragments.
 * Everything is f64, and every sum has a fixed order: an out-row in the row tiers of GL_APP_PAGERANK_VC
 * (a thread up to 32 entries, a warp up to 4096, longer rows in 4096-entry chunks folded in order).  The
 * same input on the same fragments gives bit-identical output on every run.
 * Stats: supersteps = R + 1; step k = round k (1..R), mode 2, step_frontier = ivnum, step_entries = the
 *   fragment's oe entries (a host count), so entries_scanned = R x oe entries; touched_vertices = ivnum
 *   x R.  msg_bytes_sent (F > 1) = R x 8 M, where M = the outer copies of this fragment's inner vertices
 *   held by the other fragments (the dense mirror sync of x after PEval and after rounds 1..R-1);
 *   0 on one fragment. */

/* GL_APP_BC: single-source betweenness centrality, one gl_bc_value per inner vertex in lid order: the
 * reference's Output() line `oid c sigma depth` (gl_app_result_oids gives the oid).  A directed fragment
 * is refused at gl_app_create with GL_ERR_ARG; edge data is ignored.
 *   depth: BFS level from the source; INT64_MAX for an unreached vertex (sigma = c = 0 there, and
 *          everywhere when source_oid is not in the graph).
 *   path_num (sigma): sigma(source) = 1; a depth-1 vertex has sigma = 1 however many parallel edges join
 *          it to the source; a vertex at depth d >= 2 has the sum of sigma(u) over the CSR entries (v, u)
 *          of its row with depth(u) = d - 1 (one term per copy of a parallel edge).  f64.
 *   centrality (c): an f32 value, widened exactly.  For d = L (the deepest level) down to 0, every vertex
 *          v at depth d takes cacc = f32(sum of double(t[u]) over the entries (v, u) of its row with
 *          depth(u) = d + 1); for d > 0 c = f32(double(cacc) * sigma(v)) and
 *          t[v] = f32((1.0 / sigma(v)) * (1.0 + double(c))); the source keeps c = cacc.
 * Every sum is a gather over the vertex's own row in a fixed order (a short row sequentially, a long
 * one in fixed 1024-entry chunks with fixed lane strides and shuffle tree, the chunk sums in order):
 * the same graph gives bit-identical output on every run.  depth and sigma equal the reference's
 * bit for bit while every sigma is below 2^53; c differs from it only by f32 summation error (the
 * reference keeps a running f32 sum over atomics in thread order; this app rounds one f64 sum).
 * Stats, one fragment: supersteps = forward levels + backward levels (2 (L + 1)); step i <= L is
 * forward level i (step_frontier = level size, step_mode 0 push / 1 pull discovery), step L + 1 + j
 * is backward level L - j (step_frontier = level size, step_mode 2); frontier_vertices = reached
 * vertices.  Several fragments: one worker round per forward and per backward level, step_frontier
 * is this fragment's share of the level. */
typedef struct {
  double centrality;
  double path_num;
  int64_t depth;
} gl_bc_value;

/* GL_APP_BC_SOURCES: betweenness centrality summed over a list of sources: exact Brandes BC when the
 * list is every vertex, the sampled approximation when it is a sample.  One double per inner vertex in
 * lid order (gl_app_result_oids gives the oids).  A directed fragment is refused at gl_app_create with
 * GL_ERR_ARG, as for GL_APP_BC; edge data is ignored.  The list is set by gl_app_set_sources (below)
 * and a query before the first gl_app_set_sources returns GL_ERR_ARG.  reserved[0] is the batch width
 * B, 1..32 (0: the largest that fits, at most 32; GL_ERR_ARG outside 0..32); with reserved[0] = 0,
 * reserved[1] > 0 is a test hook that stands in for the batch width free HBM allows (GL_ERR_ARG when
 * negative); every other config field is ignored.  The graph is GL_APP_BC's CSR: a multi-edge once per copy, a self loop twice.  For each entry
 * s of the list, in list order:
 *   depth_s and sigma_s follow GL_APP_BC's rules exactly (a depth-1 vertex has sigma 1 however many
 *   parallel edges join it to s);
 *   backward, from the deepest level up: cacc = the sum of t_s(w) over the entries (v, w) of v's row
 *   with depth_s(w) = depth_s(v) + 1, in row order; delta_s(v) = cacc * sigma_s(v);
 *   t_s(v) = (1.0 / sigma_s(v)) * (1.0 + delta_s(v)); all f64.  delta_s(v) = 0 when v = s, when v is
 *   unreached and when s is not in the graph.
 *   bc(v) = (((0.0 + delta_s1(v)) + delta_s2(v)) + ...), a left fold in list order.
 * No normalisation: over every vertex of an undirected graph, bc is twice networkx's
 * betweenness_centrality(G, normalized=False) (each pair is counted from both ends); for a sample of k
 * of n sources the caller scales by n / k.  f32(delta_s(v)) agrees with GL_APP_BC's c (source s, v != s)
 * within 1e-5 relative; GL_APP_BC rounds c and t to f32 at every level, this app does not.
 * Sources run in batches of B, one warp lane per source, with every per-vertex state B lanes wide
 * (20 B bytes per vertex); a row's sum is sequential up to 1024 entries, and a longer row is cut into
 * 1024-entry chunks whose sums are added in chunk order.  One fragment therefore gives bit-identical
 * output on every run and for every B.  gl_app_create returns GL_ERR_NOMEM only when B = 1 does not fit.
 * On several fragments B is decided once for the group: the smallest width any rank's free HBM and
 * mirror area allow, so every rank cuts the list into the same batches.
 * Stats, one fragment: supersteps = batches; step i = batch i, mode 2, step_frontier = the vertices its
 * sources reach (each source included; saturated at UINT32_MAX, which B sources reaching more than
 * 2^32 / B vertices each can pass), step_entries = row entries read by its gathers;
 * frontier_vertices = that sum over the whole list; touched_vertices = frontier_vertices minus the
 * list entries found in the graph; entries_scanned = row entries read by the gathers (a device count).
 * Several fragments: every rank passes the same list (checked by an all-reduce of its length and hash:
 * GL_ERR_ARG otherwise); the row order is the fragment's own, so results agree with one fragment up to
 * f64 summation order, and are bit-identical for every B within one grouping.  One worker round per
 * forward level of each batch (the last one finds nothing) and one per backward level >= 1;
 * step_frontier = this fragment's share (saturated at UINT32_MAX) of the (vertex, source) pairs of
 * the level the round finds or processes; frontier_vertices and touched_vertices are this fragment's shares of the one-fragment
 * values.  B is clamped to what the communicator's mirror_bytes holds for the B-wide rows of the
 * outer copies; gl_app_create returns GL_ERR_ARG when B = 1 does not fit. */

/* GL_APP_KCLIQUE: k = max_round, 3 <= k <= GL_KCLIQUE_MAX_K; a smaller or larger k and a directed
 * fragment are refused at gl_app_create with GL_ERR_ARG.  The result is ONE int64 (gl_app_result takes
 * bytes >= 8): the number of k-cliques of the whole fragment group, the same value on every rank.
 * Counting is on the simple graph underneath the fragments: self loops are ignored, a pair joined by
 * several CSR entries is one edge, a k-clique is a set of k distinct pairwise adjacent vertices.  On a
 * simple graph this is the sum of the reference's per-fragment clique_num at any fragment count.  On a
 * multigraph it deliberately differs: the reference weights a clique by the multiplicities of some of
 * its edges, in an order that depends on the fragment count.  The count is accumulated in uint64 and
 * wraps modulo 2^64 (the reference's size_t); the int64 holds those bits.  One fragment holds at most
 * 2^32 - 1 oriented edges (edges from one of its vertices to a higher-ranked one).
 * Stats: supersteps = worker rounds (1); entries_scanned = DAG entries iterated by the intersections;
 * frontier_vertices = oriented edges of this fragment; step_frontier[0] = the largest candidate set
 * |N+(u) ∩ N+(v)| of an oriented edge (u, v) of this fragment; step_frontier[1..3] = edges counted by
 * the warp tier (candidate set <= 32), the CTA bitmap tier (<= 1024) and the CTA list tier (> 1024),
 * for k >= 4 (0 for k = 3, which sums the candidate set sizes).
 * GL_KCLIQUE_MAX_K: the depth-first walks keep a stack of max(k - 4, 1) levels of one candidate
 * bitmap pair per warp in shared memory next to the 128 KB bitmap matrix; at k = 32 a CTA uses
 * 188 KB of the 227 KB a Hopper CTA can opt into.
 * Several fragments: a fragment with 2^32 or more oriented edges makes every rank's query return
 * GL_ERR_ARG. */
#define GL_KCLIQUE_MAX_K 32

typedef struct {
  int lb;                /* gl_lb (AppConfig::lb, cuda/app_config.h:22-27)     */
  int64_t source_oid;    /* --bfs_source / --sssp_source / --bc_source          */
  double pr_delta;       /* --pr_d                                              */
  int max_round;         /* --pr_mr / --cdlp_mr; GL_APP_KCORE: k (--kcore_k)   */
  int sssp_f64;          /* 1: fp64 distances on device (real-weight 1e-6 run)  */
  double sssp_prio;      /* 0 -> reference heuristic 32*avg_w/avg_deg           */
  int direction_opt;     /* BFS: 0 push only, 1 push/pull (bfs.h:168-261)       */
  int pr_pull;           /* PageRank: 0 push (atomicAdd), 1 pull (deterministic)*/
  int fuse_supersteps;   /* BFS: 1 = the whole query is ONE cooperative kernel per
                            GPU (levels, direction switches and, on several
                            fragments, the NVLink collectives happen inside it);
                            0 = one superstep per host round                    */
  int reserved[8];       /* tuning / test hooks, 0 = default:
                            [0] 1: WCC dense rounds as pull sweeps
                                GL_APP_BC_SOURCES: the batch width B, 1..32
                            [1] GL_APP_BC_SOURCES: the batch width free HBM is taken to allow
                            [1] 1: BFS without the hub-first shadow CSR; 2: with it also on a
                                   small graph (default: from 2^16 vertices on); 3: like 2, several
                                   fragments, without the delegated-hub lists (A/B)
                            [2] BFS pull->push threshold divisor (default 24)
                            [3] >=4: number of BFS level bitmaps (forces spills)
                            [4] 1: PageRank f32 pull without the shared-memory hub table (A/B)
                            [5] 1: PageRank pull gathers f32 contributions
                            [7] 1: fused multi-fragment BFS ships per-holder bit-compressed
                                   frontier slices (round-1 scheme) instead of replicating
                                   the global frontier bitmap
                            [6] 1: BFS result as an int64 device array + one D2H
                                   (default: u8 depths over PCIe, widened on the host) */
} gl_app_config;
void gl_app_config_default(gl_app_config*);

typedef struct gl_app gl_app_t;
/* GPUWorker::Init: PrepareToRunApp + context Init (gpu_worker.h:44-65) */
int gl_app_create(gl_app_t** out, int kind, gl_frag_t* frag, gl_comm_t* comm,
                  const gl_app_config* cfg);
/* Apps on a vertex-cut fragment (GL_APP_PAGERANK_VC only, see above); the handle is used with
 * gl_app_query / gl_app_result / gl_app_result_oids / gl_app_destroy like any other app. */
int gl_vc_app_create(gl_app_t** out, int kind, gl_vcfrag_t* frag, gl_comm_t* comm,
                     const gl_app_config* cfg);

/* Query statistics.  A superstep is one worker round; step 0 is PEval.  The k-th set of counters an
 * app records (k = 0, 1, ...) is reported as step k + 1, also when PEval itself recorded it (CDLP's
 * first round); a step nothing was recorded for reports zeros.  n_steps = min(supersteps,
 * GL_MAX_STEP_STATS): only the per-step arrays are cut there; supersteps, entries_scanned,
 * frontier_vertices and touched_vertices always cover the whole query, so the totals equal the sums
 * of the step arrays whenever supersteps <= GL_MAX_STEP_STATS.  Exceptions, stated below: the
 * one-fragment peels (n_steps = 1, totals only) and wcc_opt (step 0).  tests/test_gpu_stats.py holds
 * the lines below on one fragment; on 2 and 3 fragments it holds the "several fragments" sentences.
 *   BFS, fused or stepwise, any vertex order: step i >= 1 expands level i - 1; step_frontier =
 *     the level's size, supersteps = levels + 1 (the last expansion finds nothing), frontier_vertices
 *     = reached vertices, touched_vertices = vertices given a depth by an expansion (one fragment:
 *     every reached vertex but the source).  A push step's step_entries is the row lengths of its
 *     level, exactly.  A pull step (mode 1) reads rows of vertices not yet reached, in an order that
 *     decides how far each row is read: at least one entry per vertex it finds, at most one probe of
 *     the highest-degree neighbour plus the whole row per unreached vertex with a non-empty row.  A
 *     source that is not in the graph: every counter 0 (supersteps 1 fused, 2 stepwise: the stepwise
 *     query expands the empty frontier once).  A fused query keeps one record per level
 *     for the first GL_MAX_STEP_STATS - 1 levels.
 *     Several fragments, push steps: step_frontier and step_entries are this fragment's share (the
 *     level's vertices it owns and their rows), so they add up to the one-fragment values over the
 *     group; supersteps is the same on every rank, and one more than on one fragment (a closing step
 *     of zeros) when the last level re-reported outer copies that were already visited; a push-only stepwise query sends 4 bytes per outer
 *     vertex with an entry in the row of a reached inner vertex (a fragment learns that an outer vertex
 *     is visited only by reaching it itself).  A pull step's step_frontier is not a share: the fused
 *     query reports what the fragment found itself in the previous level, the stepwise query the whole
 *     graph's level.  touched_vertices also counts the outer copies a fragment reaches.
 *   PageRank (every variant), CDLP: each round is one step with step_frontier = ivnum, step_entries
 *     = the CSR entries of the fragment, mode 2; touched_vertices = ivnum x rounds.  supersteps =
 *     max_round + 2 (PageRank: PEval, the rounds, the round that stops) and max_round + 1 (CDLP: round
 *     1 runs in PEval).  Several fragments: the same with this fragment's ivnum and entries.  CDLP's
 *     step_entries is the size of the CSR its gather and sort are launched over, recorded by the host,
 *     not counted by a kernel.
 *   CDLP_DIRECTED: as CDLP, with step_entries = the ie entries plus the oe entries of the fragment's
 *     inner rows (both gathers and sorts); supersteps = max_round + 1, touched_vertices = ivnum x rounds.
 *   PAGERANK_DIRECTED: see GL_APP_PAGERANK_DIRECTED above; PAGERANK_LOCAL: see GL_APP_PAGERANK_LOCAL.
 *   LCC, one fragment: step 1 counts the triangles: step_frontier = ivnum, step_entries = for every
 *     entry (v, u) of the degree-ordered DAG, the length of u's DAG row; supersteps = 3.
 *   LCC_DIRECTED: step 1 counts the triangles (mode 2): step_frontier = ivnum, step_entries = for every
 *     oriented entry (v, u), the length of u's oriented row N+(u); supersteps = 3; entries_scanned and
 *     frontier_vertices carry the same values, touched_vertices = ivnum.  Several fragments: the same
 *     with this fragment's ivnum and the oriented entries of its inner vertices, so the shares add up to
 *     the one-fragment values over the group.
 *   core decomposition / k-core, one fragment: the whole peel is PEval's launch; supersteps counts its
 *     sub-rounds while n_steps stays 1, so the counters are in the totals only: entries_scanned = the rows of the peeled
 *     vertices (core decomposition: every entry), frontier_vertices = vertices peeled by a scan (k-core:
 *     those with a result below k), touched_vertices = count updates (merged per warp, so it depends on
 *     scheduling).
 *   SSSP, WCC (label propagation): a vertex is expanded again whenever its value improves, in an
 *     order threads race for, so the counts are bounded, not fixed: every reached vertex is expanded
 *     at least once and, unless it keeps its initial value, written at least once.  SSSP's step 1 is
 *     the source alone; WCC's step 1 expands every vertex; a dense WCC round (reserved[0] = 1, mode 2)
 *     reports step_frontier = ivnum and the fragment's entries.
 *   wcc_opt, one fragment: everything happens in PEval and is reported as step 0: step_frontier =
 *     ivnum, step_entries = entries_scanned = 2 sampled entries per vertex + the rows scanned outside
 *     the largest sampled component (which depends on the sampling's races); touched_vertices = ivnum.
 *   BC, k-clique: see gl_bc_value and GL_KCLIQUE_MAX_K above; BC_SOURCES: see GL_APP_BC_SOURCES. */
#define GL_MAX_STEP_STATS 512
typedef struct {
  int supersteps;            /* rounds executed (PEval counts as round 0)      */
  double query_ms;           /* device time of the whole Query()               */
  uint64_t entries_scanned;  /* CSR entries read by edge-scan kernels          */
  uint64_t frontier_vertices;/* sum over supersteps                            */
  uint64_t touched_vertices; /* distinct-destination updates (state writes)    */
  uint64_t kernel_launches;  /* kernels launched inside Query()                */
  uint64_t msg_bytes_sent;   /* halo bytes written to peers                    */
  int n_steps;               /* valid entries in the per-step arrays           */
  float step_ms[GL_MAX_STEP_STATS];
  uint64_t step_entries[GL_MAX_STEP_STATS];
  uint32_t step_frontier[GL_MAX_STEP_STATS];
  uint8_t step_mode[GL_MAX_STEP_STATS]; /* 0 push, 1 pull, 2 dense            */
} gl_query_stats;

/* GPUWorker::Query: PEval then IncEval until every fragment is idle
 * (gpu_worker.h:69-107). Asynchronous work is finished when it returns.
 * Collective on a fragment group: every rank calls it for the same query.  With
 * an opened communicator the call first meets the other ranks in a device-side
 * barrier on the app's stream (the MPI_Barrier in front of the reference's timed
 * Query(), run_cuda_app.h:117); query_ms starts after it.
 * step_frontier[] of a several-fragment fused BFS is THIS fragment's share of
 * each level's frontier. */
int gl_app_query(gl_app_t*, gl_query_stats* stats /* may be NULL */);
/* Context::Output values for the inner vertices, in lid order, to HOST memory
 * (e.g. cuda/sssp/sssp.h:104-118).  elem: see gl_app_kind. */
int gl_app_result(gl_app_t*, void* host_out, size_t bytes);
/* WCC / CDLP keep labels as gids; with a vertex map attached, gl_app_result
 * returns them as oids for ANY partition (without one: only for this library's
 * contiguous-block builders, where gid -> oid is arithmetic or the fragment's
 * own oid list).  The map is borrowed: keep it alive while the app is used. */
int gl_app_set_vertex_map(gl_app_t*, const gl_vm_t* vm);
/* GL_APP_BC_SOURCES only (any other kind: GL_ERR_ARG): copies the source list, which stays in force for
 * later queries until it is set again.  oids == NULL with n == 0: every vertex of the fragment group, in
 * gid order; a non-NULL list with n == 0 is the empty list (every result 0.0).  Duplicates count once
 * per occurrence; an oid that is not a vertex contributes nothing.  Collective on a fragment group. */
int gl_app_set_sources(gl_app_t*, const int64_t* oids, uint64_t n);
/* oid of each inner vertex (first column of Output) */
int gl_app_result_oids(gl_app_t*, int64_t* host_out, size_t count);
void gl_app_destroy(gl_app_t*);

/* ------------------------------------------------------------------ *
 * Engine primitives: fixed-function fast paths of ParallelEngine
 * (grape/cuda/parallel/parallel_engine.h:72-293,987-1013) and the frontier
 * containers of grape/cuda/utils/{bitset,vertex_set,queue}.h.
 * Pointers below are DEVICE pointers owned by the caller.
 * ------------------------------------------------------------------ */
typedef enum {
  GL_OP_BFS_LEVEL = 0,    /* if level[v]==INF: level[v]=depth; out.insert(v)  */
  GL_OP_MIN_RELAX_U32 = 1,/* atomicMin(state[v], state[u] (+w)); the sum saturates
                             at 0xFFFFFFFF (unreached), so an unreached source
                             never relaxes anything                           */
  GL_OP_MIN_RELAX_F32 = 2,/* as U32 on non-negative floats; unreached = FLT_MAX */
  GL_OP_ADD_SCATTER_F64 = 3,/* atomicAdd(state2[v], state[u])                 */
  GL_OP_COUNT = 4         /* counts scanned entries only (bandwidth probe)    */
} gl_edge_op_kind;

typedef struct {
  int kind;               /* gl_edge_op_kind                                   */
  void* state;            /* per-vertex state array (u32 / f32 / f64)          */
  void* state2;           /* ADD_SCATTER: destination array                    */
  uint32_t* out_bitmap;   /* updated vertices (atomicOr), may be NULL          */
  uint32_t depth;         /* BFS_LEVEL: level to write                         */
  int use_weight;         /* MIN_RELAX_*: 1 = add the edge's f32 weight (a
                             fragment without edge data adds 0); a fragment with
                             f64 edge data is refused with GL_ERR_ARG           */
} gl_edge_op;

/* ForEachOutgoingEdge(stream, frag, WorkSourceArray(queue,n), op, lb)
 * (parallel_engine.h:987-1013).  queue: device array of n lids, in any order;
 * an entry that repeats is scanned once per copy.  Directed fragments scan oe. */
int gl_edge_scan_queue(const gl_frag_t*, void* stream, const uint32_t* queue,
                       uint32_t n, const gl_edge_op* op, int lb,
                       uint64_t* entries_scanned_host /* may be NULL */);
/* bitmap (n_bits) -> queue of set bit positions; returns count on the host.
 * Replaces the O(V) ForEach + AppendWarp idiom (cuda/sssp/sssp.h:223-232). */
int gl_compact_bitmap(void* stream, const uint32_t* bitmap, uint32_t n_bits,
                      uint32_t* queue_out, uint32_t* count_host);

/* Frontier containers (grape/cuda/utils/bitset.h:32-196, vertex_set.h:30-163):
 * a DenseVertexSet is a device bitmap of ceil(nbits/32) words; VertexArray is
 * a plain device array (gl_dev_alloc + gl_dev_h2d / gl_dev_d2h); Queue = the
 * (queue_out, count) pair gl_compact_bitmap fills. */
int gl_bitmap_create(uint32_t** out, uint64_t nbits);               /* zeroed */
int gl_bitmap_clear(void* stream, uint32_t* bitmap, uint64_t nbits);  /* Clear(stream) */
int gl_bitmap_count(void* stream, const uint32_t* bitmap, uint64_t nbits, uint64_t* count_host); /* Count(stream): syncs */
int gl_bitmap_destroy(uint32_t* bitmap);

/* Queue<T> (grape/cuda/utils/queue.h:30-140): a device array of vertex ids + its length on the device. */
typedef struct gl_queue gl_queue_t;
int gl_queue_create(gl_queue_t** out, uint32_t capacity);
int gl_queue_clear(gl_queue_t*, void* stream);                          /* Clear(stream)            */
int gl_queue_size(gl_queue_t*, void* stream, uint32_t* size_host);      /* size(stream): syncs      */
int gl_queue_data(gl_queue_t*, uint32_t** data_dev, uint32_t** count_dev);  /* DeviceObject()       */
/* bitmap -> queue without the host round trip of gl_compact_bitmap (count stays on the device) */
int gl_queue_fill_from_bitmap(gl_queue_t*, void* stream, const uint32_t* bitmap, uint32_t n_bits);
void gl_queue_destroy(gl_queue_t*);
/* VertexArray<T> (grape/cuda/utils/vertex_array.h:34-169): device array + H2D / D2H */
int gl_varray_create(void** out, uint64_t count, int elem_bytes, int fill_byte);
int gl_varray_h2d(void* varray, const void* host, uint64_t count, int elem_bytes);
int gl_varray_d2h(const void* varray, void* host, uint64_t count, int elem_bytes);
int gl_varray_destroy(void* varray);

/* device scratch helpers so a C/ctypes caller can run the primitives */
int gl_dev_alloc(void** out, size_t bytes);
int gl_dev_free(void* p);
int gl_dev_memset(void* p, int byte, size_t bytes);
int gl_dev_h2d(void* dst, const void* src, size_t bytes);
int gl_dev_d2h(void* dst, const void* src, size_t bytes);
int gl_dev_sync(void);
/* page-locked host memory for result/ingest buffers (cudaMallocHost) */
int gl_host_alloc_pinned(void** out, size_t bytes);
int gl_host_free_pinned(void* p);
/* kernels launched by this library on the calling thread so far */
uint64_t gl_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* GRAPE_B200_H_ */
