// fragment.h — internal representation of a device-resident edge-cut fragment.
// Replaces grape::cuda::HostFragment / dev::DeviceFragment
// (grape/cuda/fragment/host_fragment.h, device_fragment.h) with an SoA CSR:
// 64-bit row pointers, 32-bit neighbour lids, separate weight array.
#pragma once
#include <utility>
#include <vector>

#include "common.cuh"

namespace gl {

struct DevCsr {
  uint64_t* rp = nullptr;     // [rows+1]
  uint32_t* col = nullptr;    // [entries]
  void* w = nullptr;          // [entries] (edata_bytes wide) or null
  uint64_t* split = nullptr;  // [rows] first outer-neighbour position
  uint64_t rows = 0;
  uint64_t entries = 0;
};

}  // namespace gl

struct gl_frag {
  uint32_t fid = 0, fnum = 1, ivnum = 0, ovnum = 0;
  uint64_t total_vnum = 0;
  int directed = 0, load_strategy = 0, edata_bytes = 0;
  int fid_offset = 31;
  uint32_t id_mask = 0x7fffffffu;
  gl::DevCsr oe, ie, ovie;
  bool ie_alias_oe = true;
  uint32_t* ovgid = nullptr;
  uint32_t* outer_range = nullptr;  // device [fnum+1]
  std::vector<uint32_t> h_outer_range;
  int64_t* inner_oids = nullptr;    // device or null
  std::vector<int64_t> h_inner_oids;   // lid order
  // (oid, lid) sorted by oid when h_inner_oids is not ascending; empty when it is (gl_frag_oid2lid
  // then searches h_inner_oids itself)
  std::vector<std::pair<int64_t, uint32_t>> h_oid_index;
  int64_t oid_base = 0;
  uint64_t part_chunk = 0;  // ceil(n/fnum) of the segmented partitioner (0 = unknown)
  // bitmap of inner vertices with out-degree > 0 (pull candidates)
  uint32_t* nonzero_deg = nullptr;
  // dense sweeps (dense.cuh): first row touching each 4096-entry tile of oe.col
  uint32_t* oe_tile_row = nullptr;
  uint32_t oe_ntiles = 0;
  uint64_t device_bytes = 0;
  uint32_t max_degree = 0, max_degree_lid = 0;
  bool offloaded = false;
  // host shadow used by Offload/ReloadTopology
  std::vector<uint64_t> sh_rp;
  std::vector<uint32_t> sh_col;
  std::vector<uint8_t> sh_w;
};

namespace gl {
void frag_fill_view(const gl_frag* f, gl_frag_view* v);
inline void id_parser_init(uint32_t fnum, int* fid_offset, uint32_t* id_mask) {
  // grape/fragment/id_parser.h:28-41
  uint32_t maxfid = fnum - 1;
  int off;
  if (maxfid == 0) {
    off = 31;
  } else {
    int i = 0;
    while (maxfid) {
      maxfid >>= 1;
      ++i;
    }
    off = 32 - i;
  }
  *fid_offset = off;
  *id_mask = (1u << off) - 1u;
}
}  // namespace gl
