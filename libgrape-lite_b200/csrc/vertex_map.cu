// vertex_map.cu — device vertex map (oid <-> gid) and the fragment's on-disk
// form (SURVEY 8f rows 1 and 3).
//
// gl_vm_*: replaces grape::cuda::DeviceVertexMap / dev::DeviceVertexMap
// (grape/cuda/vertex_map/device_vertex_map.h:33-172).  The reference keeps, per
// fragment, an lid -> oid array and a chained hash map oid -> lid
// (thirdparty/cuda_hashmap).  Here every fragment's oids live in ONE device
// array (l2o, fragment f at off[f]); oid -> lid is a binary search: over the l2o
// slice itself when it is ascending (this repo's builder and the reference's
// loaders both assign lids in ascending oid order,
// grape/fragment/basic_fragment_loader.h:95-105), else over a sorted (oid, lid)
// copy.  No pointer-chasing hash chains, 8 B per vertex instead of ~24 B.
//
// gl_frag_save / gl_frag_load: the fragment's binary cache — the role of
// ImmutableEdgecutFragment::Serialize / Deserialize
// (grape/fragment/immutable_edgecut_fragment.h:508-584,
//  grape/graph/immutable_csr.h:307-363): header + raw SoA arrays, so a reload is
// fread + H2D without rebuilding (sorting) anything.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdio>
#include <memory>
#include <vector>

#include "apps_common.cuh"

struct gl_vm {
  uint32_t fnum = 1;
  int fid_offset = 31;
  uint32_t id_mask = 0x7fffffffu;
  std::vector<uint64_t> off;   // [fnum+1]
  gl::DevBuf<int64_t> d_l2o;    // [off[fnum]]
  gl::DevBuf<uint64_t> d_off;   // [fnum+1]
  gl::DevBuf<int64_t> d_sorted_oid;   // null when every slice of l2o is ascending
  gl::DevBuf<uint32_t> d_sorted_lid;
};

namespace gl {
namespace {
__global__ void k_vm_check_sorted(const int64_t* l2o, const uint64_t* off, uint32_t fnum, uint32_t* bad) {
  const uint64_t total = off[fnum];
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i + 1 < total; i += (uint64_t) gridDim.x * blockDim.x) {
    // slice boundaries: i+1 starts a new fragment
    uint32_t f = 0;
    while (f + 1 < fnum && i + 1 >= off[f + 1]) ++f;
    if (i + 1 == off[f]) continue;
    if (l2o[i] >= l2o[i + 1]) *bad = 1;
  }
}
__global__ void k_vm_iota(uint32_t* lid, const uint64_t* off, uint32_t fnum) {
  const uint64_t total = off[fnum];
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t) gridDim.x * blockDim.x) {
    uint32_t f = 0;
    while (f + 1 < fnum && i >= off[f + 1]) ++f;
    lid[i] = (uint32_t) (i - off[f]);
  }
}
GL_DEV bool vm_find(const gl_vm_view& v, uint32_t f, int64_t oid, uint32_t* lid) {
  const int64_t* keys = (v.sorted_oid ? v.sorted_oid : v.l2o) + v.off[f];
  uint64_t lo = 0, hi = v.off[f + 1] - v.off[f];
  const uint64_t n = hi;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (keys[mid] < oid) lo = mid + 1; else hi = mid;
  }
  if (lo >= n || keys[lo] != oid) return false;
  *lid = v.sorted_lid ? v.sorted_lid[v.off[f] + lo] : (uint32_t) lo;
  return true;
}
__global__ void k_vm_oid2gid(gl_vm_view v, const int64_t* oids, uint64_t n, uint32_t* gids) {
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
    uint32_t g = 0xFFFFFFFFu, lid;
    for (uint32_t f = 0; f < v.fnum; ++f)
      if (vm_find(v, f, oids[i], &lid)) {
        g = (f << v.fid_offset) | lid;
        break;
      }
    gids[i] = g;
  }
}
__global__ void k_vm_gid2oid(gl_vm_view v, const uint32_t* gids, uint64_t n, int64_t* oids) {
  for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
    const uint32_t g = gids[i], f = g >> v.fid_offset, l = g & v.id_mask;
    oids[i] = (f < v.fnum && l < v.off[f + 1] - v.off[f]) ? v.l2o[v.off[f] + l] : -1;
  }
}
}  // namespace
}  // namespace gl

using namespace gl;

extern "C" {

int gl_vm_create(gl_vm_t** out, uint32_t fnum, const uint64_t* ivnums, const int64_t* const* oids) {
  GL_ARG(out && ivnums && oids && fnum >= 1 && fnum <= GL_MAX_FNUM, "bad argument");
  DeviceInfo* di;
  GL_TRY(device_info(&di));
  std::unique_ptr<gl_vm> vm(new gl_vm);
  vm->fnum = fnum;
  id_parser_init(fnum, &vm->fid_offset, &vm->id_mask);
  vm->off.assign(fnum + 1, 0);
  for (uint32_t f = 0; f < fnum; ++f) vm->off[f + 1] = vm->off[f] + ivnums[f];
  const uint64_t total = vm->off[fnum];
  if (vm->d_l2o.alloc(std::max<uint64_t>(total, 1)) != cudaSuccess || vm->d_off.alloc(fnum + 1) != cudaSuccess) {
    set_error("gl_vm_create: device allocation failed");
    return GL_ERR_NOMEM;
  }
  GL_CUDA(cudaMemcpy(vm->d_off, vm->off.data(), sizeof(uint64_t) * (fnum + 1), cudaMemcpyHostToDevice));
  for (uint32_t f = 0; f < fnum; ++f) {
    if (!ivnums[f]) continue;
    if (!oids[f]) {
      set_error("gl_vm_create: oid list of fragment %u is null", f);
      return GL_ERR_ARG;
    }
    if (cudaMemcpy(vm->d_l2o + vm->off[f], oids[f], sizeof(int64_t) * ivnums[f], cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("gl_vm_create: upload failed");
      return GL_ERR_CUDA;
    }
  }
  // ascending slices need no side index
  uint32_t bad = 0;
  {
    DevBuf<uint32_t> d_bad;
    if (d_bad.alloc(1) != cudaSuccess) return GL_ERR_NOMEM;
    GL_CUDA(cudaMemset(d_bad, 0, 4));
    if (total > 1) {
      k_vm_check_sorted<<<num_sms() * 4, 256>>>(vm->d_l2o, vm->d_off, fnum, d_bad);
      GL_COUNT_LAUNCH();
    }
    GL_CUDA(cudaMemcpy(&bad, d_bad, 4, cudaMemcpyDeviceToHost));
  }
  if (bad) {
    // per-slice sort of (oid, lid): one segmented radix sort
    const int64_t* k_in = vm->d_l2o;
    DevBuf<uint32_t> v_in;
    if (vm->d_sorted_oid.alloc(total) != cudaSuccess || vm->d_sorted_lid.alloc(total) != cudaSuccess ||
        v_in.alloc(total) != cudaSuccess) {
      set_error("gl_vm_create: device allocation failed");
      return GL_ERR_NOMEM;
    }
    k_vm_iota<<<num_sms() * 4, 256>>>(v_in, vm->d_off, fnum);
    GL_COUNT_LAUNCH();
    size_t tb = 0;
    cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tb, k_in, vm->d_sorted_oid.get(), v_in.get(), vm->d_sorted_lid.get(),
                                             (int) total, (int) fnum, vm->d_off.get(), vm->d_off + 1);
    DevBuf<char> tmp;
    GL_CUDA(tmp.alloc(std::max<size_t>(tb, 16)));
    cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(tmp, tb, k_in, vm->d_sorted_oid.get(), v_in.get(),
                                                             vm->d_sorted_lid.get(), (int) total, (int) fnum,
                                                             vm->d_off.get(), vm->d_off + 1);
    cudaDeviceSynchronize();
    if (e != cudaSuccess) {
      set_error("gl_vm_create: segmented sort failed: %s", cudaGetErrorString(e));
      return GL_ERR_CUDA;
    }
  }
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("gl_vm_create: %s", cudaGetErrorString(cudaGetLastError()));
    return GL_ERR_CUDA;
  }
  *out = vm.release();
  return GL_OK;
}

int gl_vm_view_get(const gl_vm_t* vm, gl_vm_view* out) {
  GL_ARG(vm && out, "null argument");
  out->fnum = vm->fnum;
  out->fid_offset = vm->fid_offset;
  out->id_mask = vm->id_mask;
  out->l2o = vm->d_l2o;
  out->off = vm->d_off;
  out->sorted_oid = vm->d_sorted_oid;
  out->sorted_lid = vm->d_sorted_lid;
  return GL_OK;
}

int gl_vm_oid2gid(const gl_vm_t* vm, void* stream, const int64_t* d_oids, uint64_t n, uint32_t* d_gids) {
  GL_ARG(vm && (n == 0 || (d_oids && d_gids)), "null argument");
  if (!n) return GL_OK;
  gl_vm_view v;
  GL_TRY(gl_vm_view_get(vm, &v));
  GL_LAUNCH(k_vm_oid2gid, num_sms() * 4, 256, (cudaStream_t) stream, v, d_oids, n, d_gids);
  return GL_OK;
}

int gl_vm_gid2oid(const gl_vm_t* vm, void* stream, const uint32_t* d_gids, uint64_t n, int64_t* d_oids) {
  GL_ARG(vm && (n == 0 || (d_oids && d_gids)), "null argument");
  if (!n) return GL_OK;
  gl_vm_view v;
  GL_TRY(gl_vm_view_get(vm, &v));
  GL_LAUNCH(k_vm_gid2oid, num_sms() * 4, 256, (cudaStream_t) stream, v, d_gids, n, d_oids);
  return GL_OK;
}

void gl_vm_destroy(gl_vm_t* vm) { delete vm; }

// ---------------------------------------------------------------------------
// on-disk fragment
// ---------------------------------------------------------------------------
namespace {
struct FragFileHeader {
  char magic[8];          // "GLFRAG01"
  uint32_t fid, fnum, ivnum, ovnum;
  uint64_t total_vnum;
  int32_t directed, load_strategy, edata_bytes, has_ie;
  uint64_t oe_entries, ie_entries;
  int32_t has_oids, pad;
  int64_t oid_base;
  uint64_t part_chunk;
};
bool put(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
bool get(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }
}  // namespace

int gl_frag_save(const gl_frag_t* f, const char* path) {
  GL_ARG(f && path, "null argument");
  if (f->offloaded) {
    set_error("fragment topology is offloaded");
    return GL_ERR_STATE;
  }
  FragFileHeader h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, "GLFRAG01", 8);
  h.fid = f->fid;
  h.fnum = f->fnum;
  h.ivnum = f->ivnum;
  h.ovnum = f->ovnum;
  h.total_vnum = f->total_vnum;
  h.directed = f->directed;
  h.load_strategy = f->load_strategy;
  h.edata_bytes = f->edata_bytes;
  h.has_ie = f->ie_alias_oe ? 0 : 1;
  h.oe_entries = f->oe.entries;
  h.ie_entries = h.has_ie ? f->ie.entries : 0;
  h.has_oids = f->h_inner_oids.empty() ? 0 : 1;
  h.oid_base = f->oid_base;
  h.part_chunk = f->part_chunk;
  FILE* fp = fopen(path, "wb");
  if (!fp) {
    set_error("gl_frag_save: cannot open %s", path);
    return GL_ERR_ARG;
  }
  bool ok = put(fp, &h, sizeof(h));
  std::vector<char> buf;
  auto dump = [&](const void* dptr, size_t bytes) {
    if (!ok || !bytes) return;
    buf.resize(bytes);
    if (cudaMemcpy(buf.data(), dptr, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) {
      ok = false;
      return;
    }
    ok = put(fp, buf.data(), bytes);
  };
  auto dump_csr = [&](const DevCsr& c, uint64_t rows) {
    dump(c.rp, sizeof(uint64_t) * (rows + 1));
    dump(c.col, sizeof(uint32_t) * c.entries);
    if (f->edata_bytes && c.w) dump(c.w, (size_t) f->edata_bytes * c.entries);
  };
  dump_csr(f->oe, f->ivnum);
  if (h.has_ie) dump_csr(f->ie, f->ivnum);
  dump(f->ovgid, sizeof(uint32_t) * f->ovnum);
  if (h.has_oids) ok = ok && put(fp, f->h_inner_oids.data(), sizeof(int64_t) * f->ivnum);
  ok = (fclose(fp) == 0) && ok;
  if (!ok) {
    set_error("gl_frag_save: write to %s failed", path);
    return GL_ERR_STATE;
  }
  return GL_OK;
}

int gl_frag_load(gl_frag_t** out, const char* path) {
  GL_ARG(out && path, "null argument");
  FILE* fp = fopen(path, "rb");
  if (!fp) {
    set_error("gl_frag_load: cannot open %s", path);
    return GL_ERR_ARG;
  }
  FragFileHeader h;
  bool ok = get(fp, &h, sizeof(h)) && memcmp(h.magic, "GLFRAG01", 8) == 0;
  if (!ok) {
    fclose(fp);
    set_error("gl_frag_load: %s is not a fragment file", path);
    return GL_ERR_ARG;
  }
  std::vector<uint64_t> orp((size_t) h.ivnum + 1), irp;
  std::vector<uint32_t> ocol((size_t) h.oe_entries), icol, ovgid(h.ovnum);
  std::vector<char> ow, iw;
  std::vector<int64_t> oids;
  ok = get(fp, orp.data(), sizeof(uint64_t) * orp.size()) && get(fp, ocol.data(), sizeof(uint32_t) * ocol.size());
  if (ok && h.edata_bytes) {
    ow.resize((size_t) h.edata_bytes * h.oe_entries);
    ok = get(fp, ow.data(), ow.size());
  }
  if (ok && h.has_ie) {
    irp.resize((size_t) h.ivnum + 1);
    icol.resize((size_t) h.ie_entries);
    ok = get(fp, irp.data(), sizeof(uint64_t) * irp.size()) && get(fp, icol.data(), sizeof(uint32_t) * icol.size());
    if (ok && h.edata_bytes) {
      iw.resize((size_t) h.edata_bytes * h.ie_entries);
      ok = get(fp, iw.data(), iw.size());
    }
  }
  ok = ok && get(fp, ovgid.data(), sizeof(uint32_t) * ovgid.size());
  if (ok && h.has_oids) {
    oids.resize(h.ivnum);
    ok = get(fp, oids.data(), sizeof(int64_t) * oids.size());
  }
  fclose(fp);
  if (!ok || orp[h.ivnum] != h.oe_entries) {
    set_error("gl_frag_load: %s is truncated or corrupt", path);
    return GL_ERR_ARG;
  }
  gl_frag_desc d;
  memset(&d, 0, sizeof(d));
  d.fid = h.fid;
  d.fnum = h.fnum;
  d.directed = h.directed;
  d.load_strategy = h.load_strategy;
  d.ivnum = h.ivnum;
  d.ovnum = h.ovnum;
  d.total_vnum = h.total_vnum;
  d.edata_bytes = h.edata_bytes;
  d.oe.row_ptr = orp.data();
  d.oe.col = ocol.data();
  d.oe.edata = h.edata_bytes ? ow.data() : nullptr;
  d.oe.rows = h.ivnum;
  if (h.has_ie) {
    d.ie.row_ptr = irp.data();
    d.ie.col = icol.data();
    d.ie.edata = h.edata_bytes ? iw.data() : nullptr;
    d.ie.rows = h.ivnum;
  }
  d.ovgid = ovgid.data();
  d.inner_oids = h.has_oids ? oids.data() : nullptr;
  d.oid_base = h.oid_base;
  GL_TRY(gl_frag_create(out, &d));
  (*out)->part_chunk = h.part_chunk;
  return GL_OK;
}

}  // extern "C"
