"""ctypes mirror of include/grape_b200.h (one class per opaque handle)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgrape_b200.so")

GL_LB = {"none": 0, "cm": 1, "wm": 2, "cta": 3, "strict": 4, "cmold": 5}
APP = {"bfs": 0, "sssp": 1, "wcc": 2, "pagerank": 3, "cdlp": 4, "lcc": 5, "wcc_opt": 6,
       "core_decomposition": 7, "kcore": 8, "kclique": 9, "bc": 10,
       "lcc_directed": 11, "pagerank_vc": 12, "cdlp_directed": 13,
       "pagerank_directed": 14, "bc_sources": 15, "pagerank_local": 16}
# gl_bc_value: the reference's Output() line `oid c sigma depth` (c is an f32 value, widened exactly)
BC_DTYPE = np.dtype([("centrality", "<f8"), ("path_num", "<f8"), ("depth", "<i8")])
RESULT_DTYPE = {0: np.int64, 1: np.float64, 2: np.int64, 3: np.float64, 4: np.int64, 5: np.float64, 6: np.int64,
                7: np.int64, 8: np.int64, 9: np.int64, 10: BC_DTYPE, 11: np.float64, 12: np.float64,
                13: np.int64, 14: np.float64, 15: np.float64, 16: np.float64}
GL_MAX_STEP_STATS = 512
GL_IPC_HANDLE_BYTES = 64


class GrapeError(RuntimeError):
    pass


class CsrDesc(C.Structure):
    _fields_ = [("row_ptr", C.c_void_p), ("col", C.c_void_p), ("edata", C.c_void_p), ("rows", C.c_uint64)]


class FragDesc(C.Structure):
    _fields_ = [("fid", C.c_uint32), ("fnum", C.c_uint32), ("directed", C.c_int), ("load_strategy", C.c_int),
                ("ivnum", C.c_uint32), ("ovnum", C.c_uint32), ("total_vnum", C.c_uint64),
                ("edata_bytes", C.c_int), ("oe", CsrDesc), ("ie", CsrDesc), ("ov_ie", CsrDesc),
                ("ovgid", C.c_void_p), ("inner_oids", C.c_void_p), ("oid_base", C.c_int64)]


class EdgesDesc(C.Structure):
    _fields_ = [("n_vertices", C.c_uint64), ("oids", C.c_void_p), ("n_edges", C.c_uint64),
                ("src", C.c_void_p), ("dst", C.c_void_p), ("edata", C.c_void_p), ("edata_bytes", C.c_int),
                ("directed", C.c_int), ("load_strategy", C.c_int), ("fid", C.c_uint32), ("fnum", C.c_uint32)]


class RmatDesc(C.Structure):
    _fields_ = [("scale", C.c_int), ("edgefactor", C.c_int), ("seed", C.c_uint64), ("weight_mode", C.c_int),
                ("fid", C.c_uint32), ("fnum", C.c_uint32)]


class FragInfo(C.Structure):
    _fields_ = [("fid", C.c_uint32), ("fnum", C.c_uint32), ("ivnum", C.c_uint32), ("ovnum", C.c_uint32),
                ("total_vnum", C.c_uint64), ("oe_num", C.c_uint64), ("ie_num", C.c_uint64),
                ("directed", C.c_int), ("load_strategy", C.c_int), ("edata_bytes", C.c_int),
                ("fid_offset", C.c_int), ("device_bytes", C.c_uint64), ("max_degree", C.c_uint32)]


class VcFragDesc(C.Structure):
    _fields_ = [("n_vertices", C.c_uint64), ("n_edges", C.c_uint64), ("src", C.c_void_p), ("dst", C.c_void_p),
                ("fid", C.c_uint32), ("fnum", C.c_uint32)]


class VcFragInfo(C.Structure):
    _fields_ = [("fid", C.c_uint32), ("fnum", C.c_uint32), ("n_vertices", C.c_uint64),
                ("master_begin", C.c_uint64), ("master_end", C.c_uint64), ("src_begin", C.c_uint64),
                ("src_end", C.c_uint64), ("dst_begin", C.c_uint64), ("dst_end", C.c_uint64),
                ("local_vnum", C.c_uint64), ("block_edges", C.c_uint64), ("entries", C.c_uint64),
                ("device_bytes", C.c_uint64)]


class AppConfig(C.Structure):
    _fields_ = [("lb", C.c_int), ("source_oid", C.c_int64), ("pr_delta", C.c_double), ("max_round", C.c_int),
                ("sssp_f64", C.c_int), ("sssp_prio", C.c_double), ("direction_opt", C.c_int),
                ("pr_pull", C.c_int), ("fuse_supersteps", C.c_int), ("reserved", C.c_int * 8)]


class QueryStats(C.Structure):
    _fields_ = [("supersteps", C.c_int), ("query_ms", C.c_double), ("entries_scanned", C.c_uint64),
                ("frontier_vertices", C.c_uint64), ("touched_vertices", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("msg_bytes_sent", C.c_uint64), ("n_steps", C.c_int),
                ("step_ms", C.c_float * GL_MAX_STEP_STATS), ("step_entries", C.c_uint64 * GL_MAX_STEP_STATS),
                ("step_frontier", C.c_uint32 * GL_MAX_STEP_STATS), ("step_mode", C.c_uint8 * GL_MAX_STEP_STATS)]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int)


class CommDesc(C.Structure):
    _fields_ = [("fid", C.c_uint32), ("fnum", C.c_uint32), ("allreduce", ALLREDUCE_FN), ("user", C.c_void_p),
                ("landing_bytes", C.c_size_t), ("mirror_bytes", C.c_size_t)]


class EdgeOp(C.Structure):
    _fields_ = [("kind", C.c_int), ("state", C.c_void_p), ("state2", C.c_void_p), ("out_bitmap", C.c_void_p),
                ("depth", C.c_uint32), ("use_weight", C.c_int)]


_LIB = None

# every symbol include/grape_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "gl_last_error", "gl_abi_version", "gl_device_info", "gl_frag_create", "gl_frag_build_from_edges",
    "gl_frag_build_rmat", "gl_rmat_edges_host", "gl_frag_get_info", "gl_frag_view_get", "gl_frag_copy_csr",
    "gl_frag_copy_ovgid", "gl_frag_oid2lid", "gl_frag_max_degree_vertex", "gl_frag_offload",
    "gl_frag_reload", "gl_frag_destroy", "gl_frag_save", "gl_frag_load", "gl_vm_create", "gl_vm_view_get",
    "gl_vm_oid2gid", "gl_vm_gid2oid", "gl_vm_destroy", "gl_app_set_vertex_map", "gl_comm_create", "gl_comm_export", "gl_comm_open",
    "gl_comm_destroy", "gl_comm_close_peers", "gl_comm_peer_write_us", "gl_mm_create", "gl_mm_init_buffer", "gl_mm_start",
    "gl_mm_start_round", "gl_mm_finish_round", "gl_mm_to_terminate", "gl_mm_force_continue", "gl_mm_view_get",
    "gl_mm_bytes_sent", "gl_mm_destroy", "gl_mm_process", "gl_mm_send_outer", "gl_mm_mirror_plan", "gl_mm_sync_values_to_ghosts", "gl_mm_sync_bits_to_ghosts",
    "gl_allreduce", "gl_bitmap_create",
    "gl_bitmap_clear", "gl_bitmap_count", "gl_bitmap_destroy", "gl_frag_prepare", "gl_queue_create", "gl_queue_clear",
    "gl_queue_size", "gl_queue_data", "gl_queue_fill_from_bitmap", "gl_queue_destroy", "gl_varray_create",
    "gl_varray_h2d", "gl_varray_d2h", "gl_varray_destroy", "gl_app_config_default", "gl_app_create", "gl_app_query", "gl_app_result",
    "gl_app_result_oids", "gl_app_set_sources", "gl_app_destroy", "gl_edge_scan_queue", "gl_compact_bitmap", "gl_dev_alloc",
    "gl_dev_free", "gl_dev_memset", "gl_dev_h2d", "gl_dev_d2h", "gl_dev_sync", "gl_kernel_launch_count",
    "gl_host_alloc_pinned", "gl_host_free_pinned", "gl_vcfrag_create", "gl_vcfrag_build_rmat",
    "gl_vcfrag_get_info", "gl_vcfrag_destroy", "gl_vc_app_create",
]


def build():
    """Compile the CUDA library in-tree (sm_90a)."""
    subprocess.check_call(["make", "-s", "-j8", "-C", _HERE])


def lib():
    """Loads libgrape_b200.so; raises if it is missing (no fallback)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise GrapeError("CUDA extension %s is missing: run __graft_entry__.build()" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.gl_last_error.restype = C.c_char_p
        L.gl_kernel_launch_count.restype = C.c_uint64
        L.gl_mm_bytes_sent.restype = C.c_uint64
        L.gl_mm_destroy.restype = None
        L.gl_vm_destroy.restype = None
        L.gl_queue_destroy.restype = None
        for f in ("gl_frag_destroy", "gl_comm_destroy", "gl_app_destroy", "gl_app_config_default",
                  "gl_vcfrag_destroy"):
            getattr(L, f).restype = None
        _LIB = L
    return _LIB


def check(st):
    if st != 0:
        raise GrapeError("gl status %d: %s" % (st, lib().gl_last_error().decode()))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def device_info():
    sm, cc, l2, hbm = C.c_int(), C.c_int(), C.c_size_t(), C.c_size_t()
    check(lib().gl_device_info(C.byref(sm), C.byref(cc), C.byref(l2), C.byref(hbm)))
    return {"sm_count": sm.value, "cc": cc.value, "l2_bytes": l2.value, "hbm_bytes": hbm.value}


def rmat_edges_host(scale, edgefactor=16, seed=1, weight_mode=0, first=0, count=None):
    d = RmatDesc(scale, edgefactor, seed, weight_mode, 0, 1)
    total = edgefactor << scale
    count = total - first if count is None else count
    src = np.empty(count, dtype=np.int64)
    dst = np.empty(count, dtype=np.int64)
    w = np.empty(count, dtype=np.float32) if weight_mode else None
    check(lib().gl_rmat_edges_host(C.byref(d), C.c_uint64(first), C.c_uint64(count), _p(src), _p(dst), _p(w)))
    return src, dst, w


class PinnedBuffer:
    """Page-locked host buffer (cudaMallocHost) exposed as a numpy array."""

    def __init__(self, nbytes):
        self.ptr = C.c_void_p()
        check(lib().gl_host_alloc_pinned(C.byref(self.ptr), C.c_size_t(max(nbytes, 16))))
        self.nbytes = nbytes

    def array(self, dtype, count):
        buf = (C.c_char * self.nbytes).from_address(self.ptr.value)
        return np.frombuffer(buf, dtype=dtype, count=count)

    def __del__(self):
        if getattr(self, "ptr", None) and self.ptr.value and _LIB is not None:
            _LIB.gl_host_free_pinned(self.ptr)
            self.ptr = C.c_void_p()


class Fragment:
    """Device-resident edge-cut fragment (HostFragment / DeviceFragment analogue)."""

    def __init__(self, handle):
        self.h = handle
        info = FragInfo()
        check(lib().gl_frag_get_info(self.h, C.byref(info)))
        self.info = info
        for k, _ in FragInfo._fields_:
            setattr(self, k, getattr(info, k))

    @classmethod
    def from_edges(cls, n_vertices, src, dst, w=None, directed=False, oids=None, fid=0, fnum=1,
                   w_dtype=np.float32):
        src = np.ascontiguousarray(src, dtype=np.int64)
        dst = np.ascontiguousarray(dst, dtype=np.int64)
        eb = 0
        if w is not None:
            w = np.ascontiguousarray(w, dtype=w_dtype)
            eb = w.dtype.itemsize
        oids_a = None if oids is None else np.ascontiguousarray(oids, dtype=np.int64)
        d = EdgesDesc(n_vertices, _p(oids_a), len(src), _p(src), _p(dst), _p(w), eb, 1 if directed else 0,
                      1 if directed else 0, fid, fnum)
        h = C.c_void_p()
        check(lib().gl_frag_build_from_edges(C.byref(h), C.byref(d)))
        return cls(h)

    @classmethod
    def rmat(cls, scale, edgefactor=16, seed=1, weight_mode=0, fid=0, fnum=1):
        d = RmatDesc(scale, edgefactor, seed, weight_mode, fid, fnum)
        h = C.c_void_p()
        check(lib().gl_frag_build_rmat(C.byref(h), C.byref(d)))
        return cls(h)

    @classmethod
    def from_csr(cls, ivnum, row_ptr, col, w=None, ovgid=None, total_vnum=None, fid=0, fnum=1,
                 directed=False, ie=None, inner_oids=None, oid_base=0):
        row_ptr = np.ascontiguousarray(row_ptr, dtype=np.uint64)
        col = np.ascontiguousarray(col, dtype=np.uint32)
        eb = 0
        if w is not None:
            w = np.ascontiguousarray(w)
            eb = w.dtype.itemsize
        d = FragDesc()
        d.fid, d.fnum, d.directed = fid, fnum, 1 if directed else 0
        d.load_strategy = 1 if directed else 0
        d.ivnum = ivnum
        d.ovnum = 0 if ovgid is None else len(ovgid)
        d.total_vnum = ivnum if total_vnum is None else total_vnum
        d.edata_bytes = eb
        d.oe = CsrDesc(_p(row_ptr), _p(col), _p(w), ivnum)
        keep = [row_ptr, col, w]
        if ie is not None:
            irp = np.ascontiguousarray(ie[0], dtype=np.uint64)
            icol = np.ascontiguousarray(ie[1], dtype=np.uint32)
            iw = None if ie[2] is None else np.ascontiguousarray(ie[2], dtype=w.dtype)
            d.ie = CsrDesc(_p(irp), _p(icol), _p(iw), ivnum)
            keep += [irp, icol, iw]
        og = None if ovgid is None else np.ascontiguousarray(ovgid, dtype=np.uint32)
        io = None if inner_oids is None else np.ascontiguousarray(inner_oids, dtype=np.int64)
        d.ovgid, d.inner_oids, d.oid_base = _p(og), _p(io), oid_base
        h = C.c_void_p()
        check(lib().gl_frag_create(C.byref(h), C.byref(d)))
        return cls(h)

    def csr(self, which=0):
        rows = self.ivnum if which < 2 else self.ovnum
        rp = np.zeros(rows + 1, dtype=np.uint64)
        check(lib().gl_frag_copy_csr(self.h, which, _p(rp), None, None))
        m = int(rp[-1])
        col = np.zeros(max(m, 1), dtype=np.uint32)
        w = None
        if self.edata_bytes and which < 2:
            w = np.zeros(max(m, 1), dtype=np.float32 if self.edata_bytes == 4 else np.float64)
        check(lib().gl_frag_copy_csr(self.h, which, None, _p(col), _p(w)))
        return rp, col[:m], (None if w is None else w[:m])

    def ovgid(self):
        g = np.zeros(max(self.ovnum, 1), dtype=np.uint32)
        check(lib().gl_frag_copy_ovgid(self.h, _p(g)))
        return g[: self.ovnum]

    def oid2lid(self, oid):
        lid = C.c_uint32()
        st = lib().gl_frag_oid2lid(self.h, C.c_int64(int(oid)), C.byref(lid))
        return lid.value if st == 0 else None

    def max_degree_vertex(self):
        lid, deg = C.c_uint32(), C.c_uint64()
        check(lib().gl_frag_max_degree_vertex(self.h, C.byref(lid), C.byref(deg)))
        return lid.value, deg.value

    def save(self, path):
        """Binary cache of the fragment (Serialize analogue)."""
        check(lib().gl_frag_save(self.h, path.encode()))

    @classmethod
    def load(cls, path):
        h = C.c_void_p()
        check(lib().gl_frag_load(C.byref(h), path.encode()))
        return cls(h)

    def offload(self):
        check(lib().gl_frag_offload(self.h))

    def reload(self):
        check(lib().gl_frag_reload(self.h))

    def close(self):
        if self.h:
            lib().gl_frag_destroy(self.h)
            self.h = None

    def __del__(self):
        if getattr(self, "h", None) and _LIB is not None:
            self.close()


class VcFragment:
    """Device-resident vertex-cut fragment (ImmutableVertexcutFragment with the 2-D VCPartitioner):
    fnum must be a perfect square; every rank may pass the whole edge list."""

    def __init__(self, handle):
        self.h = handle
        info = VcFragInfo()
        check(lib().gl_vcfrag_get_info(self.h, C.byref(info)))
        self.info = {k: getattr(info, k) for k, _ in VcFragInfo._fields_}
        self.fid, self.fnum = info.fid, info.fnum
        self.n_masters = info.master_end - info.master_begin

    @classmethod
    def from_edges(cls, n_vertices, src, dst, fid=0, fnum=1):
        src = np.ascontiguousarray(src, dtype=np.int64)
        dst = np.ascontiguousarray(dst, dtype=np.int64)
        d = VcFragDesc(n_vertices, len(src), _p(src), _p(dst), fid, fnum)
        h = C.c_void_p()
        check(lib().gl_vcfrag_create(C.byref(h), C.byref(d)))
        return cls(h)

    @classmethod
    def rmat(cls, scale, edgefactor=16, seed=1, fid=0, fnum=1):
        d = RmatDesc(scale, edgefactor, seed, 0, fid, fnum)
        h = C.c_void_p()
        check(lib().gl_vcfrag_build_rmat(C.byref(h), C.byref(d)))
        return cls(h)

    def close(self):
        if self.h:
            lib().gl_vcfrag_destroy(self.h)
            self.h = None

    def __del__(self):
        if getattr(self, "h", None) and _LIB is not None:
            self.close()


class Comm:
    """Fragment-group communicator.  `allreduce(array, op)` reduces a numpy
    array in place across the group (op: 0 sum, 1 min, 2 max)."""

    def __init__(self, fid, fnum, allreduce, landing_bytes, mirror_bytes=0):
        self._py_allreduce = allreduce

        def _cb(user, ptr, n, is_double, op):
            try:
                ty = C.c_double if is_double else C.c_int64
                arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ty)), (n,))
                self._py_allreduce(arr, op)
                return 0
            except Exception:  # pragma: no cover
                import traceback
                traceback.print_exc()
                return 1

        self._cb = ALLREDUCE_FN(_cb)
        d = CommDesc(fid, fnum, self._cb, None, landing_bytes, mirror_bytes)
        self.h = C.c_void_p()
        check(lib().gl_comm_create(C.byref(self.h), C.byref(d)))
        self.fid, self.fnum = fid, fnum

    def export(self):
        buf = (C.c_char * GL_IPC_HANDLE_BYTES)()
        check(lib().gl_comm_export(self.h, buf, GL_IPC_HANDLE_BYTES))
        return bytes(buf)

    def open(self, all_handles):
        blob = b"".join(all_handles)
        check(lib().gl_comm_open(self.h, blob, len(blob)))

    def peer_write_us(self, nbytes, vec16=True, all_peers=False, reps=20):
        us = C.c_double()
        check(lib().gl_comm_peer_write_us(self.h, C.c_size_t(nbytes), int(vec16), int(all_peers), int(reps), C.byref(us)))
        return us.value

    def close(self):
        if self.h:
            lib().gl_comm_destroy(self.h)
            self.h = None


class VertexMap:
    """Device vertex map (oid <-> gid) of a fragment group: oid_lists[f] = inner oids of fragment f in lid order."""

    def __init__(self, oid_lists):
        self._keep = [np.ascontiguousarray(o, dtype=np.int64) for o in oid_lists]
        n = len(self._keep)
        iv = (C.c_uint64 * n)(*[len(o) for o in self._keep])
        ptrs = (C.c_void_p * n)(*[o.ctypes.data if len(o) else None for o in self._keep])
        self.h = C.c_void_p()
        check(lib().gl_vm_create(C.byref(self.h), n, iv, ptrs))

    def oid2gid(self, oids):
        oids = np.ascontiguousarray(oids, dtype=np.int64)
        d_in, d_out = DeviceArray(oids), DeviceArray(nbytes=4 * max(len(oids), 1))
        check(lib().gl_vm_oid2gid(self.h, None, d_in.ptr, C.c_uint64(len(oids)), d_out.ptr))
        check(lib().gl_dev_sync())
        return d_out.download(np.uint32, len(oids))

    def gid2oid(self, gids):
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        d_in, d_out = DeviceArray(gids), DeviceArray(nbytes=8 * max(len(gids), 1))
        check(lib().gl_vm_gid2oid(self.h, None, d_in.ptr, C.c_uint64(len(gids)), d_out.ptr))
        check(lib().gl_dev_sync())
        return d_out.download(np.int64, len(gids))

    def close(self):
        if self.h:
            lib().gl_vm_destroy(self.h)
            self.h = None


class MsgOp(C.Structure):
    _fields_ = [("kind", C.c_int), ("state", C.c_void_p), ("out_bitmap", C.c_void_p)]


class MmView(C.Structure):
    _fields_ = [("fid", C.c_uint32), ("fnum", C.c_uint32), ("fid_offset", C.c_int), ("id_mask", C.c_uint32),
                ("capacity_bytes", C.c_uint32), ("send_slot", C.c_void_p), ("send_bytes", C.c_void_p),
                ("recv_slot", C.c_void_p), ("recv_bytes", C.c_void_p)]


MSG_OPS = {"set_bit": 0, "min_u32": 1, "min_f32": 2, "min_f64": 3, "add_f32": 4, "add_f64": 5}


class MessageManager:
    """Face 2 of the boundary (gl_mm_*): GPUMessageManager's round protocol and
    the fixed-function producer / consumer kernels, on the legacy stream."""

    def __init__(self, comm=None):
        self.h = C.c_void_p()
        check(lib().gl_mm_create(C.byref(self.h), comm.h if comm else None))

    def init_buffer(self, send_bytes, recv_bytes):
        check(lib().gl_mm_init_buffer(self.h, C.c_size_t(send_bytes), C.c_size_t(recv_bytes)))

    def start(self):
        check(lib().gl_mm_start(self.h))

    def start_round(self):
        check(lib().gl_mm_start_round(self.h, None))

    def finish_round(self):
        check(lib().gl_mm_finish_round(self.h, None))

    def to_terminate(self):
        t = C.c_int()
        check(lib().gl_mm_to_terminate(self.h, C.byref(t)))
        return bool(t.value)

    def force_continue(self):
        check(lib().gl_mm_force_continue(self.h))

    def view(self):
        v = MmView()
        check(lib().gl_mm_view_get(self.h, C.byref(v)))
        return v

    def bytes_sent(self):
        return int(lib().gl_mm_bytes_sent(self.h))

    def process(self, kind, state=None, out_bitmap=None):
        op = MsgOp(MSG_OPS[kind], state.ptr if state is not None else None,
                   out_bitmap.ptr if out_bitmap is not None else None)
        n = C.c_uint64()
        check(lib().gl_mm_process(self.h, None, C.byref(op), C.byref(n)))
        return n.value

    def send_outer(self, frag, remote_bitmap, state=None, value_bytes=0, clear_bits=True):
        check(lib().gl_mm_send_outer(self.h, None, frag.h, remote_bitmap.ptr,
                                     state.ptr if state is not None else None, int(value_bytes), int(clear_bits)))

    def mirror_plan(self, frag):
        """gl_mm_mirror_plan: collective, once per (manager, fragment)."""
        check(lib().gl_mm_mirror_plan(self.h, None, frag.h))

    def sync_values(self, values, elem_bytes):
        """gl_mm_sync_values_to_ghosts: every outer copy in `values` (device array over
        inner then outer vertices) takes its owner's value.  Collective."""
        check(lib().gl_mm_sync_values_to_ghosts(self.h, None, values.ptr, int(elem_bytes)))

    def sync_bits(self, bitmap):
        """gl_mm_sync_bits_to_ghosts: ghost bits |= owner bits.  Collective."""
        check(lib().gl_mm_sync_bits_to_ghosts(self.h, None, C.cast(bitmap.ptr, C.POINTER(C.c_uint32))))

    def allreduce(self, value, is_double=False, op=0):
        v = C.c_double(value) if is_double else C.c_int64(int(value))
        check(lib().gl_allreduce(self.h, None, C.byref(v), 1 if is_double else 0, int(op)))
        return v.value

    def close(self):
        if self.h:
            lib().gl_mm_destroy(self.h)
            self.h = None


def bitmap_count(bitmap_dev, nbits):
    n = C.c_uint64()
    check(lib().gl_bitmap_count(None, C.cast(bitmap_dev.ptr, C.POINTER(C.c_uint32)), C.c_uint64(nbits), C.byref(n)))
    return n.value


class App:
    """One PIE app bound to a fragment (GPUWorker analogue).  "kcore" and "kclique"
    take their k as App("kcore", frag, k=...) (carried in max_round); it has no
    default.  The result of "kclique" is one Python int: the k-clique count of the
    whole fragment group (result() takes no out array for it).  "bc" takes its
    source as App("bc", frag, source_oid=...) and returns a BC_DTYPE record
    (centrality, path_num, depth) per inner vertex.  "bc_sources" takes its list as
    App("bc_sources", frag, sources=[oids] or None (every vertex)) or later through
    set_sources(); its result is one double per inner vertex.  A VcFragment takes
    "pagerank_vc" (gl_vc_app_create); its result is one double per master vertex."""

    _NO_LIST = object()

    def __init__(self, kind, frag, comm=None, sources=_NO_LIST, **cfg):
        self.kind = APP[kind] if isinstance(kind, str) else kind
        self.frag = frag
        if self.kind in (APP["kcore"], APP["kclique"]):
            if "k" not in cfg:
                name = "kcore" if self.kind == APP["kcore"] else "kclique"
                raise GrapeError("%s needs k: App('%s', frag, k=...)" % (name, name))
            cfg["max_round"] = int(cfg.pop("k"))
        c = AppConfig()
        lib().gl_app_config_default(C.byref(c))
        for k, v in cfg.items():
            if k == "lb" and isinstance(v, str):
                v = GL_LB[v]
            if not hasattr(c, k):
                raise GrapeError("unknown app config key %r" % k)
            if k == "reserved":          # {index: value}
                for i, x in dict(v).items():
                    c.reserved[int(i)] = int(x)
                continue
            setattr(c, k, v)
        self.cfg = c
        self.h = C.c_void_p()
        create = lib().gl_vc_app_create if isinstance(frag, VcFragment) else lib().gl_app_create
        check(create(C.byref(self.h), self.kind, frag.h, comm.h if comm else None, C.byref(c)))
        self.stats = QueryStats()
        if sources is not App._NO_LIST:
            self.set_sources(sources)

    def set_sources(self, oids):
        """gl_app_set_sources: the list of source oids (None: every vertex of the fragment group)."""
        if oids is None:
            check(lib().gl_app_set_sources(self.h, None, C.c_uint64(0)))
            return
        self._sources = np.ascontiguousarray(oids, dtype=np.int64)
        check(lib().gl_app_set_sources(self.h, self._sources.ctypes.data_as(C.c_void_p),
                                       C.c_uint64(len(self._sources))))

    def set_vertex_map(self, vm):
        self._vm = vm
        check(lib().gl_app_set_vertex_map(self.h, vm.h if vm else None))

    def query(self):
        check(lib().gl_app_query(self.h, C.byref(self.stats)))
        return self.stats

    def result(self, out=None):
        dt = RESULT_DTYPE[self.kind]
        if self.kind == APP["kclique"]:
            if out is not None:
                raise GrapeError("kclique returns one int; result() takes no out array")
            one = np.zeros(1, dtype=dt)
            check(lib().gl_app_result(self.h, _p(one), one.nbytes))
            return int(one.view(np.uint64)[0])   # the uint64 count (modulo 2^64)
        if out is None:
            out = np.empty(self._count(), dtype=dt)
        check(lib().gl_app_result(self.h, _p(out), out.nbytes))
        return out

    def _count(self):
        return self.frag.n_masters if isinstance(self.frag, VcFragment) else self.frag.ivnum

    def result_oids(self):
        out = np.empty(self._count(), dtype=np.int64)
        check(lib().gl_app_result_oids(self.h, _p(out), len(out)))
        return out

    def close(self):
        if self.h:
            lib().gl_app_destroy(self.h)
            self.h = None

    def __del__(self):
        if getattr(self, "h", None) and _LIB is not None:
            self.close()


class DeviceArray:
    """Tiny device buffer helper for the engine-primitive tests."""

    def __init__(self, host=None, nbytes=None):
        self.ptr = C.c_void_p()
        self.nbytes = host.nbytes if host is not None else nbytes
        check(lib().gl_dev_alloc(C.byref(self.ptr), C.c_size_t(max(self.nbytes, 16))))
        if host is not None:
            self.upload(host)

    def upload(self, host):
        host = np.ascontiguousarray(host)
        check(lib().gl_dev_h2d(self.ptr, _p(host), C.c_size_t(host.nbytes)))

    def download(self, dtype, count):
        out = np.empty(count, dtype=dtype)
        check(lib().gl_dev_d2h(_p(out), self.ptr, C.c_size_t(out.nbytes)))
        return out

    def fill(self, byte):
        check(lib().gl_dev_memset(self.ptr, int(byte), C.c_size_t(self.nbytes)))

    def free(self):
        if self.ptr:
            lib().gl_dev_free(self.ptr)
            self.ptr = C.c_void_p()

    def __del__(self):
        if getattr(self, "ptr", None) and self.ptr.value and _LIB is not None:
            self.free()


OPS = {"bfs_level": 0, "min_relax_u32": 1, "min_relax_f32": 2, "add_scatter_f64": 3, "count": 4}


def edge_scan_queue(frag, queue_dev, n, op, lb, state=None, state2=None, out_bitmap=None, depth=0,
                    use_weight=0):
    """ForEachOutgoingEdge(WorkSourceArray(queue, n), op, lb) -> entries scanned."""
    o = EdgeOp(OPS[op] if isinstance(op, str) else op,
               state.ptr if state is not None else None,
               state2.ptr if state2 is not None else None,
               out_bitmap.ptr if out_bitmap is not None else None, depth, use_weight)
    scanned = C.c_uint64()
    lbv = GL_LB[lb] if isinstance(lb, str) else lb
    check(lib().gl_edge_scan_queue(frag.h, None, queue_dev.ptr, C.c_uint32(n), C.byref(o), lbv,
                                   C.byref(scanned)))
    return scanned.value


def compact_bitmap(bitmap_dev, n_bits, queue_dev):
    cnt = C.c_uint32()
    check(lib().gl_compact_bitmap(None, bitmap_dev.ptr, C.c_uint32(n_bits), queue_dev.ptr, C.byref(cnt)))
    return cnt.value
