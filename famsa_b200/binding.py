"""ctypes binding of libfamsa_b200.so (the C ABI declared in include/famsa_b200.h)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import profiles, seqio

_HERE = os.path.dirname(os.path.abspath(__file__))

EXPORTED_SYMBOLS = [
    "famsa_abi_version", "famsa_create", "famsa_destroy", "famsa_last_error", "famsa_kernel_launches",
    "famsa_lcs_upload", "famsa_lcs_upload_sorted", "famsa_lcs_sorted_order", "famsa_lcs_last_tiles", "famsa_lcs_n_seqs", "famsa_lcs_triangle", "famsa_lcs_triangle_device",
    "famsa_device_alloc", "famsa_device_free", "famsa_ipc_export", "famsa_ipc_open", "famsa_ipc_close", "famsa_lcs_triangle_exchange",
    "famsa_lcs_rows", "famsa_lcs_rows_device", "famsa_lcs_assign", "famsa_lcs_assign_shard", "famsa_lcs_upgma", "famsa_lcs_upgma_from_triangle", "famsa_lcs_prim", "famsa_lcs_slink", "famsa_lcs_nj", "famsa_dist_export", "famsa_transform_f64", "famsa_transform_f32",
    "famsa_lcs_last_timing", "famsa_dp_align_batch", "famsa_dp_align_batch_device", "famsa_dp_last_timing",
    "famsa_prof_set_scoring", "famsa_prof_put", "famsa_prof_merge_batch", "famsa_prof_get", "famsa_prof_drop",
    "famsa_prof_last_timing", "famsa_prof_stats", "famsa_prof_align_tree", "famsa_prof_tree_paths",
    "famsa_prof_refine", "famsa_prof_refined_rows", "famsa_prof_put_rows", "famsa_prof_tree_rows",
]

PROF_LEAF = 0x80000000            # FAMSA_PROF_LEAF

WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64)   # famsa_write_fn


class DpProfile(C.Structure):
    _fields_ = [("scores", C.c_void_p), ("counters", C.c_void_p), ("width", C.c_uint32), ("card", C.c_uint32)]


class DpJob(C.Structure):
    _fields_ = [("p1", DpProfile), ("p2", DpProfile)]


class DpResult(C.Structure):
    _fields_ = [("total_score", C.c_int64), ("last", C.c_int64 * 3), ("path_offset", C.c_uint64),
                ("dirs_offset", C.c_uint64), ("path_len", C.c_uint32), ("rows_width", C.c_uint32),
                ("cols_width", C.c_uint32), ("swapped", C.c_uint8), ("variant", C.c_uint8), ("pad", C.c_uint8 * 2)]


class ProfMerge(C.Structure):
    _fields_ = [("child1", C.c_uint32), ("child2", C.c_uint32)]


class TreeStats(C.Structure):
    _fields_ = [("wall_ms", C.c_double), ("device_ms", C.c_double), ("cells", C.c_uint64), ("n_batches", C.c_uint32),
                ("n_drains", C.c_uint32), ("max_in_flight", C.c_uint32), ("pad", C.c_uint32),
                ("peak_resident_bytes", C.c_uint64)]


class RefineStats(C.Structure):
    _fields_ = [("wall_ms", C.c_double), ("device_ms", C.c_double), ("n_tries", C.c_uint32), ("n_realigned", C.c_uint32),
                ("n_accepted", C.c_uint32), ("n_identical", C.c_uint32), ("cells", C.c_uint64)]


REFINE_NO_GAP_OPT = 1        # -dgo
REFINE_NO_TOTAL_SCORE = 2    # -dsp
REFINE_TREE_ROWS = 4         # famsa_prof_refine on the rows famsa_prof_tree_rows kept on the device
PUT_ROWS_FROM_TEXT = 1       # famsa_prof_put_rows: the profile the reference builds from rows read as text


class FamsaError(RuntimeError):
    pass


def lib_path() -> str:
    return os.path.join(_HERE, "lib", "libfamsa_b200.so")


_lib = None


def load_library() -> C.CDLL:
    """Load the CUDA library; raise (never fall back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise FamsaError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(there is no CPU fallback)")
    lib = C.CDLL(path)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    lib.famsa_abi_version.restype = i32
    lib.famsa_create.argtypes = [i32, C.POINTER(vp)]
    lib.famsa_destroy.argtypes = [vp]
    lib.famsa_destroy.restype = None
    lib.famsa_last_error.restype = C.c_char_p
    lib.famsa_kernel_launches.argtypes = [vp]
    lib.famsa_kernel_launches.restype = u64
    lib.famsa_lcs_upload.argtypes = [vp, vp, vp, vp, u32]
    lib.famsa_lcs_n_seqs.argtypes = [vp]
    lib.famsa_lcs_upload_sorted.argtypes = [vp, vp, vp, vp, u32]
    lib.famsa_lcs_sorted_order.argtypes = [vp, vp]
    lib.famsa_lcs_last_tiles.argtypes = [vp]
    lib.famsa_lcs_last_tiles.restype = u64
    lib.famsa_lcs_n_seqs.restype = u32
    lib.famsa_lcs_triangle.argtypes = [vp, u32, u32, vp, i32]
    lib.famsa_lcs_triangle_device.argtypes = [vp, u32, u32, vp, i32, vp]
    lib.famsa_device_alloc.argtypes = [vp, u64, C.POINTER(vp)]
    lib.famsa_device_free.argtypes = [vp, vp]
    lib.famsa_ipc_export.argtypes = [vp, vp, vp]
    lib.famsa_ipc_open.argtypes = [vp, vp, C.POINTER(vp)]
    lib.famsa_ipc_close.argtypes = [vp, vp]
    lib.famsa_lcs_triangle_exchange.argtypes = [vp, u32, u32, vp, vp, u32, i32, u32, vp]
    lib.famsa_lcs_rows.argtypes = [vp, vp, u32, vp, u32, vp, i32]
    lib.famsa_lcs_rows_device.argtypes = [vp, vp, u32, vp, u32, vp, i32, vp]
    lib.famsa_lcs_prim.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.famsa_lcs_slink.argtypes = [vp, i32, vp]
    lib.famsa_lcs_nj.argtypes = [vp, i32, vp]
    lib.famsa_lcs_assign.argtypes = [vp, vp, u32, i32, vp, vp]
    lib.famsa_lcs_upgma.argtypes = [vp, i32, i32, vp]
    lib.famsa_lcs_upgma_from_triangle.argtypes = [vp, i32, i32, vp, i32, vp]
    lib.famsa_lcs_assign_shard.argtypes = [vp, vp, u32, i32, u32, u32, vp, vp]
    lib.famsa_dist_export.argtypes = [vp, i32, i32, i32, vp, vp, u64, WRITE_FN, vp, C.POINTER(u64)]
    lib.famsa_debug_format_f32.argtypes = [vp, u64, vp, C.POINTER(u64)]
    lib.famsa_transform_f64.argtypes = [i32, u32, u32, u32]
    lib.famsa_transform_f64.restype = C.c_double
    lib.famsa_transform_f32.argtypes = [i32, u32, u32, u32]
    lib.famsa_transform_f32.restype = C.c_float
    lib.famsa_lcs_last_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(u64)]
    lib.famsa_prof_set_scoring.argtypes = [vp, vp]
    lib.famsa_prof_put.argtypes = [vp, vp, u32, vp]
    lib.famsa_prof_put_rows.argtypes = [vp, vp, u32, u32, vp, C.c_int, C.POINTER(u32)]
    lib.famsa_prof_merge_batch.argtypes = [vp, vp, u32, vp, vp, vp, vp, u64]
    lib.famsa_prof_get.argtypes = [vp, u32, C.POINTER(u32), C.POINTER(u32), vp, vp]
    lib.famsa_prof_drop.argtypes = [vp, vp, u32]
    lib.famsa_prof_last_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lib.famsa_prof_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    lib.famsa_prof_align_tree.argtypes = [vp, vp, u32, vp, vp, C.POINTER(u32), C.POINTER(u64), vp]
    lib.famsa_prof_tree_paths.argtypes = [vp, vp, u64]
    lib.famsa_prof_tree_rows.argtypes = [vp, vp, u32, vp, u64, C.POINTER(u32)]
    lib.famsa_prof_refine.argtypes = [vp, u32, vp, u32, u32, vp, u32, C.c_int, C.POINTER(u32), C.POINTER(u32),
                                      C.POINTER(C.c_int64), vp]
    lib.famsa_prof_refined_rows.argtypes = [vp, vp, u64]
    lib.famsa_dp_align_batch.argtypes = [vp, vp, u32, vp, vp, vp, vp]
    lib.famsa_dp_align_batch_device.argtypes = [vp, vp, u32, vp, vp, vp, vp, vp]
    lib.famsa_dp_last_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(u64)]
    _lib = lib
    return lib


def _ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def unpack_assignment(packed: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(assignments uint32[n], min_dist float32[n]) from the MIN-reduced packed array of famsa_lcs_assign_shard."""
    p = np.ascontiguousarray(packed, dtype=np.int64).view(np.uint64)
    return (p & np.uint64(0xffffffff)).astype(np.uint32), (p >> np.uint64(32)).astype(np.uint32).view(np.float32)


def tri_size(row_begin: int, row_end: int) -> int:
    f = lambda r: r * (r - 1) // 2 if r else 0
    return f(row_end) - f(row_begin)


class Engine:
    """One context on one GPU.  Mirrors the reference's per-thread CLCSBP + batch drivers:
    upload() ~ ComputeBitMasks for every sequence, triangle() ~ calculateDistanceMatrix,
    rows() ~ calculateDistanceVector / Range / RangeSV (raw LCS lengths, Transform stays on host)."""

    def __init__(self, device: int = -1):
        self.lib = load_library()
        h = C.c_void_p()
        self._check(self.lib.famsa_create(device, C.byref(h)))
        self.h = h
        self.n = 0

    def _check(self, rc: int):
        if rc != 0:
            raise FamsaError(f"[{rc}] {self.lib.famsa_last_error().decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.lib.famsa_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---------------------------------------------------------------- HP-1
    def upload(self, codes: np.ndarray, offsets: np.ndarray, lens: np.ndarray):
        codes = np.ascontiguousarray(codes, dtype=np.int8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        lens = np.ascontiguousarray(lens, dtype=np.uint32)
        self._check(self.lib.famsa_lcs_upload(self.h, _ptr(codes), _ptr(offsets), _ptr(lens), len(lens)))
        self.n = len(lens)
        self._tree_width = None

    def upload_sorted(self, codes: np.ndarray, offsets: np.ndarray, lens: np.ndarray) -> np.ndarray:
        """famsa_lcs_upload_sorted: indices of later calls are positions in the length-descending order; returns
        sorted_to_caller (position -> caller index)."""
        codes = np.ascontiguousarray(codes, dtype=np.int8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        lens = np.ascontiguousarray(lens, dtype=np.uint32)
        self._check(self.lib.famsa_lcs_upload_sorted(self.h, _ptr(codes), _ptr(offsets), _ptr(lens), len(lens)))
        self.n = len(lens)
        self._tree_width = None
        order = np.zeros(max(self.n, 1), dtype=np.uint32)
        self._check(self.lib.famsa_lcs_sorted_order(self.h, _ptr(order)))
        return order[:self.n]

    def last_tiles(self) -> int:
        return int(self.lib.famsa_lcs_last_tiles(self.h))

    def triangle(self, row_begin: int = 0, row_end: int | None = None, dtype=np.uint16,
                 out: np.ndarray | None = None) -> np.ndarray:
        row_end = self.n if row_end is None else row_end
        size = tri_size(row_begin, row_end)
        if out is None:
            out = np.empty(max(size, 1), dtype=dtype)
        self._check(self.lib.famsa_lcs_triangle(self.h, row_begin, row_end, _ptr(out), out.dtype.itemsize))
        return out[:size]

    def triangle_device(self, row_begin: int, row_end: int, d_out_ptr: int, elem_bytes: int, stream: int = 0):
        self._check(self.lib.famsa_lcs_triangle_device(self.h, row_begin, row_end, C.c_void_p(d_out_ptr),
                                                       elem_bytes, C.c_void_p(stream) if stream else None))

    # multi-GPU exchange over peer memory (famsa_lcs_triangle_exchange)
    def device_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self.lib.famsa_device_alloc(self.h, nbytes, C.byref(p)))
        return int(p.value)

    def device_free(self, d_ptr: int):
        self._check(self.lib.famsa_device_free(self.h, C.c_void_p(d_ptr)))

    def ipc_export(self, d_ptr: int) -> bytes:
        h = (C.c_uint8 * 64)()
        self._check(self.lib.famsa_ipc_export(self.h, C.c_void_p(d_ptr), h))
        return bytes(h)

    def ipc_open(self, handle: bytes) -> int:
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        p = C.c_void_p()
        self._check(self.lib.famsa_ipc_open(self.h, h, C.byref(p)))
        return int(p.value)

    def ipc_close(self, d_ptr: int):
        self._check(self.lib.famsa_ipc_close(self.h, C.c_void_p(d_ptr)))

    def triangle_exchange(self, row_begin: int, row_end: int, d_full: int, peers, elem_bytes: int, n_pieces: int = 8,
                          stream: int = 0):
        arr = (C.c_void_p * max(len(peers), 1))(*[C.c_void_p(p) for p in peers])
        self._check(self.lib.famsa_lcs_triangle_exchange(self.h, row_begin, row_end, C.c_void_p(d_full), arr, len(peers),
                                                         elem_bytes, n_pieces, C.c_void_p(stream) if stream else None))

    def rows(self, ref_ids, col_ids=None, n_col: int | None = None, dtype=np.uint32) -> np.ndarray:
        ref = np.ascontiguousarray(ref_ids, dtype=np.uint32)
        cols = None if col_ids is None else np.ascontiguousarray(col_ids, dtype=np.uint32)
        n_col = (self.n if n_col is None else n_col) if cols is None else len(cols)
        out = np.empty((len(ref), max(n_col, 1)), dtype=dtype)
        out = out[:, :n_col] if n_col else out[:, :0]
        buf = np.empty(max(len(ref) * n_col, 1), dtype=dtype)
        self._check(self.lib.famsa_lcs_rows(self.h, _ptr(ref), len(ref), _ptr(cols), n_col, _ptr(buf),
                                            buf.dtype.itemsize))
        return buf[:len(ref) * n_col].reshape(len(ref), n_col)

    def dist_export(self, ids, kind: int = 0, square: bool = False, pid: bool = False, out=None,
                    chunk_bytes: int = 0):
        """famsa_dist_export: the -dist_export CSV of the set of the last upload() (caller order), byte for byte what
        DistanceCalculator writes.  ids: the FASTA headers without '>' (str or bytes).  Returns the text as bytes, or,
        with `out` (a binary file object), writes it there chunk by chunk and returns the byte count."""
        raw = [i.encode() if isinstance(i, str) else bytes(i) for i in ids]
        if len(raw) != self.n:
            raise ValueError(f"{len(raw)} ids for {self.n} uploaded sequences")
        blob = b"".join(raw)
        offs = np.zeros(len(raw) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(r) for r in raw], dtype=np.uint64)
        buf = C.create_string_buffer(blob, max(len(blob), 1))
        parts = bytearray() if out is None else None
        failure = []

        def sink(_user, ptr, n):
            try:
                view = memoryview((C.c_char * n).from_address(ptr)).cast("B")
                if parts is None:
                    out.write(view)
                else:
                    parts.extend(view)
                return 0
            except BaseException as e:          # reported after the call; the library stops writing
                failure.append(e)
                return 1

        cb = WRITE_FN(sink)
        written = C.c_uint64()
        rc = self.lib.famsa_dist_export(self.h, kind, int(square), int(pid), buf, _ptr(offs), chunk_bytes, cb, None,
                                        C.byref(written))
        if failure:
            raise failure[0]
        self._check(rc)
        return bytes(parts) if out is None else written.value

    def debug_format_f32(self, values) -> bytes:
        """famsa_debug_format_f32: the device formatter alone, every value followed by ','."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        out = np.empty(max(40 * v.size, 1), dtype=np.uint8)
        n = C.c_uint64()
        self._check(self.lib.famsa_debug_format_f32(_ptr(v), v.size, _ptr(out), C.byref(n)))
        return out[:n.value].tobytes()

    def prim(self, kind: int = 0):
        """MSTPrim's vertex loop on the device: (edge_from, edge_to, edge_dist, prim_order)."""
        m = max(self.n - 1, 1)
        f = np.zeros(m, dtype=np.int32); t = np.zeros(m, dtype=np.int32)
        d = np.zeros(m, dtype=np.float64); o = np.zeros(max(self.n, 1), dtype=np.int32)
        self._check(self.lib.famsa_lcs_prim(self.h, kind, _ptr(f), _ptr(t), _ptr(d), _ptr(o)))
        return f[:self.n - 1], t[:self.n - 1], d[:self.n - 1], o[:self.n]

    def slink(self, kind: int = 0) -> np.ndarray:
        """famsa_lcs_slink: SingleLinkage's guide tree of the uploaded set, (n-1, 2) child ids of the internal nodes."""
        t = np.zeros((max(self.n - 1, 1), 2), dtype=np.int32)
        self._check(self.lib.famsa_lcs_slink(self.h, kind, _ptr(t)))
        return t[:max(self.n - 1, 0)]

    def nj(self, kind: int = 0) -> np.ndarray:
        """famsa_lcs_nj: NeighborJoining's guide tree of the uploaded set, (n-1, 2) child ids of the internal nodes."""
        t = np.zeros((max(self.n - 1, 1), 2), dtype=np.int32)
        self._check(self.lib.famsa_lcs_nj(self.h, kind, _ptr(t)))
        return t[:self.n - 1]

    def upgma(self, kind: int = 0, modified: bool = False, d_triangle_ptr: int = 0, elem_bytes: int = 2) -> np.ndarray:
        """famsa_lcs_upgma[_from_triangle]: the UPGMA guide tree of the uploaded set, (n-1, 2) child ids of the internal
        nodes; d_triangle_ptr: a packed LCS triangle already on the device (else it is computed)."""
        t = np.zeros((max(self.n - 1, 1), 2), dtype=np.int32)
        if d_triangle_ptr:
            self._check(self.lib.famsa_lcs_upgma_from_triangle(self.h, kind, int(modified), C.c_void_p(d_triangle_ptr), elem_bytes, _ptr(t)))
        else:
            self._check(self.lib.famsa_lcs_upgma(self.h, kind, int(modified), _ptr(t)))
        return t[:self.n - 1]

    def assign(self, seed_ids, kind: int = 0) -> tuple[np.ndarray, np.ndarray]:
        """FastTree<>::makeEvaluation's assignment loop: (assignments uint32[n], min_dist float32[n])."""
        seeds = np.ascontiguousarray(seed_ids, dtype=np.uint32)
        a = np.empty(self.n, dtype=np.uint32)
        d = np.empty(self.n, dtype=np.float32)
        self._check(self.lib.famsa_lcs_assign(self.h, _ptr(seeds), len(seeds), kind, _ptr(a), _ptr(d)))
        return a, d

    def assign_shard(self, seed_ids, shard: int, n_shards: int, d_packed_ptr: int, kind: int = 0, stream: int = 0):
        """famsa_lcs_assign_shard: this rank's slice of the medoid assignment, packed for a MIN all-reduce, into the
        device int64 array at d_packed_ptr (n entries).  unpack_assignment() splits the reduced array."""
        seeds = np.ascontiguousarray(seed_ids, dtype=np.uint32)
        self._check(self.lib.famsa_lcs_assign_shard(self.h, _ptr(seeds), len(seeds), kind, shard, n_shards,
                                                    C.c_void_p(d_packed_ptr), C.c_void_p(stream) if stream else None))

    def rows_device(self, d_ref_ptr: int, n_ref: int, d_col_ptr: int, n_col: int, d_out_ptr: int,
                    elem_bytes: int, stream: int = 0):
        self._check(self.lib.famsa_lcs_rows_device(self.h, C.c_void_p(d_ref_ptr), n_ref,
                                                   C.c_void_p(d_col_ptr) if d_col_ptr else None, n_col,
                                                   C.c_void_p(d_out_ptr), elem_bytes,
                                                   C.c_void_p(stream) if stream else None))

    # ---------------------------------------------------------------- HP-2
    def dp_align_batch(self, jobs, gaps, want_dirs: bool = False):
        """jobs: list of (scores1, counters1, card1, scores2, counters2, card2) with scores (W+1,32) int64 and
        counters (W+1,32) int32 -- the two arguments of CProfile::Align.  Returns a list of dicts
        (path, total, last, swapped, variant[, dirs]) in job order."""
        n = len(jobs)
        arr = (DpJob * max(n, 1))()
        keep = []
        path_total = dirs_total = 0
        for k, (s1, c1, k1, s2, c2, k2) in enumerate(jobs):
            s1 = np.ascontiguousarray(s1, dtype=np.int64); c1 = np.ascontiguousarray(c1, dtype=np.int32)
            s2 = np.ascontiguousarray(s2, dtype=np.int64); c2 = np.ascontiguousarray(c2, dtype=np.int32)
            keep += [s1, c1, s2, c2]
            w1, w2 = s1.shape[0] - 1, s2.shape[0] - 1
            arr[k].p1 = DpProfile(s1.ctypes.data, c1.ctypes.data, w1, k1)
            arr[k].p2 = DpProfile(s2.ctypes.data, c2.ctypes.data, w2, k2)
            path_total += w1 + w2
            dirs_total += (w1 + 1) * (w2 + 1)
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        res = (DpResult * max(n, 1))()
        path = np.zeros(max(path_total, 1), dtype=np.uint8)
        dirs = np.zeros(max(dirs_total, 1), dtype=np.uint8) if want_dirs else None
        self._check(self.lib.famsa_dp_align_batch(self.h, C.byref(arr), n, _ptr(g), C.byref(res), _ptr(path), _ptr(dirs)))
        out = []
        for k in range(n):
            r = res[k]
            d = dict(path=path[r.path_offset:r.path_offset + r.path_len].copy(), total=int(r.total_score),
                     last=np.array(list(r.last), dtype=np.int64), swapped=bool(r.swapped), variant=int(r.variant))
            if want_dirs:
                d["dirs"] = dirs[r.dirs_offset:r.dirs_offset + (r.rows_width + 1) * (r.cols_width + 1)].reshape(
                    r.rows_width + 1, r.cols_width + 1).copy()
            out.append(d)
        return out

    def dp_jobs(self, jobs):
        """ctypes job array for dp_align_batch_raw (keeps the numpy tables alive): build once, call many times."""
        n = len(jobs)
        arr = (DpJob * max(n, 1))()
        keep = []
        path_total = 0
        for k, (s1, c1, k1, s2, c2, k2) in enumerate(jobs):
            s1 = np.ascontiguousarray(s1, dtype=np.int64); c1 = np.ascontiguousarray(c1, dtype=np.int32)
            s2 = np.ascontiguousarray(s2, dtype=np.int64); c2 = np.ascontiguousarray(c2, dtype=np.int32)
            keep += [s1, c1, s2, c2]
            arr[k].p1 = DpProfile(s1.ctypes.data, c1.ctypes.data, s1.shape[0] - 1, k1)
            arr[k].p2 = DpProfile(s2.ctypes.data, c2.ctypes.data, s2.shape[0] - 1, k2)
            path_total += s1.shape[0] + s2.shape[0] - 2
        return arr, keep, path_total

    def dp_align_batch_raw(self, arr, n: int, gaps, res, path):
        """famsa_dp_align_batch on prebuilt arrays (res: (DpResult * n)(), path: uint8 numpy buffer) -- the call a C
        caller makes, without this binding's per-job Python work."""
        self._check(self.lib.famsa_dp_align_batch(self.h, C.byref(arr), n, _ptr(gaps), C.byref(res), _ptr(path), None))

    def prof_merge_batch_raw(self, arr, n: int, gaps, ids, res, path):
        """famsa_prof_merge_batch on prebuilt arrays (arr: (ProfMerge * n)(), ids: uint32 numpy, res: (DpResult * n)())."""
        self._check(self.lib.famsa_prof_merge_batch(self.h, C.byref(arr), n, _ptr(gaps), _ptr(ids), C.byref(res), _ptr(path), path.size))

    def dp_align_batch_device(self, job_array, n: int, gaps, d_results: int, d_path: int, d_dirs: int = 0, stream: int = 0):
        """job_array: ctypes (DpJob * n) whose table pointers are DEVICE pointers; d_* are device pointers."""
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        self._check(self.lib.famsa_dp_align_batch_device(self.h, C.byref(job_array), n, _ptr(g), C.c_void_p(d_results),
                                                         C.c_void_p(d_path), C.c_void_p(d_dirs) if d_dirs else None,
                                                         C.c_void_p(stream) if stream else None))

    # ---- resident profiles (ConstructProfile's merge part on the device)
    def prof_set_scoring(self, score_matrix):
        sm = np.ascontiguousarray(score_matrix, dtype=np.int64)
        assert sm.shape == (24, 24)
        self._check(self.lib.famsa_prof_set_scoring(self.h, _ptr(sm)))

    def prof_put(self, profiles) -> list[int]:
        """profiles: list of (scores (W+1,32) int64, counters (W+1,32) int32, card).  Returns resident ids."""
        n = len(profiles)
        arr = (DpProfile * max(n, 1))()
        keep = []
        for k, (s, c, card) in enumerate(profiles):
            s = np.ascontiguousarray(s, dtype=np.int64); c = np.ascontiguousarray(c, dtype=np.int32)
            keep += [s, c]
            arr[k] = DpProfile(s.ctypes.data, c.ctypes.data, s.shape[0] - 1, card)
        ids = np.zeros(max(n, 1), dtype=np.uint32)
        self._check(self.lib.famsa_prof_put(self.h, C.byref(arr), n, _ptr(ids)))
        return [int(x) for x in ids[:n]]

    def prof_put_rows(self, rows, gaps, from_text: bool = False) -> int:
        """famsa_prof_put_rows: a resident profile from a finished alignment, rows (n, width) uint8 codes with GAP = 30
        (seqio.encode_gapped), in the order the profile keeps them.  from_text: FAMSA_PUT_ROWS_FROM_TEXT, the profile
        (width - 1 columns) the reference builds from rows read as text.  Returns its id."""
        r = np.ascontiguousarray(rows, dtype=np.uint8)
        if r.ndim != 2:
            raise ValueError("rows must be an (n_rows, width) array")
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        pid = C.c_uint32()
        self._check(self.lib.famsa_prof_put_rows(self.h, _ptr(r), r.shape[0], r.shape[1], _ptr(g), PUT_ROWS_FROM_TEXT if from_text else 0,
                                                 C.byref(pid)))
        return pid.value

    def align_profiles(self, rows1: list[str], rows2: list[str], gaps) -> dict:
        """FAMSA's profile-profile mode (famsa in1 in2 out, CFAMSA::alignProfiles without its refinement): the two
        alignments' rows as text, gaps = the rescaled costs of adjustParams(n1 + n2).  Needs prof_set_scoring.
        Returns dict(order, rows, width, total, swapped, variant, path, merged_id): output row k is rows[k], input row
        order[k] of rows1 + rows2 with its letters as given; merged_id is the merged resident profile (the caller drops it)."""
        for k, rows in enumerate((rows1, rows2), 1):
            if not rows or any(len(r) != len(rows[0]) for r in rows):        # famsa.cpp:83-89 "Incorrect profile"
                raise ValueError(f"alignment {k} is empty or its rows differ in length")
        ids = [self.prof_put_rows(np.stack([seqio.encode_gapped(r) for r in rows1]), gaps, from_text=True)]
        try:
            ids.append(self.prof_put_rows(np.stack([seqio.encode_gapped(r) for r in rows2]), gaps, from_text=True))
            (merged,), (res,) = self.prof_merge_batch([tuple(ids)], gaps, [(len(rows1[0]) - 1, len(rows2[0]) - 1)])
        except Exception:
            for i in ids:                        # whichever of the inputs is still resident
                try:
                    self.prof_drop([i])
                except FamsaError:
                    pass
            raise
        order, rows = profiles.rows_after_merge(rows1, rows2, res["path"], res["swapped"], from_text=True)
        return dict(order=order, rows=rows, width=len(rows[0]), total=res["total"], swapped=res["swapped"],
                    variant=res["variant"], path=res["path"], merged_id=merged)

    def prof_merge_batch(self, merges, gaps, widths):
        """merges: list of (child1, child2) -- resident ids or PROF_LEAF | sequence id; widths: matching list of
        (W1, W2) (the caller tracks them: leaf length or an earlier merge's path length).  Consumes resident
        children.  Returns (merged ids, list of dict(path, total, last, swapped, variant))."""
        n = len(merges)
        arr = (ProfMerge * max(n, 1))()
        for k, (a, b) in enumerate(merges):
            arr[k] = ProfMerge(int(a), int(b))
        cap = int(sum(w1 + w2 for w1, w2 in widths))
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        res = (DpResult * max(n, 1))()
        path = np.zeros(max(cap, 1), dtype=np.uint8)
        ids = np.zeros(max(n, 1), dtype=np.uint32)
        self._check(self.lib.famsa_prof_merge_batch(self.h, C.byref(arr), n, _ptr(g), _ptr(ids), C.byref(res), _ptr(path), cap))
        out = []
        for k in range(n):
            r = res[k]
            out.append(dict(path=path[r.path_offset:r.path_offset + r.path_len].copy(), total=int(r.total_score),
                            last=np.array(list(r.last), dtype=np.int64), swapped=bool(r.swapped), variant=int(r.variant)))
        return [int(x) for x in ids[:n]], out

    def align_tree(self, merges, gaps, want_paths: bool = True):
        """famsa_prof_align_tree: the whole progressive alignment of the uploaded sequences along a guide tree in one
        call.  merges: (n-1, 2) child node ids (leaves 0..n-1, internal node n+k = merges[k]).  Returns
        (root id, [dict(path, total, last, swapped, variant, rows_width, cols_width) per merge], stats dict)."""
        t = np.ascontiguousarray(merges, dtype=np.int32).reshape(-1, 2)
        n = len(t)
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        res = (DpResult * max(n, 1))()
        root, nbytes = C.c_uint32(), C.c_uint64()
        st = TreeStats()
        self._tree_width = None                                     # the kept tree is replaced, or gone if the call fails
        self._check(self.lib.famsa_prof_align_tree(self.h, _ptr(t), n + 1, _ptr(g), C.byref(res), C.byref(root), C.byref(nbytes),
                                                   C.byref(st)))
        stats = {f: getattr(st, f) for f, _ in TreeStats._fields_ if f != "pad"}
        self._tree_width = int(res[n - 1].path_len)
        out = []
        if want_paths:
            path = np.zeros(max(nbytes.value, 1), dtype=np.uint8)
            self._check(self.lib.famsa_prof_tree_paths(self.h, _ptr(path), path.size))
            for k in range(n):
                r = res[k]
                out.append(dict(path=path[r.path_offset:r.path_offset + r.path_len].copy(), total=int(r.total_score),
                                last=np.array(list(r.last), dtype=np.int64), swapped=bool(r.swapped), variant=int(r.variant),
                                rows_width=int(r.rows_width), cols_width=int(r.cols_width)))
        return root.value, out, stats

    def align_tree_buffers(self, merges, gaps, stats_of_a_run):
        """Prebuilt arguments of famsa_prof_align_tree / famsa_prof_tree_paths (what a C caller holds), sized from an
        earlier run of the same tree: for align_tree_raw."""
        t = np.ascontiguousarray(merges, dtype=np.int32).reshape(-1, 2)
        n = len(t)
        nbytes = C.c_uint64()
        res = (DpResult * max(n, 1))()
        root = C.c_uint32()
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        st = TreeStats()
        self._tree_width = None
        self._check(self.lib.famsa_prof_align_tree(self.h, _ptr(t), n + 1, _ptr(g), C.byref(res), C.byref(root), C.byref(nbytes), C.byref(st)))
        self._tree_width = int(res[n - 1].path_len)
        self.prof_drop([root.value])
        return dict(tree=t, n=n, gaps=g, res=res, path=np.zeros(max(int(nbytes.value) * 2, 1), dtype=np.uint8))

    def align_tree_raw(self, b):
        """The two C calls on prebuilt buffers, without this binding's per-merge Python objects.  Returns (root id, stats)."""
        root, nbytes = C.c_uint32(), C.c_uint64()
        st = TreeStats()
        self._tree_width = None
        self._check(self.lib.famsa_prof_align_tree(self.h, _ptr(b["tree"]), b["n"] + 1, _ptr(b["gaps"]), C.byref(b["res"]), C.byref(root),
                                                   C.byref(nbytes), C.byref(st)))
        self._tree_width = int(b["res"][b["n"] - 1].path_len)
        self._check(self.lib.famsa_prof_tree_paths(self.h, _ptr(b["path"]), b["path"].size))
        return root.value, {f: getattr(st, f) for f, _ in TreeStats._fields_ if f != "pad"}

    def tree_rows(self, order=None, download: bool = True):
        """famsa_prof_tree_rows: the final alignment of the last align_tree, built on the device -- (n, W) uint8 codes with
        GAP = 30, row k = leaf order[k] (order None: leaf k).  The rows stay on the device for refine(root, rows=None);
        download=False leaves them there only and returns None."""
        o = None if order is None else np.ascontiguousarray(order, dtype=np.uint32)
        n = self.n if o is None else len(o)
        w = C.c_uint32()
        if not download:
            self._check(self.lib.famsa_prof_tree_rows(self.h, _ptr(o), n, None, 0, C.byref(w)))
            self._tree_rows_shape = (n, w.value)
            return None
        width = getattr(self, "_tree_width", None)
        if width is not None:               # W_root of the tree align_tree ran
            out = np.zeros((n, width), dtype=np.uint8)
            rc = self.lib.famsa_prof_tree_rows(self.h, _ptr(o), n, _ptr(out), out.size, C.byref(w))
            if rc == 0 and w.value == width:
                self._tree_rows_shape = (n, width)
                return out
        # a tree this binding did not run (or one run behind its back): one device-only call to learn W_root
        self._check(self.lib.famsa_prof_tree_rows(self.h, _ptr(o), n, None, 0, C.byref(w)))
        self._tree_width = width = w.value
        out = np.zeros((n, width), dtype=np.uint8)
        self._check(self.lib.famsa_prof_tree_rows(self.h, _ptr(o), n, _ptr(out), out.size, C.byref(w)))
        self._tree_rows_shape = (n, w.value)
        return out

    def refine(self, root_id: int, rows=None, gaps=None, n_refinements: int = 100, flags: int = 0):
        """famsa_prof_refine: RefineAlignment of the resident root (consumed) whose alignment is `rows` (n x width codes,
        GAP = 30, rows sorted by FASTA id); rows None: the rows the last tree_rows() kept on the device (FAMSA_REFINE_TREE_ROWS,
        built in id order).  Returns (refined rows, width, total score, stats dict, refined profile id); stats also holds
        `kernel_launches`, the launches of the call."""
        if gaps is None:
            raise ValueError("gaps are required")
        g = np.ascontiguousarray(gaps, dtype=np.int64)
        if rows is None:
            r, (n_rows, width) = None, getattr(self, "_tree_rows_shape", (0, 0))
            flags |= REFINE_TREE_ROWS
        else:
            r = np.ascontiguousarray(rows, dtype=np.uint8)
            n_rows, width = r.shape
        rid, w, tot = C.c_uint32(), C.c_uint32(), C.c_int64()
        st = RefineStats()
        l0 = self.kernel_launches()
        self._check(self.lib.famsa_prof_refine(self.h, root_id, _ptr(r), n_rows, width, _ptr(g), n_refinements, flags,
                                               C.byref(rid), C.byref(w), C.byref(tot), C.byref(st)))
        stats = {f: getattr(st, f) for f, _ in RefineStats._fields_}
        stats["kernel_launches"] = self.kernel_launches() - l0
        out = np.zeros((n_rows, w.value), dtype=np.uint8)
        self._check(self.lib.famsa_prof_refined_rows(self.h, _ptr(out), out.size))
        return out, w.value, tot.value, stats, rid.value

    def prof_get(self, pid: int, tables: bool = True):
        """(scores, counters, card) of a resident profile, or (width, card) with tables=False."""
        w, k = C.c_uint32(), C.c_uint32()
        self._check(self.lib.famsa_prof_get(self.h, pid, C.byref(w), C.byref(k), None, None))
        if not tables:
            return w.value, k.value
        s = np.zeros((w.value + 1, 32), dtype=np.int64); c = np.zeros((w.value + 1, 32), dtype=np.int32)
        self._check(self.lib.famsa_prof_get(self.h, pid, None, None, _ptr(s), _ptr(c)))
        return s, c, k.value

    def prof_drop(self, ids):
        a = np.ascontiguousarray(ids, dtype=np.uint32)
        self._check(self.lib.famsa_prof_drop(self.h, _ptr(a), len(a)))

    def prof_last_timing(self) -> tuple[float, float]:
        t, m = C.c_float(), C.c_float()
        self._check(self.lib.famsa_prof_last_timing(self.h, C.byref(t), C.byref(m)))
        return t.value, m.value

    def prof_stats(self) -> tuple[int, int]:
        a, b = C.c_uint64(), C.c_uint64()
        self._check(self.lib.famsa_prof_stats(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def dp_last_timing(self) -> tuple[float, float, int]:
        t, m, p = C.c_float(), C.c_float(), C.c_uint64()
        self._check(self.lib.famsa_dp_last_timing(self.h, C.byref(t), C.byref(m), C.byref(p)))
        return t.value, m.value, p.value

    def last_timing(self) -> tuple[float, float, int]:
        t, m, p = C.c_float(), C.c_float(), C.c_uint64()
        self._check(self.lib.famsa_lcs_last_timing(self.h, C.byref(t), C.byref(m), C.byref(p)))
        return t.value, m.value, p.value

    def kernel_launches(self) -> int:
        return int(self.lib.famsa_kernel_launches(self.h))

    def transform(self, kind: int, lcs: int, len1: int, len2: int, double: bool = True) -> float:
        f = self.lib.famsa_transform_f64 if double else self.lib.famsa_transform_f32
        return float(f(kind, lcs, len1, len2))
