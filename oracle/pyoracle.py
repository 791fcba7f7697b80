"""ctypes access to the checkers: the only module that opens one of their libraries.

  oracle/liboracle.so, oracle/libnj_oracle.so   our C restatements (oracle/*_oracle.c)
  oracle/_ref/libfamsa_ref*.so                  the unmodified reference behind oracle/ref_*harness.cpp

lib(name) opens a library of LIBS once; have(name, symbol) says whether it is there and has an entry point.  The wrappers
of liboracle.so and libfamsa_ref.so live here; tests/{nj,slink,dist_export,refine}_oracle.py wrap the others.

TEST INFRASTRUCTURE ONLY -- importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never from famsa_b200/.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

vp, cp, i32, u32, i64, u64 = C.c_void_p, C.c_char_p, C.c_int, C.c_uint32, C.c_int64, C.c_uint64
f32, f64 = C.c_float, C.c_double

# name: (file under oracle/, built on demand by `make -C oracle` when missing, {entry point: (restype, argtypes)}).
# Only oracle/Makefile builds the _ref/ libraries, and only where the reference's sources are.
LIBS = {
    "oracle": ("liboracle.so", True, {
        "lcs_oracle_rows": (None, [vp, vp, vp, vp, u32, vp, u32, vp]),
        "lcs_oracle_triangle": (None, [vp, vp, vp, u32, u32, vp]),
        "lcs_oracle_transform_f64": (f64, [i32, u32, u32, u32]),
        "lcs_oracle_transform_f32": (f32, [i32, u32, u32, u32]),
        "lcs_oracle_transform_tri_f32": (None, [i32, vp, i32, vp, u32, vp]),
        "upgma_oracle_tree": (i32, [vp, u32, i32, i32, i32, vp, vp]),
        "dp_oracle_align": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "dp_oracle_construct": (i32, [vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]),
    }),
    "nj_oracle": ("libnj_oracle.so", True, {
        "nj_oracle_tree": (i32, [vp, u32, vp, vp]),
    }),
    "ref": ("_ref/libfamsa_ref.so", False, {
        "ref_seqset_create": (vp, [vp, u32]),
        "ref_seqset_destroy": (None, [vp]),
        "ref_seqset_len": (u32, [vp, u32]),
        "ref_seqset_codes": (None, [vp, u32, vp]),
        "ref_lcs_row_prefix": (None, [vp, u32, u32, vp, i32]),
        "ref_lcs_row_ids": (None, [vp, u32, vp, u32, vp, i32]),
        "ref_lcs_triangle_mt": (f64, [vp, u32, u32, i32, i32, vp, vp]),
        "ref_mst_prim_tree": (None, [vp, i32, vp]),
        "ref_mst_to_dendogram": (None, [i32, vp, vp, vp, vp, vp]),
        "ref_upgma_tree": (None, [vp, i32, i32, vp]),
        "ref_upgma_tree_from_distances": (None, [vp, i32, i32, vp]),
        "ref_transform_f64": (f64, [i32, u32, u32, u32]),
        "ref_transform_f32": (f32, [i32, u32, u32, u32]),
        "ref_dp_create": (vp, [i32, i32, i32]),
        "ref_dp_destroy": (None, [vp]),
        "ref_dp_gaps": (None, [vp, vp]),
        "ref_dp_set_gaps": (None, [vp, vp]),
        "ref_dp_score_matrix": (None, [vp, vp]),
        "ref_profile_create": (vp, [vp, vp, vp, u32]),
        "ref_profile_leaf": (vp, [vp, cp, i32]),
        "ref_profile_destroy": (None, [vp]),
        "ref_profile_width": (u32, [vp]),
        "ref_profile_card": (u32, [vp]),
        "ref_profile_total_score": (i64, [vp]),
        "ref_profile_tables": (None, [vp, vp, vp]),
        "ref_profile_set_scores": (None, [vp, vp]),
        "ref_profile_row": (i32, [vp, u32, vp]),
        "ref_profile_align": (vp, [vp, vp, vp, i32]),
        "ref_profile_construct": (vp, [vp, vp, vp, vp, vp, i32]),
        "ref_dp_align_pairs_mt": (f64, [vp, vp, vp, u32, i32, vp]),
        "ref_align_tree_mt": (f64, [vp, vp, u32, vp, i32, vp, vp, vp, vp, u32]),
    }),
    "ref_dist": ("_ref/libfamsa_ref_dist.so", False, {
        "ref_dist_export": (i32, [vp, vp, u32, i32, i32, i32, cp, i32]),
        "ref_num2str_f32": (u64, [vp, u64, vp]),
    }),
    "ref_slink": ("_ref/libfamsa_ref_slink.so", False, {
        "ref_slink_tree": (i32, [vp, u32, i32, i32, vp]),
    }),
    "ref_nj": ("_ref/libfamsa_ref_nj.so", False, {
        "ref_nj_tree": (i32, [vp, u32, i32, vp, vp]),
        "ref_nj_tree_from_distances": (i32, [vp, i32, i32, vp]),
    }),
    "ref_refine": ("_ref/libfamsa_ref_refine.so", False, {
        "rr_create": (vp, [vp, vp, i32, i32]),
        "rr_destroy": (None, [vp]),
        "rr_total_score": (i64, [vp, vp, u32]),
        "rr_optimize_gaps": (None, [vp, vp, u32, cp]),
        "rr_align_refine": (None, [vp, vp, vp, u32, vp, u32, cp, cp, u32, vp, vp, vp, vp, u32, vp, vp]),
        "rr_refine_rows": (None, [vp, vp, vp, u32, u32, cp, u32, vp, vp, vp, vp, u32, vp, vp]),
    }),
}
_libs: dict[str, C.CDLL] = {}


def _path(name: str) -> str:
    return os.path.join(_HERE, LIBS[name][0])


def lib(name: str) -> C.CDLL:
    """The library LIBS[name], opened once.  A _ref/ library carried over from a build of an older revision (where the
    reference's sources could not be read to rebuild it) may lack newer entry points: only those the file exports are
    declared, and have(name, symbol) tells which."""
    if name not in _libs:
        _, on_demand, entry_points = LIBS[name]
        if on_demand and not os.path.exists(_path(name)):
            subprocess.run(["make", "-C", _HERE, "-j8", "all"], check=True, stdout=subprocess.DEVNULL)
        dll = C.CDLL(_path(name))
        for symbol, (restype, argtypes) in entry_points.items():
            if hasattr(dll, symbol):
                getattr(dll, symbol).restype = restype
                getattr(dll, symbol).argtypes = argtypes
        _libs[name] = dll
    return _libs[name]


def have(name: str, symbol: str | None = None) -> bool:
    """Whether the file of LIBS[name] is there and, given `symbol`, exports that entry point."""
    return os.path.exists(_path(name)) and (symbol is None or hasattr(lib(name), symbol))


def have_ref() -> bool:
    return have("ref")


def have_ref_set_scores() -> bool:
    """Is the reference library built with ref_profile_set_scores (RefDp.set_scores)?"""
    return have("ref", "ref_profile_set_scores")


def ref() -> C.CDLL:
    return lib("ref")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class DpProfile(C.Structure):
    _fields_ = [("scores", C.c_void_p), ("counters", C.c_void_p), ("width", C.c_uint32), ("card", C.c_uint32)]


def dp_align(scores1, counters1, card1, scores2, counters2, card2, gaps, score_matrix=None):
    """Oracle version of CProfile::Align + traceback.  scores: (W+1,32) int64, counters: (W+1,32) int32.
    Returns dict(path uint8[], total, last(3), swapped, variant, dirs (WR+1, WC+1) uint8)."""
    dll = lib("oracle")
    s1 = np.ascontiguousarray(scores1, dtype=np.int64); c1 = np.ascontiguousarray(counters1, dtype=np.int32)
    s2 = np.ascontiguousarray(scores2, dtype=np.int64); c2 = np.ascontiguousarray(counters2, dtype=np.int32)
    w1, w2 = s1.shape[0] - 1, s2.shape[0] - 1
    p1 = DpProfile(s1.ctypes.data, c1.ctypes.data, w1, card1)
    p2 = DpProfile(s2.ctypes.data, c2.ctypes.data, w2, card2)
    g = np.ascontiguousarray(gaps, dtype=np.int64)
    sm = None if score_matrix is None else np.ascontiguousarray(score_matrix, dtype=np.int64)
    dirs = np.zeros((w1 + 1) * (w2 + 1), dtype=np.uint8)
    path = np.zeros(w1 + w2 + 1, dtype=np.uint8)
    plen = C.c_uint32(); total = C.c_int64(); sw = C.c_int(); var = C.c_int()
    last = np.zeros(3, dtype=np.int64)
    dll.dp_oracle_align(C.byref(p1), C.byref(p2), _p(g), _p(sm), _p(dirs), _p(path), C.byref(plen), _p(last),
                        C.byref(total), C.byref(sw), C.byref(var))
    wr, wc = (w2, w1) if sw.value else (w1, w2)
    return dict(path=path[:plen.value].copy(), total=total.value, last=last, swapped=bool(sw.value),
                variant=var.value, dirs=dirs.reshape(wr + 1, wc + 1))


def dp_construct(rows_prof, cols_prof, path, gaps):
    """Oracle version of ConstructProfile's merge part.  rows_prof / cols_prof = (scores, counters, card) of the
    DP matrix's row / column profile (i.e. after the orientation swap); path = forward direction bytes.
    Returns (scores (W+1,32) int64, counters (W+1,32) int32, gap runs of the row profile's members (m,2),
    gap runs of the column profile's members (m,2)) -- runs are (first merged column, length)."""
    dll = lib("oracle")
    s1 = np.ascontiguousarray(rows_prof[0], dtype=np.int64); c1 = np.ascontiguousarray(rows_prof[1], dtype=np.int32)
    s2 = np.ascontiguousarray(cols_prof[0], dtype=np.int64); c2 = np.ascontiguousarray(cols_prof[1], dtype=np.int32)
    p1 = DpProfile(s1.ctypes.data, c1.ctypes.data, s1.shape[0] - 1, int(rows_prof[2]))
    p2 = DpProfile(s2.ctypes.data, c2.ctypes.data, s2.shape[0] - 1, int(cols_prof[2]))
    path = np.ascontiguousarray(path, dtype=np.uint8)
    w = len(path)
    g = np.ascontiguousarray(gaps, dtype=np.int64)
    os_ = np.zeros((w + 1, 32), dtype=np.int64); oc = np.zeros((w + 1, 32), dtype=np.int32)
    g1 = np.zeros((max(w, 1), 2), dtype=np.uint32); g2 = np.zeros((max(w, 1), 2), dtype=np.uint32)
    n1 = C.c_uint32(); n2 = C.c_uint32()
    rc = dll.dp_oracle_construct(C.byref(p1), C.byref(p2), _p(path), w, _p(g), _p(os_), _p(oc), _p(g1), C.byref(n1),
                                 _p(g2), C.byref(n2))
    if rc:
        raise ValueError(f"dp_oracle_construct: path does not span the two profiles (rc={rc})")
    return os_, oc, g1[:n1.value].copy(), g2[:n2.value].copy()


def lcs_rows(codes, offsets, lens, ref_ids, col_ids=None, n_col=None) -> np.ndarray:
    dll = lib("oracle")
    ref = np.ascontiguousarray(ref_ids, dtype=np.uint32)
    cols = None if col_ids is None else np.ascontiguousarray(col_ids, dtype=np.uint32)
    n_col = (len(lens) if n_col is None else n_col) if cols is None else len(cols)
    out = np.zeros(max(len(ref) * n_col, 1), dtype=np.uint32)
    dll.lcs_oracle_rows(_p(codes), _p(offsets), _p(lens), _p(ref), len(ref), _p(cols), n_col, _p(out))
    return out[:len(ref) * n_col].reshape(len(ref), n_col)


def lcs_triangle(codes, offsets, lens, row_begin=0, row_end=None) -> np.ndarray:
    dll = lib("oracle")
    row_end = len(lens) if row_end is None else row_end
    f = lambda r: r * (r - 1) // 2 if r else 0
    size = f(row_end) - f(row_begin)
    out = np.zeros(max(size, 1), dtype=np.uint32)
    dll.lcs_oracle_triangle(_p(codes), _p(offsets), _p(lens), row_begin, row_end, _p(out))
    return out[:size]


def transform(kind: int, lcs: int, len1: int, len2: int, double=True) -> float:
    dll = lib("oracle")
    return float((dll.lcs_oracle_transform_f64 if double else dll.lcs_oracle_transform_f32)(kind, lcs, len1, len2))


def transform_triangle(kind: int, lcs_tri: np.ndarray, lens) -> np.ndarray:
    """transform(kind, ..., double=False) of every pair of a packed LCS triangle (uint16 or uint32, row i at i(i-1)/2,
    row i = seq0): the float distance triangle UPGMA's computeDistances fills."""
    t = np.ascontiguousarray(lcs_tri)
    if t.dtype not in (np.uint16, np.uint32):
        t = t.astype(np.uint32)
    ln = np.ascontiguousarray(lens, dtype=np.uint32)
    n = len(ln)
    assert t.size == n * (n - 1) // 2
    out = np.empty(max(t.size, 1), dtype=np.float32)
    lib("oracle").lcs_oracle_transform_tri_f32(kind, _p(t), t.dtype.itemsize, _p(ln), n, _p(out))
    return out[:t.size]


UPGMA_AVG_AS_REFERENCE, UPGMA_AVG_ROUNDED_ONCE, UPGMA_AVG_FUSED = 0, 1, 2


def upgma_tree(dist_tri: np.ndarray, n: int, modified: bool = False, avg_mode: int = UPGMA_AVG_AS_REFERENCE,
               fresh_cache: bool = False, overwrite: bool = False):
    """The restated UPGMA<>::computeTree (oracle/upgma_oracle.c) on a float distance triangle, left untouched unless
    `overwrite` (then a float32 array is averaged in place, as the reference does, which saves a copy of a large one).
    Returns (status, merges): status 0 with the n-1 merges as (n-1, 2) int32, or 1 (no finite distance left) with the
    merges made before that.  avg_mode / fresh_cache select the variants that only witness generation uses."""
    ok_in_place = overwrite and isinstance(dist_tri, np.ndarray) and dist_tri.dtype == np.float32 and dist_tri.flags.c_contiguous
    d = dist_tri if ok_in_place else np.array(dist_tri, dtype=np.float32, copy=True)
    assert d.size == n * (n - 1) // 2
    out = np.zeros((max(n - 1, 1), 2), dtype=np.int32)
    done = C.c_uint32()
    rc = lib("oracle").upgma_oracle_tree(_p(d), n, int(modified), avg_mode, int(fresh_cache), _p(out), C.byref(done))
    return rc, out[:done.value]


# ------------------------------------------------------------------ the real reference
def mst_to_dendogram(edge_from, edge_to, edge_dist, prim_orders) -> np.ndarray:
    """The reference's own mst_to_dendogram on external MST edges (Prim order)."""
    n = len(prim_orders)
    f = np.ascontiguousarray(edge_from, dtype=np.int32); t = np.ascontiguousarray(edge_to, dtype=np.int32)
    d = np.ascontiguousarray(edge_dist, dtype=np.float64); o = np.ascontiguousarray(prim_orders, dtype=np.int32)
    out = np.zeros((2 * n - 1, 2), dtype=np.int32)
    lib("ref").ref_mst_to_dendogram(n, _p(f), _p(t), _p(d), _p(o), _p(out))
    return out


def upgma_tree_from_distances(tri: np.ndarray, n: int, modified: bool = False) -> np.ndarray:
    """The reference's UPGMA agglomeration (computeTree) on an external float distance triangle."""
    t = np.ascontiguousarray(tri, dtype=np.float32)
    out = np.zeros((2 * n - 1, 2), dtype=np.int32)
    lib("ref").ref_upgma_tree_from_distances(_p(t), n, int(modified), _p(out))
    return out


class RefDp:
    """The reference's CProfile machinery behind oracle/ref_harness.cpp."""

    def __init__(self, n_seqs_for_rescale: int = 0, matrix_type: int = 2, pool_threads: int = 2):
        self.lib = lib("ref")
        self.h = C.c_void_p(self.lib.ref_dp_create(n_seqs_for_rescale, matrix_type, pool_threads))

    def close(self):
        if self.h:
            self.lib.ref_dp_destroy(self.h)
            self.h = None

    def gaps(self) -> np.ndarray:
        g = np.zeros(4, dtype=np.int64)
        self.lib.ref_dp_gaps(self.h, _p(g))
        return g

    def set_gaps(self, g):
        g = np.ascontiguousarray(g, dtype=np.int64)
        self.lib.ref_dp_set_gaps(self.h, _p(g))

    def score_matrix(self) -> np.ndarray:
        m = np.zeros((24, 24), dtype=np.int64)
        self.lib.ref_dp_score_matrix(self.h, _p(m))
        return m

    def profile(self, gapped: list[str], seq_nos: list[int]):
        arr = (C.c_char_p * len(gapped))(*[s.encode("ascii") for s in gapped])
        nos = np.ascontiguousarray(seq_nos, dtype=np.int32)
        return C.c_void_p(self.lib.ref_profile_create(self.h, arr, _p(nos), len(gapped)))

    def leaf(self, letters: str, seq_no: int):
        return C.c_void_p(self.lib.ref_profile_leaf(self.h, letters.encode("ascii"), seq_no))

    def free(self, p):
        self.lib.ref_profile_destroy(p)

    def tables(self, p):
        w = self.lib.ref_profile_width(p)
        sc = np.zeros((w + 1, 32), dtype=np.int64)
        cn = np.zeros((w + 1, 32), dtype=np.int32)
        self.lib.ref_profile_tables(p, _p(sc), _p(cn))
        return sc, cn, int(self.lib.ref_profile_card(p))

    def set_scores(self, p, scores: np.ndarray):
        """Replaces the profile's score table (counters untouched): Align then runs on the given scores."""
        w = self.lib.ref_profile_width(p)
        s = np.ascontiguousarray(scores, dtype=np.int64)
        assert s.shape == (w + 1, 32)
        self.lib.ref_profile_set_scores(p, _p(s))

    def rows(self, p) -> dict[int, str]:
        w = self.lib.ref_profile_width(p)
        out = {}
        buf = C.create_string_buffer(w + 2)
        for i in range(self.lib.ref_profile_card(p)):
            no = self.lib.ref_profile_row(p, i, buf)
            out[no] = buf.value.decode()
        return out

    def construct(self, p1, p2, dirs: np.ndarray, last, swapped: bool):
        """The reference's ConstructProfile on an externally produced direction matrix.  Consumes p1, p2."""
        d = np.ascontiguousarray(dirs, dtype=np.uint8)
        l = np.ascontiguousarray(last, dtype=np.int64)
        m = C.c_void_p(self.lib.ref_profile_construct(self.h, p1, p2, _p(d), _p(l), int(swapped)))
        self.lib.ref_profile_destroy(p1)
        self.lib.ref_profile_destroy(p2)
        return m

    def align_pairs_mt(self, p1s, p2s, n_threads: int):
        """Times len(p1s) independent merges on n_threads threads; consumes the profiles."""
        n = len(p1s)
        a = (C.c_void_p * n)(*[p.value for p in p1s])
        b = (C.c_void_p * n)(*[p.value for p in p2s])
        cells = C.c_uint64()
        sec = self.lib.ref_dp_align_pairs_mt(self.h, a, b, n, n_threads, C.byref(cells))
        return sec, cells.value

    def align_tree_mt(self, seqs: list[str], merges, n_threads: int, want_rows: bool = False):
        """The reference's whole ComputeAlignment (CProfileQueue + worker threads) over a guide tree.  merges: (n-1, 2)
        child ids of the internal nodes.  Returns (seconds, cells, total score, width[, {seq_no: gapped row}])."""
        n = len(seqs)
        arr = (C.c_char_p * n)(*[s.encode("ascii") for s in seqs])
        tree = np.full((2 * n - 1, 2), -1, dtype=np.int32)
        tree[n:] = np.asarray(merges, dtype=np.int32).reshape(-1, 2)
        cells, total, width = C.c_uint64(), C.c_int64(), C.c_uint32()
        stride = int(sum(len(s) for s in seqs)) + 1 if want_rows else 0
        stride = min(stride, 1 << 20)
        rows = np.zeros(n * stride, dtype=np.uint8) if want_rows else None
        sec = self.lib.ref_align_tree_mt(self.h, arr, n, _p(tree), n_threads, C.byref(cells), C.byref(total), C.byref(width),
                                         _p(rows), stride)
        out = (sec, cells.value, total.value, width.value)
        if want_rows:
            out += ({i: bytes(rows[i * stride:i * stride + width.value]).decode() for i in range(n)},)
        return out

    def align(self, p1, p2, no_threads: int = 1):
        """Returns (merged profile handle, total_score).  p1 and p2 are consumed and freed."""
        m = C.c_void_p(self.lib.ref_profile_align(self.h, p1, p2, no_threads))
        self.lib.ref_profile_destroy(p1)
        self.lib.ref_profile_destroy(p2)
        return m, int(self.lib.ref_profile_total_score(m))


def path_from_rows(rows: dict[int, str], members1: set, members2: set, swapped: bool) -> np.ndarray:
    """Reconstruct the traceback path (0 D, 1 H, 2 V in (row profile, column profile) terms) from
    the merged alignment: every child column holds at least one residue."""
    width = len(next(iter(rows.values())))
    in1 = np.zeros(width, dtype=bool)
    in2 = np.zeros(width, dtype=bool)
    for no, s in rows.items():
        a = np.frombuffer(s.encode(), dtype=np.uint8) != ord("-")
        if no in members1:
            in1 |= a
        else:
            in2 |= a
    inr, inc = (in2, in1) if swapped else (in1, in2)
    assert np.all(inr | inc)
    return np.where(inr & inc, 0, np.where(inc, 1, 2)).astype(np.uint8)


class RefSeqSet:
    """A set of CSequence objects inside the reference, built from residue letters."""

    def __init__(self, letters: list[str]):
        self.lib = lib("ref")
        arr = (C.c_char_p * len(letters))(*[s.encode("ascii") for s in letters])
        self.n = len(letters)
        self.h = C.c_void_p(self.lib.ref_seqset_create(arr, self.n))

    def close(self):
        if self.h:
            self.lib.ref_seqset_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def codes(self) -> list[np.ndarray]:
        out = []
        for i in range(self.n):
            ln = self.lib.ref_seqset_len(self.h, i)
            a = np.zeros(max(ln, 1), dtype=np.int8)
            self.lib.ref_seqset_codes(self.h, i, _p(a))
            out.append(a[:ln])
        return out

    def row_prefix(self, ref_id: int, n_cols: int, isa: int = 2) -> np.ndarray:
        out = np.zeros(max(n_cols, 1), dtype=np.uint32)
        self.lib.ref_lcs_row_prefix(self.h, ref_id, n_cols, _p(out), isa)
        return out[:n_cols]

    def row_ids(self, ref_id: int, ids, isa: int = 2) -> np.ndarray:
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.zeros(max(len(ids), 1), dtype=np.uint32)
        self.lib.ref_lcs_row_ids(self.h, ref_id, _p(ids), len(ids), _p(out), isa)
        return out[:len(ids)]

    def mst_prim_tree(self, n_threads: int = 2) -> np.ndarray:
        """The reference's default (-gt sl) guide tree of this set: (2n-1, 2) child ids."""
        out = np.zeros((2 * self.n - 1, 2), dtype=np.int32)
        self.lib.ref_mst_prim_tree(self.h, n_threads, _p(out))
        return out

    def upgma_tree(self, modified: bool = False, n_threads: int = 2) -> np.ndarray:
        """The reference's UPGMA guide tree of this set: (2n-1, 2) child ids, leaves are (-1, -1)."""
        out = np.zeros((2 * self.n - 1, 2), dtype=np.int32)
        self.lib.ref_upgma_tree(self.h, int(modified), n_threads, _p(out))
        return out

    def triangle_mt(self, row_begin: int, row_end: int, n_threads: int, isa: int = 2, want_lcs: bool = False):
        f = lambda r: r * (r - 1) // 2 if r else 0
        out = np.zeros(max(f(row_end) - f(row_begin), 1), dtype=np.uint32) if want_lcs else None
        pairs = C.c_uint64()
        sec = self.lib.ref_lcs_triangle_mt(self.h, row_begin, row_end, n_threads, isa, _p(out), C.byref(pairs))
        return sec, pairs.value, (out[:f(row_end) - f(row_begin)] if want_lcs else None)
