"""ctypes access to the checkers: oracle/liboracle.so (our C restatement) and
oracle/_ref/libfamsa_ref.so (the unmodified reference behind oracle/ref_harness.cpp).

TEST INFRASTRUCTURE ONLY -- importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never from famsa_b200/.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "liboracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libfamsa_ref.so")


def build(quiet: bool = True):
    """(Re)build the checkers: liboracle.so always, _ref only where /root/reference exists."""
    subprocess.run(["make", "-C", _HERE, "-j8", "all"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


_oracle = None


def oracle() -> C.CDLL:
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_SO):
            build()
        lib = C.CDLL(ORACLE_SO)
        vp, u32 = C.c_void_p, C.c_uint32
        lib.lcs_oracle_rows.argtypes = [vp, vp, vp, vp, u32, vp, u32, vp]
        lib.lcs_oracle_triangle.argtypes = [vp, vp, vp, u32, u32, vp]
        lib.lcs_oracle_transform_f64.argtypes = [C.c_int, u32, u32, u32]
        lib.lcs_oracle_transform_f64.restype = C.c_double
        lib.lcs_oracle_transform_f32.argtypes = [C.c_int, u32, u32, u32]
        lib.lcs_oracle_transform_f32.restype = C.c_float
        lib.lcs_oracle_transform_tri_f32.argtypes = [C.c_int, vp, C.c_int, vp, u32, vp]
        lib.upgma_oracle_tree.argtypes = [vp, u32, C.c_int, C.c_int, C.c_int, vp, vp]
        lib.upgma_oracle_tree.restype = C.c_int
        lib.dp_oracle_align.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.dp_oracle_construct.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
        _oracle = lib
    return _oracle


class DpProfile(C.Structure):
    _fields_ = [("scores", C.c_void_p), ("counters", C.c_void_p), ("width", C.c_uint32), ("card", C.c_uint32)]


def dp_align(scores1, counters1, card1, scores2, counters2, card2, gaps, score_matrix=None):
    """Oracle version of CProfile::Align + traceback.  scores: (W+1,32) int64, counters: (W+1,32) int32.
    Returns dict(path uint8[], total, last(3), swapped, variant, dirs (WR+1, WC+1) uint8)."""
    lib = oracle()
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
    lib.dp_oracle_align(C.byref(p1), C.byref(p2), _p(g), _p(sm), _p(dirs), _p(path), C.byref(plen), _p(last),
                        C.byref(total), C.byref(sw), C.byref(var))
    wr, wc = (w2, w1) if sw.value else (w1, w2)
    return dict(path=path[:plen.value].copy(), total=total.value, last=last, swapped=bool(sw.value),
                variant=var.value, dirs=dirs.reshape(wr + 1, wc + 1))


def dp_construct(rows_prof, cols_prof, path, gaps):
    """Oracle version of ConstructProfile's merge part.  rows_prof / cols_prof = (scores, counters, card) of the
    DP matrix's row / column profile (i.e. after the orientation swap); path = forward direction bytes.
    Returns (scores (W+1,32) int64, counters (W+1,32) int32, gap runs of the row profile's members (m,2),
    gap runs of the column profile's members (m,2)) -- runs are (first merged column, length)."""
    lib = oracle()
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
    rc = lib.dp_oracle_construct(C.byref(p1), C.byref(p2), _p(path), w, _p(g), _p(os_), _p(oc), _p(g1), C.byref(n1),
                                 _p(g2), C.byref(n2))
    if rc:
        raise ValueError(f"dp_oracle_construct: path does not span the two profiles (rc={rc})")
    return os_, oc, g1[:n1.value].copy(), g2[:n2.value].copy()


def lcs_rows(codes, offsets, lens, ref_ids, col_ids=None, n_col=None) -> np.ndarray:
    lib = oracle()
    ref = np.ascontiguousarray(ref_ids, dtype=np.uint32)
    cols = None if col_ids is None else np.ascontiguousarray(col_ids, dtype=np.uint32)
    n_col = (len(lens) if n_col is None else n_col) if cols is None else len(cols)
    out = np.zeros(max(len(ref) * n_col, 1), dtype=np.uint32)
    lib.lcs_oracle_rows(_p(codes), _p(offsets), _p(lens), _p(ref), len(ref), _p(cols), n_col, _p(out))
    return out[:len(ref) * n_col].reshape(len(ref), n_col)


def lcs_triangle(codes, offsets, lens, row_begin=0, row_end=None) -> np.ndarray:
    lib = oracle()
    row_end = len(lens) if row_end is None else row_end
    f = lambda r: r * (r - 1) // 2 if r else 0
    size = f(row_end) - f(row_begin)
    out = np.zeros(max(size, 1), dtype=np.uint32)
    lib.lcs_oracle_triangle(_p(codes), _p(offsets), _p(lens), row_begin, row_end, _p(out))
    return out[:size]


def transform(kind: int, lcs: int, len1: int, len2: int, double=True) -> float:
    lib = oracle()
    return float((lib.lcs_oracle_transform_f64 if double else lib.lcs_oracle_transform_f32)(kind, lcs, len1, len2))


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
    oracle().lcs_oracle_transform_tri_f32(kind, _p(t), t.dtype.itemsize, _p(ln), n, _p(out))
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
    rc = oracle().upgma_oracle_tree(_p(d), n, int(modified), avg_mode, int(fresh_cache), _p(out), C.byref(done))
    return rc, out[:done.value]


# ------------------------------------------------------------------ the real reference
_ref = None


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def have_ref_set_scores() -> bool:
    """Is the reference library built with ref_profile_set_scores (RefDp.set_scores)?"""
    return have_ref() and hasattr(ref(), "ref_profile_set_scores")


def ref() -> C.CDLL:
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_SO)
        vp, u32 = C.c_void_p, C.c_uint32
        lib.ref_seqset_create.argtypes = [vp, u32]
        lib.ref_seqset_create.restype = vp
        lib.ref_seqset_destroy.argtypes = [vp]
        lib.ref_seqset_len.argtypes = [vp, u32]
        lib.ref_seqset_len.restype = u32
        lib.ref_seqset_codes.argtypes = [vp, u32, vp]
        lib.ref_lcs_row_prefix.argtypes = [vp, u32, u32, vp, C.c_int]
        lib.ref_lcs_row_ids.argtypes = [vp, u32, vp, u32, vp, C.c_int]
        lib.ref_lcs_triangle_mt.argtypes = [vp, u32, u32, C.c_int, C.c_int, vp, vp]
        lib.ref_lcs_triangle_mt.restype = C.c_double
        lib.ref_mst_prim_tree.argtypes = [vp, C.c_int, vp]
        lib.ref_mst_to_dendogram.argtypes = [C.c_int, vp, vp, vp, vp, vp]
        lib.ref_upgma_tree.argtypes = [vp, C.c_int, C.c_int, vp]
        lib.ref_upgma_tree_from_distances.argtypes = [vp, C.c_int, C.c_int, vp]
        lib.ref_transform_f64.argtypes = [C.c_int, u32, u32, u32]
        lib.ref_transform_f64.restype = C.c_double
        lib.ref_transform_f32.argtypes = [C.c_int, u32, u32, u32]
        lib.ref_transform_f32.restype = C.c_float
        i64 = C.c_int64
        lib.ref_dp_create.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.ref_dp_create.restype = vp
        lib.ref_dp_destroy.argtypes = [vp]
        lib.ref_dp_gaps.argtypes = [vp, vp]
        lib.ref_dp_set_gaps.argtypes = [vp, vp]
        lib.ref_dp_score_matrix.argtypes = [vp, vp]
        lib.ref_profile_create.argtypes = [vp, vp, vp, u32]
        lib.ref_profile_create.restype = vp
        lib.ref_profile_leaf.argtypes = [vp, C.c_char_p, C.c_int]
        lib.ref_profile_leaf.restype = vp
        lib.ref_profile_destroy.argtypes = [vp]
        lib.ref_profile_width.argtypes = [vp]
        lib.ref_profile_width.restype = u32
        lib.ref_profile_card.argtypes = [vp]
        lib.ref_profile_card.restype = u32
        lib.ref_profile_total_score.argtypes = [vp]
        lib.ref_profile_total_score.restype = i64
        lib.ref_profile_tables.argtypes = [vp, vp, vp]
        if hasattr(lib, "ref_profile_set_scores"):       # absent from a library built before the harness had it
            lib.ref_profile_set_scores.argtypes = [vp, vp]
        lib.ref_profile_row.argtypes = [vp, u32, vp]
        lib.ref_profile_row.restype = C.c_int
        lib.ref_profile_align.argtypes = [vp, vp, vp, C.c_int]
        lib.ref_profile_align.restype = vp
        lib.ref_profile_construct.argtypes = [vp, vp, vp, vp, vp, C.c_int]
        lib.ref_profile_construct.restype = vp
        lib.ref_dp_align_pairs_mt.argtypes = [vp, vp, vp, u32, C.c_int, vp]
        lib.ref_dp_align_pairs_mt.restype = C.c_double
        lib.ref_align_tree_mt.argtypes = [vp, vp, u32, vp, C.c_int, vp, vp, vp, vp, u32]
        lib.ref_align_tree_mt.restype = C.c_double
        _ref = lib
    return _ref


def mst_to_dendogram(edge_from, edge_to, edge_dist, prim_orders) -> np.ndarray:
    """The reference's own mst_to_dendogram on external MST edges (Prim order)."""
    n = len(prim_orders)
    f = np.ascontiguousarray(edge_from, dtype=np.int32); t = np.ascontiguousarray(edge_to, dtype=np.int32)
    d = np.ascontiguousarray(edge_dist, dtype=np.float64); o = np.ascontiguousarray(prim_orders, dtype=np.int32)
    out = np.zeros((2 * n - 1, 2), dtype=np.int32)
    ref().ref_mst_to_dendogram(n, _p(f), _p(t), _p(d), _p(o), _p(out))
    return out


def upgma_tree_from_distances(tri: np.ndarray, n: int, modified: bool = False) -> np.ndarray:
    """The reference's UPGMA agglomeration (computeTree) on an external float distance triangle."""
    t = np.ascontiguousarray(tri, dtype=np.float32)
    out = np.zeros((2 * n - 1, 2), dtype=np.int32)
    ref().ref_upgma_tree_from_distances(_p(t), n, int(modified), _p(out))
    return out


class RefDp:
    """The reference's CProfile machinery behind oracle/ref_harness.cpp."""

    def __init__(self, n_seqs_for_rescale: int = 0, matrix_type: int = 2, pool_threads: int = 2):
        self.lib = ref()
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
        self.lib = ref()
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
