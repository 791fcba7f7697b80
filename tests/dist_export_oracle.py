"""Plain restatement of the -dist_export text (reference src/tree/DistanceCalculator.cpp:10-122 and
src/utils/conversion.h:52-119), built from an LCS matrix with the row as seq0.  Test infrastructure only.

Values are printed by NumericConversions::Double2PChar((double) v, 6) as the reference's x86-64 build runs it:
    a = (int64) v;  b = (int64) ((1.0 + (v - a)) * 1e6 + 0.5)          (each operation rounded on its own)
    text = digits of (uint64) a, then digits of (uint64) b with the first one replaced by '.'
where (int64) of NaN or of a value outside the int64 range is 0x8000000000000000 (cvttsd2si)."""
from __future__ import annotations

import math

import numpy as np

from oracle import pyoracle

_INT64_MIN = np.int64(-2**63)


def _x86_trunc(x: np.ndarray) -> np.ndarray:
    ok = (x >= -2.0**63) & (x < 2.0**63)            # False for NaN
    out = np.full(x.shape, _INT64_MIN, dtype=np.int64)
    out[ok] = np.trunc(x[ok]).astype(np.int64)
    return out


def split_values(values) -> tuple[np.ndarray, np.ndarray]:
    """(a, b) of Double2PChar as uint64 arrays."""
    d = np.asarray(values, dtype=np.float32).astype(np.float64)
    a = _x86_trunc(d)
    with np.errstate(invalid="ignore", over="ignore"):
        t = (1.0 + (d - a.astype(np.float64))) * 1e6    # numpy rounds the product before the sum: no FMA
        t = t + 0.5
    b = _x86_trunc(t)
    return a.view(np.uint64), b.view(np.uint64)


def num2str(values) -> list[bytes]:
    a, b = split_values(values)
    return [(b"%d" % x) + b"." + (b"%d" % y)[1:] for x, y in zip(a.tolist(), b.tolist())]


def pow075_table(max_len: int) -> np.ndarray:
    """(double) pow(i, 0.75) by the C library, like Transform<double, indel075_div_lcs>'s table."""
    return np.array([math.pow(i, 0.75) for i in range(2 * max_len + 2)], dtype=np.float64)


def transform_matrix(lcs: np.ndarray, len_r: np.ndarray, len_c: np.ndarray, kind: int, pid: bool) -> np.ndarray:
    """float32 cells: Transform<float, pairwise_identity> with pid, else Transform<double, kind> rounded to float."""
    lcs = np.asarray(lcs, dtype=np.int64)
    lr = np.asarray(len_r, dtype=np.int64)[:, None] + np.zeros_like(lcs)
    lc = np.asarray(len_c, dtype=np.int64)[None, :] + np.zeros_like(lcs)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if pid:
            return lcs.astype(np.float32) / np.minimum(lr, lc).astype(np.float32)
        indel = lr + lc - 2 * lcs
        if kind == 0:
            num = pow075_table(int(max(lr.max(initial=0), lc.max(initial=0))))[indel]
        else:
            num = indel.astype(np.float64)
        d = num / lcs.astype(np.float64)
        d[lcs == 0] = np.nextafter(np.finfo(np.float64).max, 0)
        return d.astype(np.float32)


def csv_from_lcs(lcs_sq: np.ndarray, lens, ids, kind: int = 0, square: bool = False, pid: bool = False) -> bytes:
    """The file DistanceCalculator<kind>::run writes for a set whose LCS matrix (row = seq0) is lcs_sq."""
    lens = np.asarray(lens, dtype=np.int64)
    ids = [i.encode() if isinstance(i, str) else bytes(i) for i in ids]
    n = len(ids)
    vals = transform_matrix(lcs_sq, lens, lens, kind, pid) if n else np.zeros((0, 0), np.float32)
    out = []
    if square:
        out.append(b"".join(b"," + i for i in ids) + b"\n")
    for r in range(n):
        cols = n if square else r
        row = ids[r] + b"," + b"".join(s + b"," for s in num2str(vals[r, :cols]))
        out.append(row[:-1] + b"\n")
    return b"".join(out)


def lcs_square(codes, offsets, lens) -> np.ndarray:
    """n x n LCS lengths with the row as seq0, by the C restatement of the reference recurrence."""
    n = len(lens)
    return pyoracle.lcs_rows(codes, offsets, lens, list(range(n)), n_col=n).astype(np.int64)


def expected(code_list, ids, kind: int, square: bool, pid: bool, live: bool = True) -> bytes:
    """The export of (code_list, ids): the reference's DistanceCalculator where oracle/_ref is built and `live`, else
    the restatement."""
    from famsa_b200 import seqio
    if live and pyoracle.have("ref_dist"):
        return ref_dist_export([seqio.decode(s) for s in code_list], ids, kind, square, pid, n_threads=8)
    codes, offsets, lens = seqio.pack(code_list)
    return csv_from_lcs(lcs_square(codes, offsets, lens), lens, ids, kind, square, pid)


# ---------------------------------------------------------------- the reference itself (oracle/_ref, where built)
def ref_num2str(values) -> list[bytes]:
    """The reference's num2str on float32 values (one call for all of them)."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    out = np.zeros(max(40 * v.size, 1), dtype=np.uint8)
    n = pyoracle.lib("ref_dist").ref_num2str_f32(v.ctypes.data, v.size, out.ctypes.data)
    return out[:n].tobytes().split(b",")[:-1]


def ref_dist_export(letters, ids, kind: int = 0, square: bool = False, pid: bool = False, path: str = None,
                    n_threads: int = 1) -> bytes | None:
    """The reference's DistanceCalculator<kind>::run on (letters, ids); returns the file's bytes (or None with `path`,
    where the file is then left)."""
    import ctypes as C
    import os
    import tempfile
    n = len(letters)
    lb = [s.encode() if isinstance(s, str) else bytes(s) for s in letters]
    ib = [s.encode() if isinstance(s, str) else bytes(s) for s in ids]
    la = (C.c_char_p * max(n, 1))(*lb)
    ia = (C.c_char_p * max(n, 1))(*ib)
    keep = path is not None
    if path is None:
        fd, path = tempfile.mkstemp(suffix=".csv")
        os.close(fd)
    try:
        rc = pyoracle.lib("ref_dist").ref_dist_export(la, ia, n, kind, int(square), int(pid), path.encode(), n_threads)
        assert rc == 0
        if keep:
            return None
        with open(path, "rb") as fh:
            return fh.read()
    finally:
        if not keep:
            os.unlink(path)
