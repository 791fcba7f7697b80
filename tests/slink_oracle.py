"""SingleLinkage<d>::run (-gt slink) for the tests: a verbatim restatement of the reference's pointer loops, and the
reference's own run through oracle/_ref/libfamsa_ref_slink.so (oracle/ref_slink_harness.cpp, opened by
oracle/pyoracle.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

DBL_MAX = float(np.finfo(np.float64).max)


def _ids_to_uint64(a: int, b: int) -> int:
    lo, hi = (a, b) if a < b else (b, a)
    return (lo << 32) + hi


def slink_restated(n: int, tri) -> list[tuple[int, int]]:
    """SingleLinkage.cpp:30-189 with SLINK_HANDLE_TIES (SingleLinkage.h:16-38): the two pointer loops over rows i = 0..n-1
    (row i against j < i, distance tri[i*(i-1)/2 + j]), slink_dist_t order (distance ascending, then ids_to_uint64(j, i)
    descending: sorting on (distance, -id) reproduces its < and <=), stable_sort of lambda and the index relabelling.
    Returns the n-1 merges (left, right); internal node n+k is merge k."""
    pi = [0] * n
    lam = [None] * n
    for i in range(n):
        pi[i] = i
        lam[i] = (DBL_MAX, 0)
        base = i * (i - 1) // 2
        dv = [(float(tri[base + j]), -_ids_to_uint64(j, i)) for j in range(i)] + [None] * (n - i)
        for j in range(i):
            nx = pi[j]
            if lam[j] < dv[j]:
                dv[nx] = dv[j] if dv[nx] is None else min(dv[nx], dv[j])
            else:
                dv[nx] = lam[j] if dv[nx] is None else min(dv[nx], lam[j])
                pi[j] = i
                lam[j] = dv[j]
        for j in range(i):
            if lam[pi[j]] <= lam[j]:
                pi[j] = i
    elements = sorted(range(n - 1), key=lambda x: lam[x])             # sorted() is stable, as stable_sort
    index = list(range(n))
    tree = []
    for k, j in enumerate(elements):
        nx = pi[j]
        tree.append((index[j], index[nx]))
        index[nx] = n + k
    return tree


def slink_distances(lcs_square: np.ndarray, lens, kind: int) -> np.ndarray:
    """The packed distance triangle SLINK reads: row i (the row, seq0) against j < i through Transform<double, kind>."""
    n = len(lens)
    out = np.zeros(n * (n - 1) // 2, dtype=np.float64)
    at = 0
    for i in range(1, n):
        for j in range(i):
            out[at] = pyoracle.transform(kind, int(lcs_square[i, j]), int(lens[i]), int(lens[j]), True)
            at += 1
    return out


def ref_slink_tree(letters: list[str], kind: int, n_threads: int = 8) -> np.ndarray:
    """The reference's own SingleLinkage<kind>::run on the set in this order: the n-1 merges, (n-1, 2) int32."""
    n = len(letters)
    arr = (C.c_char_p * max(n, 1))(*[s.encode("ascii") for s in letters])
    out = np.zeros((max(2 * n - 1, 1), 2), dtype=np.int32)
    rc = pyoracle.lib("ref_slink").ref_slink_tree(arr, n, kind, n_threads, out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out[n:2 * n - 1] if n else out[:0]
