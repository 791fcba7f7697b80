"""NeighborJoining<d> (-gt nj) for the tests: the plain-C restatement of computeTree (oracle/libnj_oracle.so,
oracle/nj_oracle.c) and the reference's own run and computeTree through oracle/_ref/libfamsa_ref_nj.so
(oracle/ref_nj_harness.cpp), both opened by oracle/pyoracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

FLT_MAX = float(np.finfo(np.float32).max)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def restated(dist_tri, n: int):
    """The restated computeTree on a float distance triangle (row i against j < i at i(i-1)/2 + j; left untouched).
    Returns (status, merges): status 0 with the n-1 merges as (n-1, 2) int32, or 1 (a step without a candidate) with
    the merges made before that step."""
    d = np.array(dist_tri, dtype=np.float32, copy=True)
    assert d.size == n * (n - 1) // 2 and n >= 2
    out = np.zeros((n - 1, 2), dtype=np.int32)
    done = C.c_uint32()
    rc = pyoracle.lib("nj_oracle").nj_oracle_tree(_p(d), n, _p(out), C.byref(done))
    assert rc in (0, 1)
    return rc, out[:done.value]


def ref_tree(letters: list[str], kind: int):
    """The reference's own NeighborJoining<kind>::run on the set in this order: ((n-1, 2) int32 merges, seconds)."""
    n = len(letters)
    arr = (C.c_char_p * max(n, 1))(*[s.encode("ascii") for s in letters])
    out = np.zeros((max(2 * n - 1, 1), 2), dtype=np.int32)
    sec = C.c_double()
    assert pyoracle.lib("ref_nj").ref_nj_tree(arr, n, kind, _p(out), C.byref(sec)) == 0
    return out[n:2 * n - 1], sec.value


def ref_tree_from_distances(dist_tri, n: int, kind: int = 0) -> np.ndarray:
    """The reference's computeTree on an external float triangle (left untouched): the n-1 merges as it emits them,
    including a self-merge (0-th cluster with itself) where a step has no candidate."""
    d = np.array(dist_tri, dtype=np.float32, copy=True)
    assert d.size == n * (n - 1) // 2
    out = np.zeros((max(n - 1, 1), 2), dtype=np.int32)
    assert pyoracle.lib("ref_nj").ref_nj_tree_from_distances(_p(d), n, kind, _p(out)) == 0
    return out[:n - 1]
