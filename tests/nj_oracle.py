"""NeighborJoining<d> (-gt nj) for the tests: the plain-C restatement of computeTree (oracle/libnj_oracle.so,
oracle/nj_oracle.c) and ctypes access to the reference's own run and computeTree through
oracle/_ref/libfamsa_ref_nj.so (oracle/ref_nj_harness.cpp).  Both libraries are built by oracle/nj.mk."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NJ_ORACLE_SO = os.path.join(_ROOT, "oracle", "libnj_oracle.so")
REF_NJ_SO = os.path.join(_ROOT, "oracle", "_ref", "libfamsa_ref_nj.so")
FLT_MAX = float(np.finfo(np.float32).max)

_oracle = None
_ref = None


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def oracle() -> C.CDLL:
    global _oracle
    if _oracle is None:
        if not os.path.exists(NJ_ORACLE_SO):
            subprocess.run(["make", "-C", os.path.join(_ROOT, "oracle"), "-f", "nj.mk", "all"], check=True,
                           stdout=subprocess.DEVNULL)
        lib = C.CDLL(NJ_ORACLE_SO)
        lib.nj_oracle_tree.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        lib.nj_oracle_tree.restype = C.c_int
        _oracle = lib
    return _oracle


def restated(dist_tri, n: int):
    """The restated computeTree on a float distance triangle (row i against j < i at i(i-1)/2 + j; left untouched).
    Returns (status, merges): status 0 with the n-1 merges as (n-1, 2) int32, or 1 (a step without a candidate) with
    the merges made before that step."""
    d = np.array(dist_tri, dtype=np.float32, copy=True)
    assert d.size == n * (n - 1) // 2 and n >= 2
    out = np.zeros((n - 1, 2), dtype=np.int32)
    done = C.c_uint32()
    rc = oracle().nj_oracle_tree(_p(d), n, _p(out), C.byref(done))
    assert rc in (0, 1)
    return rc, out[:done.value]


def have_ref() -> bool:
    return os.path.exists(REF_NJ_SO)


def ref() -> C.CDLL:
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_NJ_SO)
        lib.ref_nj_tree.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        lib.ref_nj_tree.restype = C.c_int
        lib.ref_nj_tree_from_distances.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lib.ref_nj_tree_from_distances.restype = C.c_int
        _ref = lib
    return _ref


def ref_tree(letters: list[str], kind: int):
    """The reference's own NeighborJoining<kind>::run on the set in this order: ((n-1, 2) int32 merges, seconds)."""
    n = len(letters)
    arr = (C.c_char_p * max(n, 1))(*[s.encode("ascii") for s in letters])
    out = np.zeros((max(2 * n - 1, 1), 2), dtype=np.int32)
    sec = C.c_double()
    assert ref().ref_nj_tree(arr, n, kind, _p(out), C.byref(sec)) == 0
    return out[n:2 * n - 1], sec.value


def ref_tree_from_distances(dist_tri, n: int, kind: int = 0) -> np.ndarray:
    """The reference's computeTree on an external float triangle (left untouched): the n-1 merges as it emits them,
    including a self-merge (0-th cluster with itself) where a step has no candidate."""
    d = np.array(dist_tri, dtype=np.float32, copy=True)
    assert d.size == n * (n - 1) // 2
    out = np.zeros((max(n - 1, 1), 2), dtype=np.int32)
    assert ref().ref_nj_tree_from_distances(_p(d), n, kind, _p(out)) == 0
    return out[:n - 1]
