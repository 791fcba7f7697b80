"""Generates the neighbour-joining (-gt nj) fixtures from the reference's own NeighborJoining<d>::run
(oracle/_ref/libfamsa_ref_nj.so, built by oracle/Makefile).  The reference ships no nj.dnd, so these trees are the goldens.

Run where the reference's sources are at hand:  python tests/golden/make_nj.py
Outputs (small, committed):
  adeno_nj_tree.npz   test/adeno_fiber in FAMSA's order (length-descending, msa.cpp:245-256; the set of
                      adeno_slink_tree.npz) and the reference's trees for kinds 0 and 1.
  hemopexin_nj.npz    the 4 188-sequence set of hemopexin_sl.npz in its order and the reference's trees for kinds 0 and 1.
Generation asserts that the restatement (oracle/nj_oracle.c) rebuilds every tree from the float Transform of the C
oracle's LCS triangle.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
from famsa_b200 import seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402
import nj_oracle as N  # noqa: E402


def trees_of(letters):
    codes, offsets, lens = seqio.pack([seqio.encode(s) for s in letters])
    lcs = pyoracle.lcs_triangle(codes, offsets, lens)
    out = {}
    for kind in (0, 1):
        tree, sec = N.ref_tree(letters, kind)
        rc, want = N.restated(pyoracle.transform_triangle(kind, lcs, lens), len(letters))
        assert rc == 0 and np.array_equal(tree, want), f"restatement differs from the reference (kind {kind})"
        out[f"tree{kind}"] = tree
        print(f"  kind {kind}: reference {sec:.2f} s")
    return out


def make(name, letters):
    np.savez_compressed(os.path.join(HERE, name), seqs=np.array(letters), **trees_of(letters))
    print(f"{name}: {len(letters)} sequences")


if __name__ == "__main__":
    make("adeno_nj_tree.npz", [str(s) for s in np.load(os.path.join(HERE, "adeno_slink_tree.npz"))["seqs"]])
    make("hemopexin_nj.npz", [str(s) for s in np.load(os.path.join(HERE, "hemopexin_sl.npz"))["seqs"]])
