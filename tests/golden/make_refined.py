"""Generates tests/golden/adeno_refined.npz: FAMSA's own refined alignments of test/adeno_fiber, the goldens upgma.fasta
(-gt upgma) and sl.fasta (default -gt sl), as the device refinement must reproduce them.

Run where the reference's test data and oracle/_ref are at hand:  python tests/golden/make_refined.py

Both goldens were made with many threads, so RefineAlignment ran the unbanded Align, which is what famsa_prof_refine and
oracle/ref_refine_harness.cpp do.  For each golden the fixture holds, in the leaf order of its guide tree:
  <name>_ids    the FASTA ids as the reference keeps them (the whole header line, '>' included; RefineAlignment sorts the
                rows by these bytes);
  <name>_rows   the refined rows, n x W codes of famsa_b200.seqio's alphabet, GAP = 30 (the golden upper-cased: the
                reference writes the input's lower-case residues back in lower case).
The guide trees and sequences are the committed adeno_upgma_merges.npz (upgma.dnd) and adeno_sl_tree.npz (sl.dnd in
FAMSA's length-sorted order).  Generation first asserts that the harness' progressive alignment along that tree followed
by its restated RefineAlignment loop, with these ids, reproduces the golden byte for byte.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
from famsa_b200 import seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402

REF = "/root/reference/test"
OUT = os.path.join(HERE, "adeno_refined.npz")
GAP = 30


def codes(row: str) -> np.ndarray:
    return np.array([GAP if ch == "-" else seqio.ALPHABET.index(ch) for ch in row], dtype=np.uint8)


def cases():
    """(name, golden file, leaf names, sequences, merges) of each golden."""
    from treeutil import parse_newick
    T = os.path.join(REF, "adeno_fiber")
    z = np.load(os.path.join(HERE, "adeno_upgma_merges.npz"))
    leaves, merges = parse_newick(open(os.path.join(T, "upgma.dnd")).read())
    assert np.array_equal(np.asarray(merges), z["merges"]), "adeno_upgma_merges.npz is not the tree of upgma.dnd"
    ids, seqs = seqio.read_fasta(os.path.join(T, "adeno_fiber"))
    name2seq = dict(zip(ids, seqs))
    assert [name2seq[nm].upper() for nm in leaves] == [str(s) for s in z["seqs"]]
    yield "upgma", "upgma.fasta", leaves, [str(s) for s in z["seqs"]], z["merges"]
    s = np.load(os.path.join(HERE, "adeno_sl_tree.npz"))
    n = len(s["names"])
    yield "sl", "sl.fasta", [str(x) for x in s["names"]], [str(x) for x in s["seqs"]], s["tree"][n:]


def main():
    import refine_cases as rc
    import refine_oracle as ro
    if not pyoracle.have("ref_refine"):
        raise SystemExit("oracle/_ref/libfamsa_ref_refine.so is not built")
    out = {}
    for name, golden, leaves, seqs, merges in cases():
        gi, gs = seqio.read_fasta(os.path.join(REF, "adeno_fiber", golden))
        gold = {i: r.upper() for i, r in zip(gi, gs)}
        n = len(leaves)
        ids = [">" + nm for nm in leaves]
        g, sm = rc.scoring(n)
        ref = ro.RefRefine(sm, g)
        got = ref.align_refine(seqs, merges, 100, ids=ids)
        ref.close()
        same = [got["refined"][i] == gold[leaves[i]] for i in range(n)]
        assert all(same), f"{golden}: the harness differs in {n - sum(same)} of {n} rows"
        out[f"{name}_ids"] = np.array(ids)
        out[f"{name}_rows"] = np.stack([codes(gold[nm]) for nm in leaves])
        print(f"{golden}: {n} rows x {got['width']} columns reproduced, {got['counts']}")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
