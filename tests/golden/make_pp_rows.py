"""Generates adeno_pp_rows.npz: the reference's profile-profile golden as rows.

FAMSA's CI runs  famsa -refine_mode off upgma.no_refine.part1.fasta upgma.no_refine.part2.fasta out  and diffs the result
against test/adeno_fiber/upgma.pp.fasta.  The fixture holds the ids and the case-preserved rows of both inputs, the
golden's ids and rows in file order, the rescaled gap costs (adjustParams(n1 + n2), famsa.cpp:94) and the score matrix.
Generation asserts that the reference's own CProfile (oracle/_ref: profile() of each input, align(..., 1), rows in data
order) reproduces the golden's rows in the golden's order, and that profiles.rows_after_merge, driven by the oracle's
path, gives the golden's rows with their letter case.

Run where the reference's sources and oracle/_ref are at hand:  python tests/golden/make_pp_rows.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from famsa_b200 import profiles, seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402

T = "/root/reference/test/adeno_fiber"


def main():
    i1, s1 = seqio.read_fasta(os.path.join(T, "upgma.no_refine.part1.fasta"))
    i2, s2 = seqio.read_fasta(os.path.join(T, "upgma.no_refine.part2.fasta"))
    ig, sg = seqio.read_fasta(os.path.join(T, "upgma.pp.fasta"))
    n1, n2 = len(s1), len(s2)
    dp = pyoracle.RefDp(n1 + n2)
    gaps, sm = dp.gaps(), dp.score_matrix()
    p1 = dp.profile([s.upper() for s in s1], list(range(n1)))
    p2 = dp.profile([s.upper() for s in s2], list(range(n1, n1 + n2)))
    t1, c1, k1 = dp.tables(p1)
    t2, c2, k2 = dp.tables(p2)
    m, total = dp.align(p1, p2, 1)
    rows = dp.rows(m)                                   # data order: seq_no -> row
    dp.free(m)
    dp.close()
    names = i1 + i2
    assert [names[no] for no in rows] == ig, "the reference's data order is not upgma.pp.fasta's order"
    assert list(rows.values()) == [s.upper() for s in sg], "the reference's rows are not upgma.pp.fasta's"
    o = pyoracle.dp_align(t1, c1, k1, t2, c2, k2, gaps, sm)
    assert o["total"] == total
    order, merged = profiles.rows_after_merge(s1, s2, o["path"], o["swapped"], from_text=True)
    assert [names[k] for k in order] == ig and merged == sg, "rows_after_merge does not give upgma.pp.fasta"
    np.savez_compressed(os.path.join(HERE, "adeno_pp_rows.npz"), ids1=np.array(i1), rows1=np.array(s1), ids2=np.array(i2),
                        rows2=np.array(s2), gold_ids=np.array(ig), gold_rows=np.array(sg), gaps=gaps, score_matrix=sm,
                        total=np.array(total), path=o["path"], swapped=np.array(o["swapped"]))
    print(f"adeno_pp_rows.npz: {n1} + {n2} rows, widths {len(s1[0])} / {len(s2[0])} -> {len(sg[0])}, total {total}")


if __name__ == "__main__":
    main()
