"""Writes tests/golden/construct_shapes.npz from the reference (oracle/_ref): for every case of tests/construct_shapes.py
the CRC32 of the reference's merged scores and counters, its total score, and the CRC32 of the path and the orientation
of the C restatement's Align (pinned against the reference's by tests/test_oracle_dp.py, and its total must be the
reference's here); for every tree
of construct_shapes.tree_cases() the totals and the CRC32 of the root's tables; and the score matrix, so that
tests/test_construct_shapes_gpu.py runs where the reference library is absent.

    python tests/golden/make_construct.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import numpy as np  # noqa: E402

import construct_shapes as S  # noqa: E402
import dp_cases  # noqa: E402
from oracle import pyoracle  # noqa: E402


def main():
    assert pyoracle.have_ref_set_scores(), "needs oracle/_ref/libfamsa_ref.so with ref_profile_set_scores (build() where the reference sources are)"
    names, crcs, totals, swapped = [], [], [], []
    for c in S.cases():
        res, _, _ = S.oracle_merge(c)
        ref = S.reference_merge(c)
        assert ref["total"] == res["total"], c["name"]
        names.append(c["name"])
        crcs.append([S.crc(ref["scores"]), S.crc(ref["counters"]), S.crc(res["path"]), ref["card"]])
        totals.append(ref["total"])
        swapped.append(int(res["swapped"]))
    out = dict(score_matrix=S.score_matrix(), names=np.array(names), crcs=np.array(crcs, dtype=np.int64),
               totals=np.array(totals, dtype=np.int64), swapped=np.array(swapped, dtype=np.int8))
    for t in S.tree_cases():
        g, recs = dp_cases.reference_merges(t["seqs"], t["merges"], threads=(1,), want_merged=True)
        s, c, k = recs[-1]["merged"]
        out[f"tree_{t['name']}_gaps"] = np.asarray(g, dtype=np.int64)
        out[f"tree_{t['name']}_totals"] = np.array([r["total"] for r in recs], dtype=np.int64)
        out[f"tree_{t['name']}_root"] = np.array([S.crc(s), S.crc(c), k], dtype=np.int64)
    np.savez_compressed(S.FIXTURE, **out)
    print(f"{len(names)} cases, {len(S.tree_cases())} trees -> {S.FIXTURE}")


if __name__ == "__main__":
    main()
