"""Generates tests/golden/adeno_dist_export.npz from the reference's own test data.

Run where the reference's test directory is at hand:  python tests/golden/make_dist_export.py

adeno_dist_export.npz holds the ids of test/adeno_fiber/adeno_fiber and the bytes of the reference's four
-dist_export files (dist, pid, dist_sq, pid_sq; test/scripts/generate.sh:77-80), compressed.  Generation checks that
the restatement in tests/dist_export_oracle.py rebuilds all four from adeno_fiber_lcs.npz (make_golden.py).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
from famsa_b200 import seqio  # noqa: E402
import dist_export_oracle  # noqa: E402

REF = "/root/reference/test"
MODES = (("dist", False, False), ("pid", False, True), ("dist_sq", True, False), ("pid_sq", True, True))


def make_dist_export():
    ids, seqs = seqio.read_fasta(os.path.join(REF, "adeno_fiber", "adeno_fiber"))
    z = np.load(os.path.join(HERE, "adeno_fiber_lcs.npz"))
    assert [str(i) for i in z["ids"]] == ids
    lens = np.array([len(seqio.encode(s)) for s in seqs])
    files = {}
    for name, square, pid in MODES:
        with open(os.path.join(REF, "adeno_fiber", name + ".csv"), "rb") as fh:
            files[name] = fh.read()
        assert dist_export_oracle.csv_from_lcs(z["lcs"], lens, ids, 0, square, pid) == files[name], name
    np.savez_compressed(os.path.join(HERE, "adeno_dist_export.npz"), ids=np.array(ids),
                        **{k: np.frombuffer(v, dtype=np.uint8) for k, v in files.items()})
    print("adeno_dist_export.npz:", {k: len(v) for k, v in files.items()})


if __name__ == "__main__":
    make_dist_export()
