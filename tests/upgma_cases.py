"""Sequence sets, crafted LCS triangles and the restated tree for the UPGMA tests (test_upgma_host.py, test_upgma_gpu.py).

Every expected tree comes from the restatement of UPGMA<>::computeTree in oracle/upgma_oracle.c, run on the host float
Transform (oracle/lcs_oracle.c) of the same LCS triangle the device reads."""
import os

import numpy as np

from conftest import GOLDEN, random_set
from famsa_b200 import seqio
from oracle import pyoracle as P

WITNESS = os.path.join(GOLDEN, "upgma_witness.npz")

# crafted triangles: n sequences of CRAFT_LEN residues each, so a distance depends on the LCS alone
CRAFT_LEN = 100
BACKGROUND, CLOSEST, SECOND, THIRD = 40, 90, 80, 70                  # LCS values; a larger LCS is a smaller distance
CRAFT_SIZES = [2, 3, 31, 32, 33, 1023, 1024, 1025, 2049, 2055]
BIG_N = 32769                                                       # 33 blocks of 1024 rows: the last one holds row 32768


def tri_index(i, j):
    hi, lo = max(i, j), min(i, j)
    return hi * (hi - 1) // 2 + lo


def restated_tree(kind, modified, lcs_tri, lens, overwrite=False):
    """(status, merges) of the restatement on Transform<float, kind> of a packed LCS triangle (row i = seq0)."""
    dist = P.transform_triangle(kind, lcs_tri, lens)
    return P.upgma_tree(dist, len(lens), modified, overwrite=overwrite)


def expected_tree(kind, modified, lcs_tri, lens):
    rc, tree = restated_tree(kind, modified, lcs_tri, lens, overwrite=True)
    assert rc == 0, "the restatement found no finite distance"
    return tree


def letters_of(codes, offsets, lens):
    return [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(offsets, lens)]


# ------------------------------------------------------------------ sequence sets
def famsa_sorted(code_list):
    return sorted(code_list, key=lambda c: (-len(c), c.tobytes()))


def dropped_carry_codes(rng):
    """Short sequences over a 4-letter alphabet next to flagged ones (runs of 64 k equal residues, some behind a 64-residue
    prefix): with such a sequence as the row, its LCS can exceed the shorter length (lcsbp_classic.h:85-92).  Every
    sequence ends in residue 0, so every pair has a common residue and a finite distance."""
    zero = np.zeros(1, np.int8)
    cl = [np.concatenate([c, zero]) for c in random_set(rng, 50, 1, 8, alphabet=4, with_specials=False)]
    for k in range(8):
        run = np.full(64 * (1 + k % 3), k % 4, np.int8)
        cl.append(np.concatenate([random_set(rng, 1, 0, 64 * (k % 2), alphabet=4)[0], run, zero]))
    return cl


def sequence_set(name):
    """(codes, offsets, lens) of a named set, in the order the tree is built on."""
    rng = np.random.default_rng(71)
    if name == "family400":
        return seqio.synth_family(400, 150, seed=72)
    if name == "ragged":
        cl = famsa_sorted(random_set(rng, 300, 12, 60, alphabet=3, with_specials=False)
                          + random_set(rng, 100, 12, 40, alphabet=4, with_specials=False))
    elif name == "twice":
        cl = random_set(rng, 60, 20, 200)
        cl = famsa_sorted(cl + [c.copy() for c in cl])
    elif name == "carry_sorted":
        cl = famsa_sorted(dropped_carry_codes(rng))
    elif name == "carry_shuffled":
        cl = dropped_carry_codes(rng)
        cl = [cl[i] for i in rng.permutation(len(cl))]
    elif name in ("n2", "n3"):
        cl = famsa_sorted(random_set(rng, int(name[1:]), 5, 60))
    else:
        raise KeyError(name)
    return seqio.pack(cl)


SETS = ["family400", "ragged", "twice", "carry_sorted", "carry_shuffled", "n2", "n3"]


def oracle_triangle(codes, offsets, lens):
    return P.lcs_triangle(codes, offsets, lens)


# ------------------------------------------------------------------ crafted LCS triangles
def craft(n, case, seed=0):
    """(LCS triangle uint16, lens) of n equal-length sequences.
    random    tie-heavy: every LCS drawn from four values
    block_tie rows 3, 1027 and 2051 (the same offset in blocks 0, 1 and 2 of 1024 rows) hold equal cached minima
    last_row  the unique smallest distance is in row n-1, the last row of the last block
    stale     (0,1) closest, (1, n-1) next: merging 0 and 1 relabels row n-1's neighbour to 0 but keeps its old distance,
              so the new row's minimum and the next merge's minimum both lie in row n-1
    new_tie   (0,1) closest; rows 700, 1500 and 2050 at equal distance from both, so the new row's minimum is a
              three-way tie across blocks"""
    m = n * (n - 1) // 2
    if case == "random":
        lcs = np.random.default_rng(seed).choice(np.array([30, 40, 50, 60], np.uint16), size=m)
    else:
        lcs = np.full(m, BACKGROUND, dtype=np.uint16)
    if case == "block_tie":
        lcs[tri_index(3, 1027)] = CLOSEST
        lcs[tri_index(1027, 2051)] = CLOSEST
    elif case == "last_row":
        lcs[tri_index(n - 1, 5)] = CLOSEST
    elif case == "stale":
        lcs[tri_index(0, 1)] = CLOSEST
        lcs[tri_index(1, n - 1)] = SECOND
    elif case == "new_tie":
        lcs[tri_index(0, 1)] = CLOSEST
        for j in (700, 1500, 2050):
            lcs[tri_index(0, j)] = THIRD
            lcs[tri_index(1, j)] = THIRD
    elif case != "random":
        raise KeyError(case)
    return lcs, np.full(n, CRAFT_LEN, dtype=np.uint32)


CRAFTED = [("random", n) for n in CRAFT_SIZES] + [("block_tie", 2055), ("last_row", 1025), ("last_row", 2049),
                                                   ("last_row", 2055), ("stale", 1025), ("stale", 2055),
                                                   ("new_tie", 2055)]


def crafted_codes(n):
    """n sequences of CRAFT_LEN residues to upload beside a crafted triangle (only their lengths are read)."""
    return seqio.pack([np.arange(CRAFT_LEN, dtype=np.int8) % 20 for _ in range(n)])


# ------------------------------------------------------------------ witness fixture
def witness_cases():
    z = np.load(WITNESS)
    out = {}
    for name in (str(s) for s in z["names"]):
        out[name] = dict(lcs=z[f"{name}_lcs"], lens=z[f"{name}_lens"], kind=int(z[f"{name}_kind"]),
                         modified=bool(int(z[f"{name}_modified"])), tree=z[f"{name}_tree"])
    return out


WITNESS_VARIANT = {"stale": dict(fresh_cache=True), "stale_modified": dict(fresh_cache=True),
                   "rounded_once": dict(avg_mode=P.UPGMA_AVG_ROUNDED_ONCE),
                   "rounded_once_kind1": dict(avg_mode=P.UPGMA_AVG_ROUNDED_ONCE),
                   "fused": dict(avg_mode=P.UPGMA_AVG_FUSED), "fused_kind1": dict(avg_mode=P.UPGMA_AVG_FUSED)}
