"""Generates the single-linkage (-gt slink) fixtures from the reference's test data and its own SingleLinkage<d>::run
(oracle/_ref/libfamsa_ref_slink.so, built by oracle/Makefile).

Run where the reference's sources are at hand:  python tests/golden/make_slink.py [lrr]
Outputs (small, committed):
  adeno_slink_tree.npz   test/adeno_fiber in FAMSA's order (length-descending, msa.cpp:245-256) and the reference's
                         SLINK tree on it (kind 0); generation asserts that its clades are exactly those of
                         test/adeno_fiber/slink.dnd and that the restatement in tests/slink_oracle.py and the MST
                         labelling of famsa_b200.mst.slink_tree both rebuild it.
  slink_pruning_case.npz a small dropped-carry set, in an order that puts flagged sequences after shorter ones, on which
                         the sequential MST loop WITH MSTPrim's lower-bound skip (MSTPrim.cpp:450-467) loses an edge
                         SLINK keeps; generation asserts that difference.  Holds the reference's trees (kinds 0 and 1)
                         in that order and in FAMSA's sorted order.
  lrr_slink.npz          (argument `lrr`, about a quarter of an hour on 8 cores) the CRC32 of the reference's SLINK tree
                         on the set of lrr_sl.npz.
"""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
from famsa_b200 import mst, seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402
import slink_oracle as S  # noqa: E402

REF = "/root/reference/test"


def famsa_order(code_list):
    return sorted(range(len(code_list)), key=lambda i: (-len(code_list[i]), code_list[i].tobytes()))


def lcs_square(letters):
    codes, offsets, lens = seqio.pack([seqio.encode(s) for s in letters])
    return pyoracle.lcs_rows(codes, offsets, lens, np.arange(len(lens))), lens


def make_adeno():
    from treeutil import parse_newick
    T = os.path.join(REF, "adeno_fiber")
    ids, seqs = seqio.read_fasta(os.path.join(T, "adeno_fiber"))
    code_list = [seqio.encode(s) for s in seqs]
    order = famsa_order(code_list)
    names = [ids[i] for i in order]
    letters = [seqs[i] for i in order]
    n = len(letters)
    tree = S.ref_slink_tree(letters, 0)
    sq, lens = lcs_square(letters)
    dist = S.slink_distances(sq, lens, 0)
    assert [tuple(int(x) for x in r) for r in tree] == S.slink_restated(n, dist), "restatement differs from the reference"
    assert np.array_equal(mst.slink_tree(n, mst.kruskal_total_order(n, dist)), tree), "MST labelling differs from the reference"

    def clades(n_leaves, merges, leaf_names):
        sets = [frozenset([nm]) for nm in leaf_names]
        for a, b in merges:
            sets.append(sets[a] | sets[b])
        return set(sets[n_leaves:])
    gl, gm = parse_newick(open(os.path.join(T, "slink.dnd")).read())
    assert clades(n, [tuple(int(x) for x in r) for r in tree], names) == clades(len(gl), gm, gl), \
        "tree differs from the golden slink.dnd"
    np.savez_compressed(os.path.join(HERE, "adeno_slink_tree.npz"), names=np.array(names), seqs=np.array(letters), tree=tree)
    print("adeno_slink_tree.npz:", n, "sequences, clades equal to slink.dnd")


def prim_with_skip(n, lens, dist, kind):
    """The sequential MST loop on SLINK's distances, with MSTPrim's lower-bound skip: a candidate j of vertex v is only
    computed when Transform(min(len v, len j), len v, len j) <= its current distance.  Returns (from, to, dist) edges."""
    best = [(S.DBL_MAX, 0)] * n
    visited = [False] * n
    visited[0] = True
    v, edges = 0, []
    for _ in range(1, n):
        for j in range(n):
            if visited[j]:
                continue
            lo_bound = pyoracle.transform(kind, int(min(lens[v], lens[j])), int(lens[v]), int(lens[j]), True)
            if lo_bound <= best[j][0]:
                hi, lo = max(v, j), min(v, j)
                cand = (float(dist[hi * (hi - 1) // 2 + lo]), mst.edge_key(v, j))
                if cand < best[j]:
                    best[j] = cand
        nxt = min((j for j in range(n) if not visited[j]), key=lambda j: best[j])
        p = mst._FULL ^ best[nxt][1]
        edges.append((p >> 32, p & 0xFFFFFFFF, best[nxt][0]))
        visited[nxt] = True
        v = nxt
    return edges


def make_pruning_case():
    rng = np.random.default_rng(2)
    AA = "ACDEFGHIKLMNPQRSTVWY"
    for trial in range(2000):
        n = int(rng.integers(5, 14))
        seqs = []
        for _ in range(n):
            a = "ACDEFGHIKL"[rng.integers(0, 10)]
            if rng.integers(0, 3) == 0:
                pre = "".join(AA[x] for x in rng.integers(0, 20, size=64 * rng.integers(0, 2)))
                s = pre + a * int(64 * rng.integers(1, 4)) + "".join(AA[x] for x in rng.integers(0, 20, size=rng.integers(0, 5)))
            else:
                s = a * int(rng.integers(1, 6)) + "".join(AA[x] for x in rng.integers(0, 20, size=rng.integers(0, 4)))
            seqs.append(s)
        sq, lens = lcs_square(seqs)
        dist = S.slink_distances(sq, lens, 0)
        want = S.ref_slink_tree(seqs, 0)
        if np.array_equal(mst.slink_tree(n, prim_with_skip(n, lens, dist, 0)), want):
            continue
        assert np.array_equal(mst.slink_tree(n, mst.kruskal_total_order(n, dist)), want), "MST labelling differs from the reference"
        sorted_seqs = [seqs[i] for i in famsa_order([seqio.encode(s) for s in seqs])]
        trees = {f"tree{k}": S.ref_slink_tree(seqs, k) for k in (0, 1)}
        trees.update({f"sorted_tree{k}": S.ref_slink_tree(sorted_seqs, k) for k in (0, 1)})
        np.savez_compressed(os.path.join(HERE, "slink_pruning_case.npz"), seqs=np.array(seqs), sorted_seqs=np.array(sorted_seqs), **trees)
        print("slink_pruning_case.npz: trial", trial, n, "sequences; the loop with the skip gives a different tree")
        return
    raise SystemExit("no witness found")


def make_lrr():
    z = np.load(os.path.join(HERE, "lrr_sl.npz"))
    letters = bytes(z["seqs"]).decode().split("\n")
    n = len(letters)
    tree = S.ref_slink_tree(letters, 0, n_threads=os.cpu_count())
    crc = zlib.crc32(np.ascontiguousarray(tree, dtype=np.int32).tobytes())
    np.savez_compressed(os.path.join(HERE, "lrr_slink.npz"), tree_crc=np.array([crc], dtype=np.uint64), n=np.array([n]))
    print("lrr_slink.npz:", n, "sequences, tree crc", crc)


if __name__ == "__main__":
    if sys.argv[1:] == ["lrr"]:
        make_lrr()
    else:
        make_adeno()
        make_pruning_case()
