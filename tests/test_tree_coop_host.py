"""The claims of tree_coop_cases.py on the CPU: the tree.cu constants it is built on, sizes that cross the cooperative
grid's thread count for their cap, the big pattern's offsets past 2^32 and its hand-derived merges (confirmed by the
restated computeTree on the small analogue), the crafted triangles' first merges, and the vectorised Prim against the
slow restatement, the pruning fixture and, where oracle/_ref is built, the reference's MSTPrim tree."""
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, random_set
from famsa_b200 import mst, seqio
from oracle import pyoracle as P
import tree_coop_cases as T
import upgma_cases as U
from treeutil import prim_restated

SRC = open(os.path.join(ROOT, "famsa_b200", "csrc", "tree.cu")).read()


def test_constants_match_tree_cu():
    for kern in ("k_prim", "k_upgma", "k_nj"):
        assert re.search(r"__launch_bounds__\(%d\) %s\(" % (T.COOP_THREADS, kern), SRC), kern
    assert len(re.findall(r"cudaLaunchCooperativeKernel\([^;]*dim3\(%d\)" % T.COOP_THREADS, SRC)) == 3
    assert re.search(r"coop_cap\(std::max\(1u, std::min\([^;]*\(n \+ %d\) / %d\)\)\);" % (T.COOP_THREADS - 1, T.COOP_THREADS), SRC)          # coop_blocks
    assert re.search(r"constexpr uint32_t kMstChunk = %d;" % T.K_MST_CHUNK, SRC)
    assert re.search(r"coop_cap\(std::max\(1u, std::min\([^;]*\(n \+ %d\) / %d\)\)\);" % (T.NJ_ROWS_PER_BLOCK - 1, T.NJ_ROWS_PER_BLOCK), SRC)  # lcs_nj
    # each knob is read in one place, the one the cooperative launches go through
    assert SRC.count('getenv("FAMSA_TREE_MAX_BLOCKS")') == 1
    assert SRC.count('getenv("FAMSA_TREE_DEBUG")') == 1


@pytest.mark.parametrize("cap", T.CAPS)
def test_sizes_cross_the_passes(cap):
    t = T.COOP_THREADS * cap
    s = T.sizes(cap)
    passes = [(n + t - 1) // t for n in s]
    assert passes == [1, 2, 2, 2, 3, 4]
    assert s[1] - 1 == t and s[4] - 1 == 2 * t                         # the first sequence of a second / third pass
    # with 2 or 3 blocks the sequences a thread owns second belong to blocks other than 0 as well
    owners = {(j % t) // T.COOP_THREADS for j in range(t, s[-1])}
    assert owners == set(range(cap))
    cases = [c for c in T.CASES if c[0] == cap]
    assert {c[2] for c in cases} == set(T.SETS) and {c[1] for c in cases} == set(s)


@pytest.mark.parametrize("cap", T.CAPS)
def test_carry_sequences_sit_in_the_loop_path(cap):
    t = T.COOP_THREADS * cap
    for n in T.sizes(cap):
        pos = T.carry_positions(n, cap)
        assert len(pos) == 8 and len(set(pos)) == 8 and max(pos) < n
        if n >= t + 8:
            assert min(pos) >= t
    codes, offsets, lens, exact = T.sequence_set("carry", t + 1, cap)
    assert len(lens) == t + 1 and exact == T.carry_positions(t + 1, cap)
    assert all(lens[i] >= 64 for i in exact) and int(np.sum(lens >= 64)) == 8


def test_big_pattern_offsets():
    n = T.BIG_N
    assert n * (n - 1) // 2 == 4_324_453_500
    assert T.tri_index(92682, 37074) < T.TWO32 == T.tri_index(92682, 37075)          # the straddling row
    assert T.tri_index(92683, 0) > T.TWO32
    cells = T.big_cells()
    offs = [o for o, _ in cells]
    assert all(o >= T.TWO32 for o in offs) and len(set(offs)) == len(offs)
    assert max(max(p[:2]) for p in T.BIG_PAIRS) < n and max(T.BIG_TRIPLE) < n
    # a truncated offset lands on a background cell, none on another's image
    low = [o % T.TWO32 for o in offs]
    assert len(set(low)) == len(low) and not set(low) & set(offs)
    # the row the triple's cluster writes lies wholly past 2^32, and so does the cell read back for c
    a, b, c = T.BIG_TRIPLE
    assert T.tri_index(a, 0) > T.TWO32 and T.tri_index(c, a) > T.TWO32
    # every planted index is its own: pairs and triple are disjoint
    ids = [i for p in T.BIG_PAIRS for i in p[:2]] + list(T.BIG_TRIPLE)
    assert len(set(ids)) == len(ids)
    # the pairs' LCS values exceed the triple's, in descending order, and the background is the smallest
    v = [p[2] for p in T.BIG_PAIRS] + list(T.BIG_TRIPLE_LCS)
    assert v == sorted(v, reverse=True) and len(set(v)) == len(v) and min(v) > T.BIG_BG


@pytest.mark.parametrize("modified", [False, True])
def test_big_expectation_on_small_analogue(modified):
    """The hand-derived first merges of the big pattern, on the same pattern in a small set, equal the restated tree's."""
    n, pairs, triple, lcs, lens = T.small_analogue()
    want = T.big_upgma_expected(n, pairs, triple, modified)
    got = U.expected_tree(0, modified, lcs, lens)
    assert [tuple(m) for m in got[:len(want)].tolist()] == want
    assert T.valid_tree(got, n)
    # the merge the written row decides: had row a read background instead of its averaged values, c's stale cache would
    # win the next pick and the merge would come out reversed
    k = n + len(pairs)
    assert want[-1] in ((k, triple[2]), (triple[2], k))
    if P.have_ref():
        ref = P.upgma_tree_from_distances(P.transform_triangle(0, lcs, lens), n, modified)[n:]
        assert np.array_equal(ref, got)


def test_valid_tree_rejects():
    assert T.valid_tree(np.array([[0, 3], [1, 2]]), 3) is False              # node 3 used before it exists
    assert T.valid_tree(np.array([[0, 1], [1, 3]]), 3) is False
    assert T.valid_tree(np.array([[0, 1], [3, 2]]), 3) and T.valid_tree(np.array([[0, 1], [2, 3]]), 3)


@pytest.mark.parametrize("cap,n,case", [c for c in T.CRAFT_CASES if c[1] < 4000],
                         ids=[f"{c}-{n}-cap{k}" for k, n, c in T.CRAFT_CASES if n < 4000])
def test_crafted_first_merges(cap, n, case):
    lcs, lens = T.craft_coop(n, case, cap)
    want = T.craft_first_merges(n, case, cap)
    for modified in (False, True):
        got = U.expected_tree(0, modified, lcs, lens)
        assert [tuple(m) for m in got[:len(want)].tolist()] == want, modified


def restated_vs_vectorised(codes, offsets, lens, kind, prune, exact=()):
    want = prim_restated(codes, offsets, lens, kind, prune=prune)
    rows = T.LcsRows(P.lcs_triangle(codes, offsets, lens), codes, offsets, lens, exact)
    got = T.prim_vectorised(rows, lens, kind, prune=prune)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    return got


def host_sets():
    rng = np.random.default_rng(5)
    out = {"family": (*seqio.synth_family(150, 60, seed=6), [])}
    out["abc3"] = (*seqio.pack(U.famsa_sorted([c for c in random_set(rng, 120, 5, 30, alphabet=3,
                                                                          with_specials=False)])), [])
    base = random_set(rng, 15, 5, 20, alphabet=4, with_specials=False)
    out["dups"] = (*seqio.pack([base[i % 15] for i in rng.permutation(120)]), [])
    for name in ("carry_sorted", "carry_shuffled"):
        codes, offsets, lens = U.sequence_set(name)
        out[name] = (codes, offsets, lens, [int(i) for i in np.flatnonzero(lens >= 64)])
    return out


@pytest.mark.parametrize("prune", [True, False])
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", ["family", "abc3", "dups", "carry_sorted", "carry_shuffled"])
def test_vectorised_prim_equals_restatement(case, kind, prune):
    codes, offsets, lens, exact = host_sets()[case]
    restated_vs_vectorised(codes, offsets, lens, kind, prune, exact)


def test_vectorised_prim_carry_generator():
    """A cooperative-case carry set at a reduced size: flagged rows away from the start, rows and columns from the oracle."""
    codes, offsets, lens, exact = T.sequence_set("carry", 300, 1)
    for kind in (0, 1):
        restated_vs_vectorised(codes, offsets, lens, kind, True, exact)


def test_vectorised_prim_pruning_fixture():
    z = np.load(os.path.join(GOLDEN, "prim_pruning_case.npz"))
    codes, offsets, lens = seqio.pack([seqio.encode(str(s)) for s in z["seqs"]])
    exact = list(range(len(lens)))
    ef, et, ed, order = T.prim_vectorised(T.LcsRows(P.lcs_triangle(codes, offsets, lens), codes, offsets, lens, exact),
                                          lens, 0)
    assert np.array_equal(ef, z["edge_from"]) and np.array_equal(et, z["edge_to"])
    assert np.array_equal(ed, z["edge_dist"]) and np.array_equal(order, z["prim_order"])


def test_vectorised_prim_equals_kruskal_replay():
    """Without flagged sequences the vectorised loop's edges and order are the unique MST under (distance, key) replayed
    from vertex 0: what the Boruvka rounds are compared with."""
    codes, offsets, lens = seqio.synth_family(400, 50, seed=9)
    tri = P.lcs_triangle(codes, offsets, lens)
    for kind in (0, 1):
        n = len(lens)
        want = mst.prim_replay(n, mst.kruskal_total_order(n, T.distance_triangle_f64(kind, tri, lens)))
        got = T.prim_vectorised(T.LcsRows(tri, codes, offsets, lens), lens, kind)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)


@pytest.mark.skipif(not P.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")
@pytest.mark.parametrize("case", ["family", "abc3", "carry_sorted", "carry_shuffled"])
def test_vectorised_prim_gives_reference_tree(case):
    codes, offsets, lens, exact = host_sets()[case]
    ef, et, ed, order = T.prim_vectorised(T.LcsRows(P.lcs_triangle(codes, offsets, lens), codes, offsets, lens, exact),
                                          lens, 0)
    letters = U.letters_of(codes, offsets, lens)
    assert np.array_equal(P.mst_to_dendogram(ef, et, ed, order), P.RefSeqSet(letters).mst_prim_tree(2))
