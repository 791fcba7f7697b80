"""famsa_lcs_upgma and famsa_lcs_upgma_from_triangle on the device against the restated UPGMA<>::computeTree
(oracle/upgma_oracle.c) pair for pair, at the edges of the cooperative kernel k_upgma: both distance kinds and averaging
rules, both entry points and triangle widths, ties inside and across blocks of 1024 rows, the last row of the last
block, more than 32 blocks (n = 32 769: the candidate gather loops), a 4-byte internal triangle, the witness fixture
(stale cache, float rounding of the MAFFT average, ties), the no-finite-distance error and reuse of the context.

The restatement runs on the host float Transform of the LCS triangle the device reads: the C oracle's triangle for small
sets, the device's own triangle downloaded for large ones (the triangle itself is checked by test_lcs_gpu.py).  Where
oracle/_ref is built, sets of real sequences are also compared with the reference's own UPGMA run (kind 0)."""
import functools

import numpy as np
import pytest
import torch

from conftest import random_set
from famsa_b200 import seqio
from famsa_b200.binding import FamsaError
from oracle import pyoracle as P
import upgma_cases as U

pytestmark = pytest.mark.gpu


def device_triangle(lcs, eb):
    """A packed LCS triangle in a CUDA tensor of element width eb (the library reads it as unsigned)."""
    a = np.ascontiguousarray(lcs, dtype=np.uint16 if eb == 2 else np.uint32)
    t = torch.from_numpy(a.view(np.int16 if eb == 2 else np.int32)).to("cuda")
    torch.cuda.synchronize()
    return t


def tree_from_triangle(engine, kind, modified, t):
    return engine.upgma(kind, modified, t.data_ptr(), t.element_size())


def upload_lens(engine, lens):
    """Sequences of the given lengths (their residues do not matter to _from_triangle: it reads only the lengths)."""
    engine.upload(*seqio.pack([np.arange(int(n), dtype=np.int8) % 20 for n in lens]))


@functools.lru_cache(maxsize=None)
def small_set(case):
    codes, offsets, lens = U.sequence_set(case)
    return codes, offsets, lens, U.oracle_triangle(codes, offsets, lens)


@pytest.mark.parametrize("entry", ["upgma", "triangle2", "triangle4"])
@pytest.mark.parametrize("modified", [False, True])
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", U.SETS)
def test_sets(engine, case, kind, modified, entry):
    """famsa_lcs_upgma, and _from_triangle on the triangle famsa_lcs_triangle_device wrote at 2 and 4 bytes."""
    codes, offsets, lens, lcs = small_set(case)
    n = len(lens)
    want = U.expected_tree(kind, modified, lcs, lens)
    engine.upload(codes, offsets, lens)
    if entry == "upgma":
        got = engine.upgma(kind, modified)
        assert engine.last_timing()[2] == n * (n - 1) // 2
    else:
        eb = int(entry[-1])
        t = torch.empty(n * (n - 1) // 2, dtype=torch.int16 if eb == 2 else torch.int32, device="cuda")
        engine.triangle_device(0, n, t.data_ptr(), eb)
        got = tree_from_triangle(engine, kind, modified, t)
    assert got.shape == (n - 1, 2) and np.array_equal(got, want)
    if kind == 0 and entry == "upgma" and P.have_ref():
        ref = P.RefSeqSet(U.letters_of(codes, offsets, lens)).upgma_tree(modified)[n:]
        assert np.array_equal(got, ref)


@pytest.mark.parametrize("case,n", U.CRAFTED, ids=[f"{c}-{n}" for c, n in U.CRAFTED])
def test_crafted_triangles(engine, case, n):
    """Chosen LCS values through _from_triangle at 2 and 4 bytes, both averaging rules: sizes around the 32-row warp
    and the 1024-row block, equal minima at the same offset of three blocks, the unique minimum in the last row, a stale
    cache that puts two consecutive minima in the last row, and a three-way new-row tie across blocks."""
    lcs, lens = U.craft(n, case, seed=n)
    upload_lens(engine, lens)
    for modified in (False, True):
        want = U.expected_tree(0, modified, lcs, lens)
        if case == "stale":
            assert [tuple(m) for m in want[:2].tolist()] == [(0, 1), (n - 1, n)]
        if case == "block_tie":
            assert tuple(want[0]) == (3, 1027)
        if case == "new_tie":
            assert [tuple(m) for m in want[:2].tolist()] == [(0, 1), (n, 700)]
        for eb in (2, 4):
            got = tree_from_triangle(engine, 0, modified, device_triangle(lcs, eb))
            assert np.array_equal(got, want), (modified, eb)


@pytest.mark.parametrize("eb", [2, 4])
def test_witness_cases(engine, eb):
    """Every case of upgma_witness.npz: the reference's tree, which the stale-cache-free, once-rounded and fused
    variants (and reversed tie-breaking) do not reproduce."""
    for name, c in U.witness_cases().items():
        upload_lens(engine, c["lens"])
        got = tree_from_triangle(engine, c["kind"], c["modified"], device_triangle(c["lcs"], eb))
        assert np.array_equal(got, c["tree"]), name


def test_more_than_32_blocks_crafted(engine):
    """n = 32 769 rows take 33 blocks of 1024: the block holding row 32 768 is the 33rd, whose candidate the gather reaches
    only on its second pass over the blocks.  (0, 1) closest and (1, 32 768) next: the first new row's minimum is row
    32 768, and so is the next merge's (its cache was relabelled from 1 to 0 and kept the smaller distance).  About 1 GB
    of uint16 triangle, built on the host."""
    n = U.BIG_N
    lcs, lens = U.craft(n, "stale")
    upload_lens(engine, lens)
    t = device_triangle(lcs, 2)
    got = tree_from_triangle(engine, 0, False, t)
    del t
    torch.cuda.empty_cache()
    want = U.expected_tree(0, False, lcs, lens)
    assert [tuple(m) for m in want[:2].tolist()] == [(0, 1), (n - 1, n)]
    assert np.array_equal(got, want)


def test_more_than_32_blocks_real_set(engine):
    """synth_family(33000, 40) through famsa_lcs_upgma (modified average), against the restatement on the device's
    own triangle, downloaded."""
    codes, offsets, lens = seqio.synth_family(33000, 40, seed=73)
    n = len(lens)
    engine.upload(codes, offsets, lens)
    got = engine.upgma(0, True)
    lcs = engine.triangle(dtype=np.uint16)
    assert np.array_equal(got, U.expected_tree(0, True, lcs, lens))


@pytest.mark.parametrize("modified", [False, True])
@pytest.mark.parametrize("kind", [0, 1])
def test_four_byte_internal_triangle(engine, kind, modified):
    """A sequence of 70 000 residues makes the triangle famsa_lcs_upgma builds 4 bytes wide."""
    rng = np.random.default_rng(74)
    cl = [rng.integers(0, 20, 70000).astype(np.int8)] + U.famsa_sorted(random_set(rng, 30, 20, 80, with_specials=False))
    codes, offsets, lens = seqio.pack(cl)
    engine.upload(codes, offsets, lens)
    got = engine.upgma(kind, modified)
    assert np.array_equal(got, U.expected_tree(kind, modified, U.oracle_triangle(codes, offsets, lens), lens))


def test_no_finite_distance_then_reuse(engine):
    """A sequence sharing no residue with the others: the agglomeration runs out of finite distances, the call returns
    FAMSA_E_INVALID with its message (both entry points), and the same context then builds the right trees -- a valid set,
    a large set followed by a smaller one, and two upgma calls with prim and slink between them."""
    rng = np.random.default_rng(75)
    cl = [c for c in random_set(rng, 8, 10, 40, alphabet=10, with_specials=False)] + [np.full(12, 15, np.int8)]
    engine.upload(*seqio.pack(cl))
    for kind in (0, 1):
        with pytest.raises(FamsaError, match="no finite distance"):
            engine.upgma(kind, False)
    rc, _ = U.restated_tree(0, False, U.oracle_triangle(*seqio.pack(cl)), np.array([len(c) for c in cl], np.uint32))
    assert rc == 1
    lcs, lens = U.craft(40, "random", seed=3)
    upload_lens(engine, lens)
    # one pair without a common residue does not always end the agglomeration: a stale cache can still hold a finite
    # distance to the cluster whose true distance is FLT_MAX, and the reference merges through it
    lcs[U.tri_index(39, 7)] = 0
    rc, want = U.restated_tree(0, True, lcs, lens)
    assert rc == 0
    assert np.array_equal(tree_from_triangle(engine, 0, True, device_triangle(lcs, 2)), want)
    # a sequence sharing nothing with any other always does: no cache ever points at it
    lcs[[U.tri_index(39, j) for j in range(39)]] = 0
    assert U.restated_tree(0, True, lcs, lens)[0] == 1
    with pytest.raises(FamsaError, match="no finite distance"):
        tree_from_triangle(engine, 0, True, device_triangle(lcs, 2))

    codes, offsets, lens, lcs = small_set("ragged")
    engine.upload(codes, offsets, lens)
    assert np.array_equal(engine.upgma(0, False), U.expected_tree(0, False, lcs, lens))

    big = seqio.synth_family(3000, 60, seed=76)
    engine.upload(*big)
    assert np.array_equal(engine.upgma(1, True), U.expected_tree(1, True, engine.triangle(dtype=np.uint16), big[2]))
    codes, offsets, lens, lcs = small_set("family400")
    engine.upload(codes, offsets, lens)
    want = U.expected_tree(0, True, lcs, lens)
    assert np.array_equal(engine.upgma(0, True), want)
    engine.prim(0)
    engine.slink(1)
    assert np.array_equal(engine.upgma(0, True), want)
