"""The UPGMA oracle on the host: the restated UPGMA<>::computeTree (oracle/upgma_oracle.c) against the reference's own
computeTree pair for pair (where oracle/_ref is built), its no-finite-distance status, the batch float Transform against
the scalar ones, and the witness fixture (tests/golden/make_upgma.py)."""
import numpy as np
import pytest

from conftest import GOLDEN, random_set
from famsa_b200 import seqio
from oracle import pyoracle as P
import upgma_cases as U

need_ref = pytest.mark.skipif(not P.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")
NEVER = np.float32(np.nextafter(np.float64(np.finfo(np.float32).max), 0.0))     # Transform of LCS 0


def against_reference(dist, n, modified):
    rc, got = P.upgma_tree(dist, n, modified)
    assert rc == 0
    want = P.upgma_tree_from_distances(dist, n, modified)[n:]
    assert got.shape == (n - 1, 2) and np.array_equal(got, want)


@need_ref
@pytest.mark.parametrize("modified", [False, True])
@pytest.mark.parametrize("values", ["uniform", "few", "few_and_zeros"])
def test_restatement_matches_reference_on_random_triangles(modified, values):
    """n = 2..300: continuous distances, and heavy exact ties (every distance one of five floats, with and without
    zeros), where the first-minimum scans and the stale cache decide the tree."""
    rng = np.random.default_rng({"uniform": 1, "few": 2, "few_and_zeros": 3}[values])
    sizes = list(range(2, 34)) + [63, 64, 65, 100, 128, 177, 255, 300]
    palette = {"few": np.array([0.5, 0.625, 0.75, 1.0, 1.5], np.float32),
               "few_and_zeros": np.array([0.0, 0.0, 0.25, 0.5, 1.0], np.float32)}
    for n in sizes:
        m = n * (n - 1) // 2
        dist = rng.random(m).astype(np.float32) if values == "uniform" else rng.choice(palette[values], size=m)
        against_reference(dist, n, modified)


def adeno_triangle():
    z = np.load(f"{GOLDEN}/adeno_fiber_lcs.npz")
    seqs = [str(s) for s in z["seqs"]]
    order = sorted(range(len(seqs)), key=lambda i: (-len(seqs[i]), seqio.encode(seqs[i]).tobytes()))
    lcs = z["lcs"].astype(np.uint32)[np.ix_(order, order)]                  # row = seq0, in FAMSA's order
    i, j = np.tril_indices(len(order), -1)
    return lcs[i, j], np.array([len(seqio.encode(seqs[k])) for k in order], np.uint32)


@need_ref
@pytest.mark.parametrize("modified", [False, True])
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", ["adeno", "ragged", "carry_sorted", "carry_shuffled", "twice"])
def test_restatement_matches_reference_on_lcs_sets(case, kind, modified):
    """Triangles of real LCS lengths: adeno_fiber (golden pid_sq.csv), a ragged tie-heavy set, the dropped-carry set
    with row = seq0 (its triangle is not symmetric in the pair's order) and every sequence twice (zero distances)."""
    if case == "adeno":
        lcs, lens = adeno_triangle()
    else:
        codes, offsets, lens = U.sequence_set(case)
        lcs = U.oracle_triangle(codes, offsets, lens)
    against_reference(P.transform_triangle(kind, lcs, lens), len(lens), modified)


@need_ref
@pytest.mark.parametrize("modified", [False, True])
def test_restatement_matches_the_reference_run(modified):
    """The reference's whole UPGMA<indel075_div_lcs>::run on a ragged set equals the restatement on the oracle's
    LCS triangle: computeDistances is the batch Transform."""
    codes, offsets, lens = U.sequence_set("ragged")
    want = P.RefSeqSet(U.letters_of(codes, offsets, lens)).upgma_tree(modified)[len(lens):]
    assert np.array_equal(U.expected_tree(0, modified, U.oracle_triangle(codes, offsets, lens), lens), want)


@pytest.mark.parametrize("modified", [False, True])
def test_no_finite_distance_is_reported(modified):
    """A pair without a common residue has distance FLT_MAX; every average with it stays >= BIG_DIST = 1e29, so once
    only such pairs are left no row has a finite cached distance.  The reference would index out of range there; the
    restatement stops with status 1 after the merges it could make."""
    n = 6
    lcs = np.full(n * (n - 1) // 2, 30, np.uint32)
    for j in range(n - 1):
        lcs[U.tri_index(n - 1, j)] = 0                                      # the last sequence shares nothing
    rc, tree = U.restated_tree(0, modified, lcs, np.full(n, 50, np.uint32))
    assert rc == 1 and tree.shape == (n - 2, 2)
    assert (n - 1) not in set(tree.ravel().tolist())
    rc, tree = P.upgma_tree(np.full(n * (n - 1) // 2, NEVER, np.float32), n, modified)
    assert rc == 1 and tree.shape == (0, 2)
    # a finite distance left behind a cache that holds FLT_MAX: two clusters with no common residue, each solvable
    lcs = np.zeros(n * (n - 1) // 2, np.uint32)
    for a, b in ((1, 0), (2, 0), (2, 1), (4, 3), (5, 3), (5, 4)):
        lcs[U.tri_index(a, b)] = 20
    rc, tree = U.restated_tree(1, modified, lcs, np.full(n, 50, np.uint32))
    assert rc == 1 and tree.shape == (4, 2)


@need_ref
@pytest.mark.parametrize("modified", [False, True])
def test_one_unrelated_pair_merges_through_the_stale_cache(modified):
    """One pair without a common residue need not end the agglomeration: a row's stale cache can keep a finite
    distance to a cluster whose true distance is FLT_MAX, and the reference merges through it.  The restatement does
    the same, merge for merge."""
    lcs, lens = U.craft(40, "random", seed=3)
    lcs[U.tri_index(39, 7)] = 0
    dist = P.transform_triangle(0, lcs, lens)
    assert (dist >= 1e29).sum() == 1
    against_reference(dist, 40, modified)


def transform_grid():
    """Lengths 1..9 and 64/65/200, with LCS 0, LCS = the shorter length (indel 0 for equal lengths) and values between."""
    rng = np.random.default_rng(8)
    lens = np.array([1, 1, 2, 3, 5, 5, 8, 9, 64, 64, 65, 200, 200, 7], np.uint32)
    n = len(lens)
    lcs = np.zeros(n * (n - 1) // 2, np.uint32)
    for i in range(1, n):
        for j in range(i):
            short = int(min(lens[i], lens[j]))
            lcs[U.tri_index(i, j)] = (0, short, int(rng.integers(0, short + 1)))[(i + j) % 3]
    return lcs, lens


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.uint16, np.uint32])
def test_batch_transform_matches_scalar(kind, dtype):
    lcs, lens = transform_grid()
    got = P.transform_triangle(kind, lcs.astype(dtype), lens)
    n = len(lens)
    i, j = np.tril_indices(n, -1)
    want = np.array([P.transform(kind, int(l), int(lens[a]), int(lens[b]), double=False)
                     for l, a, b in zip(lcs, i, j)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))                # bit for bit
    assert (lcs == 0).any() and (lcs == np.minimum(lens[i], lens[j])).any() and (lens[i] == lens[j]).any()
    if kind != 2:
        assert (got[lcs == 0] == NEVER).all()
    if P.have_ref():
        ref = np.array([P.ref().ref_transform_f32(kind, int(l), int(lens[a]), int(lens[b]))
                        for l, a, b in zip(lcs, i, j)], np.float32)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_batch_transform_on_a_dropped_carry_set():
    """LCS lengths above the shorter length (a flagged sequence as the row, after a shorter one): the table lookup
    agrees with pow."""
    codes, offsets, lens = U.sequence_set("carry_shuffled")
    lcs = U.oracle_triangle(codes, offsets, lens)
    i, j = np.tril_indices(len(lens), -1)
    assert (lcs > np.minimum(lens[i], lens[j])).any()
    for kind in (0, 1):
        want = np.array([P.transform(kind, int(l), int(lens[a]), int(lens[b]), double=False)
                         for l, a, b in zip(lcs, i, j)], np.float32)
        assert np.array_equal(P.transform_triangle(kind, lcs, lens), want)


@pytest.mark.parametrize("name", ["stale", "stale_modified", "rounded_once", "rounded_once_kind1", "fused", "fused_kind1",
                                  "cross_tie"])
def test_witness_fixture(name):
    """Each witness: the restatement rebuilds the stored tree, and the variant it witnesses against builds another
    (cross_tie: the same triangle with the sequences in reverse order has different clades)."""
    c = U.witness_cases()[name]
    n = len(c["lens"])
    assert 6 <= n <= 16
    dist = P.transform_triangle(c["kind"], c["lcs"], c["lens"])
    rc, tree = P.upgma_tree(dist, n, c["modified"])
    assert rc == 0 and np.array_equal(tree, c["tree"])
    if name in U.WITNESS_VARIANT:
        rc, other = P.upgma_tree(dist, n, c["modified"], **U.WITNESS_VARIANT[name])
        assert rc == 0 and not np.array_equal(other, tree)
    else:
        assert np.count_nonzero(dist == dist.min()) >= 3
    if P.have_ref():
        assert np.array_equal(P.upgma_tree_from_distances(dist, n, c["modified"])[n:], tree)
