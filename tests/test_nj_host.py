"""CPU tests of the restated NeighborJoining<>::computeTree (oracle/nj_oracle.c), the yardstick of famsa_lcs_nj.

Where oracle/_ref is built, the restatement is compared merge for merge with the reference's own computeTree (through a
derived class in oracle/ref_nj_harness.cpp) on random triangles, tie-heavy triangles (small integer distances, duplicate
rows), triangles with FLT_MAX entries whose q values are -inf and NaN, n = 2, 3, 4, and the step without a candidate,
where the restatement reports what the reference turns into a cluster merged with itself; and the reference's run end to
end with the restatement on the oracle's distances.  The adeno fixture is rebuilt by the restatement everywhere.
Also compiles the C++ mirror's NeighborJoiningTree case."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, random_set
from famsa_b200 import seqio
from oracle import pyoracle as P
import nj_oracle as N
import upgma_cases as U
from cpp_build import build_cpp

need_ref = pytest.mark.skipif(not P.have("ref_nj"), reason="oracle/_ref/libfamsa_ref_nj.so not built")
FLT_MAX = np.float32(N.FLT_MAX)


def tri_size(n):
    return n * (n - 1) // 2


def random_triangle(rng, n, values):
    m = tri_size(n)
    if values == "float":
        return rng.random(m, dtype=np.float32) * np.float32(3)
    if values == "small_int":
        return rng.integers(0, 4, m).astype(np.float32)
    if values == "duplicate_rows":                       # sequences in groups of equal rows: D = 0 inside, equal outside
        g = rng.integers(0, max(2, n // 3), n)
        ii, jj = np.tril_indices(n, -1)
        base = rng.integers(1, 5, (n, n)).astype(np.float32)
        base = np.minimum(base, base.T)
        return np.where(g[ii] == g[jj], np.float32(0), base[g[ii], g[jj]]).astype(np.float32)
    if values == "flt_max":                              # Transform's "no common residue" next to ordinary distances
        t = rng.integers(1, 6, m).astype(np.float32) / np.float32(4)
        t[rng.random(m) < 0.3] = FLT_MAX
        return t
    raise KeyError(values)


@need_ref
@pytest.mark.parametrize("values", ["float", "small_int", "duplicate_rows", "flt_max"])
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8, 33, 64, 65, 130, 200])
def test_restatement_matches_reference_on_triangles(n, values):
    rng = np.random.default_rng(7 * n + len(values))
    for _ in range(3):
        tri = random_triangle(rng, n, values)
        rc, got = N.restated(tri, n)
        want = N.ref_tree_from_distances(tri, n)
        if rc == 0:
            assert np.array_equal(got, want)
        else:                                            # the reference's step without a candidate: cluster 0 with itself
            k = len(got)
            assert np.array_equal(got, want[:k]) and want[k, 0] == want[k, 1]


@need_ref
def test_one_unrelated_sequence_gives_minus_inf():
    """One row of FLT_MAX among finite distances: that row's sum overflows to +inf, so every ordinary pair has q = -inf
    (the first one wins) and the pairs of the unrelated row have q = NaN."""
    rng = np.random.default_rng(5)
    n = 12
    ii, jj = np.tril_indices(n, -1)
    tri = (rng.integers(1, 8, tri_size(n)) / 8).astype(np.float32)
    tri[(ii == 5) | (jj == 5)] = FLT_MAX
    rc, got = N.restated(tri, n)
    assert rc == 0 and tuple(got[0]) == (0, 1)
    assert np.array_equal(got, N.ref_tree_from_distances(tri, n))


@need_ref
@pytest.mark.parametrize("n", [4, 5, 9])
def test_no_candidate_is_reported(n):
    """All distances FLT_MAX (no two sequences share a residue): the sums overflow, q = inf - inf = NaN for every pair, so
    the first step has no candidate.  The reference merges cluster 0 with itself there; the restatement returns 1."""
    tri = np.full(tri_size(n), FLT_MAX, dtype=np.float32)
    rc, got = N.restated(tri, n)
    assert rc == 1 and len(got) == 0
    assert tuple(N.ref_tree_from_distances(tri, n)[0]) == (0, 0)


def test_three_unrelated_sequences_still_join():
    """n = 3 has q = FLT_MAX - inf - inf = -inf, a candidate: no error below four sequences."""
    rc, got = N.restated(np.full(3, FLT_MAX, dtype=np.float32), 3)
    assert rc == 0 and [tuple(r) for r in got] == [(0, 1), (3, 2)]


def random_sorted_set(alphabet):
    rng = np.random.default_rng(90 + alphabet)
    return seqio.pack(U.famsa_sorted(random_set(rng, 120, 5, 60, alphabet=alphabet, with_specials=False)))


@need_ref
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", ["random3", "random20", "twice", "carry_sorted", "carry_shuffled", "n2", "n3"])
def test_reference_run_matches_restatement(case, kind):
    """NeighborJoining<kind>::run end to end against the restatement on the oracle's float Transform of the oracle's LCS
    triangle (row = seq0, the triangle calculateDistanceMatrix fills)."""
    if case.startswith("random"):
        codes, offsets, lens = random_sorted_set(int(case[6:]))
    else:
        codes, offsets, lens = U.sequence_set(case)
    letters = U.letters_of(codes, offsets, lens)
    rc, want = N.restated(P.transform_triangle(kind, P.lcs_triangle(codes, offsets, lens), lens), len(lens))
    got, _ = N.ref_tree(letters, kind)
    assert rc == 0 and np.array_equal(got, want)


@pytest.mark.parametrize("kind", [0, 1])
def test_adeno_fixture_matches_restatement(kind):
    """adeno_nj_tree.npz from the oracle's LCS alone (generation asserts the same for hemopexin_nj.npz, whose
    restatement takes minutes on one core)."""
    z = np.load(os.path.join(GOLDEN, "adeno_nj_tree.npz"))
    codes, offsets, lens = seqio.pack([seqio.encode(str(s)) for s in z["seqs"]])
    rc, want = N.restated(P.transform_triangle(kind, P.lcs_triangle(codes, offsets, lens), lens), len(lens))
    assert rc == 0 and np.array_equal(z[f"tree{kind}"], want)


def test_host_mirror_nj_compiles(tmp_path):
    build_cpp("test_host_nj", tmp_path, famsa=True)
