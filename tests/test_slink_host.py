"""CPU tests of famsa_b200.mst.slink_tree: SingleLinkage<d>::run with SLINK_HANDLE_TIES orders distances strictly (the
order of kruskal_total_order), so its tree is the unique MST merged in Kruskal order and labelled by the largest member
of each side.  Checked against a verbatim restatement of the reference's pointer loops (tests/slink_oracle.py) on
random triangles full of ties, and on the committed adeno fixture from its LCS values alone.  Also compiles the C++
mirror's SingleLinkageTree case."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from famsa_b200 import mst, seqio
from oracle import pyoracle
import slink_oracle as S
from cpp_build import build_cpp

NEVER = float(np.nextafter(S.DBL_MAX, 0.0))      # Transform's distance for LCS 0


def random_triangle(rng, n, kind, max_len):
    """Distances of random (LCS, lengths) through the oracle's Transform<double, kind>: few distinct values, LCS 0 included."""
    lens = rng.integers(1, max_len + 1, size=n)
    ii, jj = np.tril_indices(n, -1)
    lcs = (rng.random(len(ii)) * (np.minimum(lens[ii], lens[jj]) + 1)).astype(np.int64)
    cache = {}
    out = np.empty(len(ii), dtype=np.float64)
    for e, key in enumerate(zip(lcs.tolist(), lens[ii].tolist(), lens[jj].tolist())):
        if key not in cache:
            cache[key] = pyoracle.transform(kind, *key, True)
        out[e] = cache[key]
    return out


SIZES = [1, 2, 3, 4, 5, 7, 8, 13, 31, 32, 33, 64, 100, 300]


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("n", SIZES)
def test_mst_labelling_equals_restated_slink(n, kind):
    rng = np.random.default_rng(1000 * kind + n)
    for max_len in (1, 2, 4):
        tri = random_triangle(rng, n, kind, max_len)
        assert n < 8 or len(np.unique(tri)) < len(tri) // 2               # ties are the rule
        got = mst.slink_tree(n, mst.kruskal_total_order(n, tri))
        assert [tuple(int(x) for x in r) for r in got] == S.slink_restated(n, tri)


@pytest.mark.parametrize("value", [0.0, 0.5, NEVER])
@pytest.mark.parametrize("n", [1, 2, 9, 40, 120])
def test_all_distances_equal(n, value):
    """Only the pair order decides; NEVER is what Transform gives sequences without a common residue."""
    tri = np.full(n * (n - 1) // 2, value)
    got = mst.slink_tree(n, mst.kruskal_total_order(n, tri))
    assert [tuple(int(x) for x in r) for r in got] == S.slink_restated(n, tri)


def test_lcs_zero_next_to_finite_distances():
    rng = np.random.default_rng(3)
    n = 60
    tri = np.where(rng.random(n * (n - 1) // 2) < 0.7, NEVER, rng.integers(0, 3, n * (n - 1) // 2) / 4.0)
    got = mst.slink_tree(n, mst.kruskal_total_order(n, tri))
    assert [tuple(int(x) for x in r) for r in got] == S.slink_restated(n, tri)


@pytest.mark.parametrize("kind", [0, 1])
def test_adeno_fixture_from_golden_lcs(kind):
    """adeno_slink_tree.npz holds the reference's tree (kind 0), checked at generation against slink.dnd.  Here it is
    rebuilt from the LCS values of adeno_fiber_lcs.npz (pid_sq.csv, row = seq0) by the restatement and by the MST
    labelling; kind 1 has no golden, so the two only have to agree."""
    z = np.load(os.path.join(GOLDEN, "adeno_slink_tree.npz"))
    lz = np.load(os.path.join(GOLDEN, "adeno_fiber_lcs.npz"))
    where = {str(s): i for i, s in enumerate(lz["seqs"])}
    idx = np.array([where[str(s)] for s in z["seqs"]])
    lcs = lz["lcs"][np.ix_(idx, idx)]
    lens = np.array([len(seqio.encode(str(s))) for s in z["seqs"]])
    n = len(lens)
    tri = S.slink_distances(lcs, lens, kind)
    want = S.slink_restated(n, tri)
    assert [tuple(int(x) for x in r) for r in mst.slink_tree(n, mst.kruskal_total_order(n, tri))] == want
    if kind == 0:
        assert [tuple(int(x) for x in r) for r in z["tree"]] == want


def test_host_mirror_slink_compiles(tmp_path):
    build_cpp("test_host_slink", tmp_path, famsa=True)
