"""Generates tests/golden/upgma_witness.npz: small LCS triangles (plus sequence lengths) on which the reference's UPGMA
agglomeration (UPGMA<>::computeTree, src/tree/UPGMA.cpp:114-295) gives a different tree from a plausible alternative.
A kernel that drifts towards the alternative then fails on them.

Run where oracle/_ref is built:  python tests/golden/make_upgma.py   (seeded: rewrites the file byte for byte)

Cases (each stored as <case>_lcs (uint32 packed triangle, row i at i(i-1)/2), <case>_lens, <case>_kind,
<case>_modified and <case>_tree, the reference's n-1 merges):
  stale, stale_modified     the nearest-neighbour cache as the reference keeps it (a row whose neighbour was merged away
                            is relabelled and keeps its old distance) gives a different tree from a cache refreshed
                            after every merge.
  rounded_once, rounded_once_kind1
                            the MAFFT average 0.05f*(x+y) + 0.9f*min(x,y) rounded after each product and the sum (as the
                            reference's build evaluates it) gives a different tree from the same average rounded once.
  fused, fused_kind1        ... and from fmaf(0.05f, x+y, 0.9f*min(x,y)).
  cross_tie                 the first merges are decided by ties: the minimum distance is shared by several pairs, and
                            the tree of the same triangle with the sequences in reverse order has different clades.
Generation asserts, for every case, that the reference's computeTree equals the restatement (oracle/upgma_oracle.c)
and differs from the variant.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import pyoracle as P  # noqa: E402

OUT = os.path.join(HERE, "upgma_witness.npz")


def reference_tree(dist, n, modified):
    return P.upgma_tree_from_distances(dist, n, modified)[n:]


def restated(dist, n, modified, **variant):
    rc, tree = P.upgma_tree(dist, n, modified, **variant)
    assert rc == 0
    return tree


def clades(n, merges):
    sets = [frozenset([i]) for i in range(n)]
    for a, b in merges:
        sets.append(sets[a] | sets[b])
    return set(sets[n:])


def random_lcs(rng, lens):
    n = len(lens)
    out = np.zeros(n * (n - 1) // 2, dtype=np.uint32)
    for i in range(1, n):
        for j in range(i):
            out[i * (i - 1) // 2 + j] = rng.integers(1, min(lens[i], lens[j]) + 1)
    return out


def two_valued_lcs(rng, n, length):
    vals = rng.choice(np.arange(5, length), size=2, replace=False)
    return rng.choice(vals, size=n * (n - 1) // 2).astype(np.uint32), np.full(n, length, dtype=np.uint32)


def reverse_order(lcs, n):
    """The same pairs with sequence i renamed n-1-i (packed triangle of the reversed set)."""
    out = np.zeros_like(lcs)
    for i in range(1, n):
        for j in range(i):
            a, b = n - 1 - j, n - 1 - i                                      # a > b
            out[a * (a - 1) // 2 + b] = lcs[i * (i - 1) // 2 + j]
    return out


def search(seed, draw, differs, tries=20000):
    rng = np.random.default_rng(seed)
    for t in range(tries):
        lcs, lens, kind, modified = draw(rng)
        n = len(lens)
        dist = P.transform_triangle(kind, lcs, lens)
        want = reference_tree(dist, n, modified)
        assert np.array_equal(restated(dist, n, modified), want), "restatement differs from the reference"
        if differs(lcs, lens, kind, modified, dist, want):
            return t, dict(lcs=lcs, lens=lens, kind=np.array(kind), modified=np.array(int(modified)), tree=want)
    raise SystemExit(f"no witness for seed {seed}")


def main():
    if not P.have_ref():
        raise SystemExit("oracle/_ref is not built")
    cases = {}

    def stale_draw(modified, kind):
        def draw(rng):
            n = int(rng.integers(6, 17))
            lens = rng.integers(20, 60, size=n).astype(np.uint32)
            return random_lcs(rng, lens), lens, kind, modified
        return draw

    def differs_from(**variant):
        def differs(lcs, lens, kind, modified, dist, want):
            return not np.array_equal(restated(dist, len(lens), modified, **variant), want)
        return differs

    def rounding_draw(kind):
        def draw(rng):
            n = int(rng.integers(6, 17))
            lcs, lens = two_valued_lcs(rng, n, int(rng.integers(20, 60)))
            return lcs, lens, kind, True
        return draw

    def cross_tie_draw(rng):
        n = int(rng.integers(6, 17))
        lcs, lens = two_valued_lcs(rng, n, int(rng.integers(20, 60)))
        return lcs, lens, 0, False

    def ties_decide(lcs, lens, kind, modified, dist, want):
        n = len(lens)
        if np.count_nonzero(dist == dist.min()) < 3:
            return False
        rev = reverse_order(lcs, n)
        back = [(n - 1 - a if a < n else a, n - 1 - b if b < n else b) for a, b in restated(P.transform_triangle(kind, rev, lens), n, modified)]
        return clades(n, back) != clades(n, [tuple(int(x) for x in m) for m in want])

    plan = [("stale", 1, stale_draw(False, 0), differs_from(fresh_cache=True)),
            ("stale_modified", 2, stale_draw(True, 1), differs_from(fresh_cache=True)),
            ("rounded_once", 3, rounding_draw(0), differs_from(avg_mode=P.UPGMA_AVG_ROUNDED_ONCE)),
            ("rounded_once_kind1", 4, rounding_draw(1), differs_from(avg_mode=P.UPGMA_AVG_ROUNDED_ONCE)),
            ("fused", 5, rounding_draw(0), differs_from(avg_mode=P.UPGMA_AVG_FUSED)),
            ("fused_kind1", 6, rounding_draw(1), differs_from(avg_mode=P.UPGMA_AVG_FUSED)),
            ("cross_tie", 7, cross_tie_draw, ties_decide)]
    for name, seed, draw, differs in plan:
        t, case = search(seed, draw, differs)
        for k, v in case.items():
            cases[f"{name}_{k}"] = v
        print(f"{name}: try {t}, n = {len(case['lens'])}, kind {int(case['kind'])}, modified {int(case['modified'])}")
    np.savez_compressed(OUT, names=np.array([p[0] for p in plan]), **cases)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
