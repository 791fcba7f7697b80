"""famsa_prof_refine (CFAMSA::RefineAlignment as with no_threads > 1) against the reference's own CProfile run through
oracle/ref_refine_harness.cpp: refined rows, width, total score and the loop's counts."""
from __future__ import annotations

import numpy as np
import pytest

import dp_cases
import refine_cases as rc
import refine_oracle
from famsa_b200.binding import REFINE_NO_GAP_OPT, REFINE_NO_TOTAL_SCORE, FamsaError
from oracle import pyoracle

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not pyoracle.have("ref_refine"), reason="oracle/_ref/libfamsa_ref_refine.so not built")]


@pytest.fixture(scope="module")
def eng():
    import famsa_b200
    e = famsa_b200.Engine(0)
    yield e
    e.close()


def check(eng, seqs, merges, n_refinements=100, flags=0, gaps=None):
    n = len(seqs)
    g, sm = rc.scoring(n)
    if gaps is not None:
        g = np.asarray(gaps, dtype=np.int64)
    ref = refine_oracle.RefRefine(sm, g, flags)
    want = ref.align_refine(seqs, merges, n_refinements)
    ref.close()
    # without a gap run of length 1 the reference's CalculateTotalScore reads memory it never zeroed (profile.cpp:1475-1480)
    runs = [ln for r in want["unrefined"] for ln, _ in refine_oracle.gap_runs(rc.to_codes(r))]
    assert not runs or 1 in runs, "the input alignment has gap runs but none of length 1"
    rows, width, total, stats, rid = rc.device_refine(eng, seqs, merges, g, sm, n_refinements, flags)
    got = [rows[i] for i in range(n)]
    if got != want["refined"] or total != want["total"]:
        t = want["trace"]
        acc = t[t[:, 4] == 1]
        first = f"the reference's first accepted try: {acc[0].tolist()}" if len(acc) else "the reference accepted no try"
        pytest.fail(f"n={n}: refined alignment differs (width {width} vs {want['width']}, total {total} vs {want['total']}, "
                    f"device counts {stats}, reference {want['counts']}; {first}; trace rows are "
                    f"[i_ref, column, split hash, identical, accepted, total])")
    assert width == want["width"]
    for k, v in want["counts"].items():
        assert stats[k] == v, f"{k}: {stats[k]} != {v}"
    # the resident tables of the refined profile are the reference's final CProfile's
    sc, cn, card = eng.prof_get(rid)
    assert card == n and sc.shape[0] == width + 1
    assert np.array_equal(cn, want["counters"]), "counters of the refined profile differ from the reference's"
    assert np.array_equal(sc, want["scores"]), "scores of the refined profile differ from the reference's"
    eng.prof_drop([rid])
    return stats


@pytest.mark.parametrize("n", [2, 3, 5, 99, 100, 101, 300, 1000])
def test_random_families(eng, n):
    seqs = rc.family(n, 60 if n < 1000 else 40, seed=n)
    stats = check(eng, seqs, dp_cases.random_tree(n, np.random.default_rng(n)))
    assert stats["n_realigned"] >= 1
    print(f"n={n}: {stats}, {stats['kernel_launches'] / max(stats['n_tries'], 1):.1f} launches per try")


def test_identical_rows_take_the_random_split(eng):
    seqs = rc.family(1, 50, seed=3) * 6
    stats = check(eng, seqs, dp_cases.random_tree(6, np.random.default_rng(1)))
    assert stats["n_identical"] > 0


@pytest.mark.parametrize("n_ref", [0, 1])
@pytest.mark.parametrize("n", [20, 300])
def test_refinement_counts(eng, n, n_ref):
    check(eng, rc.family(n, 50, seed=7), dp_cases.random_tree(n, np.random.default_rng(7)), n_refinements=n_ref)


@pytest.mark.parametrize("flags", [REFINE_NO_GAP_OPT, REFINE_NO_TOTAL_SCORE, REFINE_NO_GAP_OPT | REFINE_NO_TOTAL_SCORE])
def test_flags(eng, flags):
    stats = check(eng, rc.family(30, 70, seed=11), dp_cases.random_tree(30, np.random.default_rng(11)), flags=flags)
    if flags & REFINE_NO_TOTAL_SCORE:
        assert stats["n_accepted"] == stats["n_realigned"] - stats["n_identical"]


def test_non_default_gaps(eng):
    check(eng, rc.family(40, 80, seed=5), dp_cases.random_tree(40, np.random.default_rng(5)), gaps=[-700, -70, -350, -60])


def test_errors_leave_the_context_usable(eng):
    import famsa_b200
    seqs = rc.family(12, 40, seed=2)
    merges = dp_cases.random_tree(12, np.random.default_rng(2))
    g, sm = rc.scoring(12)
    fresh = famsa_b200.Engine(0)
    with pytest.raises(FamsaError):                               # no scoring matrix
        fresh.refine(0, np.zeros((2, 3), dtype=np.uint8), g)
    fresh.close()
    eng.upload(*rc.seqio.pack([rc.seqio.encode(s) for s in seqs]))
    eng.prof_set_scoring(sm)
    root, res, _ = eng.align_tree(merges, g)
    rows = dp_cases.assemble_rows(seqs, merges, res)
    arr = np.stack([rc.to_codes(rows[i]) for i in rc.id_order([f"s{i}" for i in range(12)])])
    for bad in (lambda: eng.refine(root + 1000, arr, g),                    # unknown root
                lambda: eng.refine(root, arr[:, :-1], g),                   # width differs
                lambda: eng.refine(root, arr[:-1], g),                      # n_rows != card
                lambda: eng.refine(root, arr, g, flags=4)):                 # unknown flag
        with pytest.raises(FamsaError):
            bad()
    eng.prof_drop([root])
    check(eng, seqs, merges)
