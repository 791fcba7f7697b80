"""CPU checks of famsa_prof_refine's checkers: the numpy restatements of CalculateTotalScore and OptimizeGaps
(tests/refine_oracle.py) against the reference's own functions on random gapped alignments, the formulation of the
gap-open count against brute force, the reference defect of a missing length-1 run, and the restated RefineAlignment loop
of oracle/ref_refine_harness.cpp (its per-try trace agrees with its counts, and its two entry points run one loop);
the vectorised total_score_rows against both totals."""
from __future__ import annotations

import numpy as np
import pytest

import dp_cases
import refine_cases as rc
import refine_oracle as ro
from famsa_b200 import profiles
from oracle import pyoracle

need_ref = pytest.mark.skipif(not pyoracle.have("ref_refine"), reason="oracle/_ref/libfamsa_ref_refine.so not built")
GAP = ro.GAP


def alignment(kind: str, seed: int) -> np.ndarray:
    """n x W codes with GAP = 30, every row with a residue and (except kind 'no_len1') a gap run of length 1."""
    rng = np.random.default_rng(seed)
    n, W = int(rng.integers(2, 12)), int(rng.integers(4, 40))
    if kind == "one_column":
        return rng.integers(0, 24, size=(n, 1)).astype(np.uint8)
    a = rng.integers(0, 24, size=(n, W)).astype(np.uint8)
    if kind == "random":
        a[rng.random((n, W)) < 0.35] = GAP
    elif kind == "terminal":
        for r in range(n):
            lo, hi = sorted(rng.integers(0, W, size=2))
            a[r, :lo] = GAP; a[r, hi + 1:] = GAP
    elif kind == "single_residue":
        a[:] = GAP
        for r in range(n):
            a[r, rng.integers(0, W)] = rng.integers(0, 24)
    elif kind in ("wide", "no_len1"):
        for r in range(n):
            for _ in range(2):
                s = int(rng.integers(0, W)); a[r, s:s + int(rng.integers(2, 12))] = GAP
    for r in range(n):
        if np.all(a[r] == GAP):
            a[r, rng.integers(0, W)] = 0
    if kind == "no_len1":                                    # widen every run of length 1
        for r in range(n):
            for ln, st in ro.gap_runs(a[r]):
                if ln == 1:
                    nb = st if st < W and a[r, st] != GAP and np.sum(a[r] != GAP) > 1 else st - 2
                    if 0 <= nb < W and np.sum(a[r] != GAP) > 1:
                        a[r, nb] = GAP
    elif not any(ln == 1 for row in a for ln, _ in ro.gap_runs(row)):
        extra = rng.integers(0, 24, size=(1, W)).astype(np.uint8)   # the reference reads gap_matrix[1] unzeroed without one
        extra[0, 1] = GAP
        a = np.vstack([a, extra])
    return a


def has_len1(a) -> bool:
    return any(ln == 1 for row in a for ln, _ in ro.gap_runs(row))


def counters(a, sm, g):
    return profiles.tables_from_rows(np.where(a == GAP, -1, a).astype(np.int8), sm, g)[1]


KINDS = ["random", "terminal", "one_column", "single_residue", "wide"]


@need_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(6))
def test_total_score_restatement_equals_reference(kind, seed):
    a = alignment(kind, seed)
    if a.shape[1] > 1 and np.any(a == GAP):
        assert has_len1(a), "the reference's value is only defined with a gap run of length 1"
    g, sm = rc.scoring(a.shape[0])
    ref = ro.RefRefine(sm, g)
    want = ref.total_score([rc.to_letters(r) for r in a])
    ref.close()
    assert ro.total_score(a, counters(a, sm, g), sm, g) == want


@pytest.mark.parametrize("kind", KINDS + ["no_len1"])
@pytest.mark.parametrize("seed", range(6))
def test_total_score_rows_equals_restatement_and_reference(kind, seed):
    """The vectorised count (a run opens against every row with a residue inside it) is the same total."""
    a = alignment(kind, seed)
    g, sm = rc.scoring(a.shape[0])
    cn = counters(a, sm, g)
    got = ro.total_score_rows(a, cn, sm, g)
    assert got == ro.total_score(a, cn, sm, g)
    if pyoracle.have("ref_refine") and kind != "no_len1":
        ref = ro.RefRefine(sm, g)
        assert got == ref.total_score([rc.to_letters(r) for r in a])
        ref.close()


def long_run_alignments():
    """Runs longer than 256 columns (one block of k_ref_score_runs' suffix scan), terminal runs at column 1 and W."""
    import refine_shapes as S
    yield S.alignment(4, 600, seed=1, runs=[(1, 10, 266), (2, 1, 300)])
    yield S.alignment(3, 400, seed=2, runs=[(1, 1, 399)])
    yield S.alignment(3, 400, seed=3, runs=[(1, 2, 400)])
    yield S.alignment(6, 900, seed=4, runs=[(1, 1, 1), (2, 900, 900), (3, 300, 899), (4, 2, 258)])


@need_ref
@pytest.mark.parametrize("case", range(4))
def test_total_score_rows_equals_reference_on_long_runs(case):
    a = list(long_run_alignments())[case]
    assert max(ln for row in a for ln, _ in ro.gap_runs(row)) > 256 and has_len1(a)
    g, sm = rc.scoring(a.shape[0])
    ref = ro.RefRefine(sm, g)
    want = ref.total_score([rc.to_letters(r) for r in a])
    ref.close()
    cn = counters(a, sm, g)
    assert ro.total_score_rows(a, cn, sm, g) == ro.total_score(a, cn, sm, g) == want


@need_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(6))
def test_optimize_gaps_restatement_equals_reference(kind, seed):
    a = alignment(kind, seed)
    g, sm = rc.scoring(a.shape[0])
    ref = ro.RefRefine(sm, g)
    want = ref.optimize_gaps([rc.to_letters(r) for r in a])
    ref.close()
    assert [rc.to_letters(r) for r in ro.optimize_gaps(a)] == want


@pytest.mark.parametrize("kind", KINDS + ["no_len1"])
@pytest.mark.parametrize("seed", range(6))
def test_gap_open_count_formulations_agree(kind, seed):
    """The inclusion-exclusion table (reference) and the containing-run count (the device's histogram) are one sum."""
    a = alignment(kind, seed)
    assert ro.containing_runs_table(a) == ro.containing_runs_brute(a)


def test_missing_length1_run_is_defined_as_zero():
    """Gap runs of length 2 and more but none of length 1: the reference's gap_ranges[2] then reads gap_matrix[1], a row
    it never zeroed (profile.cpp:1439-1442, 1475-1480), so its total depends on heap contents.  The restatement and the
    device define that row as zero, which is what the containing-run count gives."""
    a = np.array([[0, GAP, GAP, 1, 2, 3],
                  [0, 1, 2, GAP, GAP, 3],
                  [0, 1, 2, 3, 4, 5]], dtype=np.uint8)
    assert not has_len1(a) and np.any(a == GAP)
    assert ro.containing_runs_table(a) == ro.containing_runs_brute(a) == 2
    g, sm = rc.scoring(3)
    assert isinstance(ro.total_score(a, counters(a, sm, g), sm, g), int)


@need_ref
@pytest.mark.parametrize("n,flags", [(3, 0), (40, 0), (40, 1), (40, 2)])
def test_trace_matches_counts(n, flags):
    g, sm = rc.scoring(n)
    ref = ro.RefRefine(sm, g, flags)
    r = ref.align_refine(rc.family(n, 60, seed=n), dp_cases.random_tree(n, np.random.default_rng(n)))
    ref.close()
    t, c = r["trace"], r["counts"]
    assert len(t) == c["n_tries"]
    assert (t[:, 3] >= 0).sum() == c["n_realigned"]
    assert (t[:, 3] == 1).sum() == c["n_identical"]
    assert t[:, 4].sum() == c["n_accepted"]
    if flags & 2:
        assert r["total"] == 0 and c["n_accepted"] == c["n_realigned"] - c["n_identical"]
    else:
        assert r["total"] >= r["prev_total"]
        acc = t[t[:, 4] == 1]
        assert (len(acc) == 0 and r["total"] == r["prev_total"]) or acc[-1, 5] == r["total"]
    assert c["n_realigned"] == 100 or c["n_tries"] == 2000


@pytest.mark.skipif(not pyoracle.have("ref_refine", "rr_refine_rows"),
                    reason="oracle/_ref/libfamsa_ref_refine.so not built, or built without rr_refine_rows")
def test_refine_rows_is_the_loop_of_align_refine():
    """rr_refine_rows on the unrefined rows of rr_align_refine gives the same refinement, try for try."""
    n = 30
    g, sm = rc.scoring(n)
    ref = ro.RefRefine(sm, g)
    ids = [f"s{i}" for i in range(n)]
    a = ref.align_refine(rc.family(n, 60, seed=4), dp_cases.random_tree(n, np.random.default_rng(4)), ids=ids)
    b = ref.refine_rows(a["unrefined"], ids)
    ref.close()
    assert b["refined"] == a["refined"] and b["counts"] == a["counts"] and (b["prev_total"], b["total"]) == (a["prev_total"], a["total"])
    assert np.array_equal(b["trace"], a["trace"]) and np.array_equal(b["scores"], a["scores"])
    assert np.array_equal(b["counters"], a["counters"])
