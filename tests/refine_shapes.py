"""Case generator for the refinement shape tests (tests/test_refine_shapes_host.py, tests/test_refine_shapes_gpu.py).

The kernels of famsa_b200/csrc/refine.cu loop in blocks of fixed size and keep one shared-memory histogram whose size
follows the width.  Realistic families never leave a few hundred columns; the cases here are hand-built alignments
(n x W codes, GAP = 30) at the boundaries the code is built around:

  * score_cases(): famsa_prof_refine with n_refinements = 0, i.e. the input's CalculateTotalScore alone, at widths around
    the per-column block (kRT), the single-block scans (kScanT), the default 48 KiB dynamic shared-memory limit of
    k_ref_score_runs (less its static shared memory), the opt-in and the largest width accepted; row counts around kRT
    and kScanT; gap runs longer than kRT and kScanT (several passes of the histogram's suffix scan), runs from column 1
    and to column W;
  * refine_cases(): the whole loop at widths and row counts past kScanT (multi-pass column, row and path scans), and
    two-group alignments whose every split is one partition with sides of 511 / 512 / 513 and 1023 / 1024 / 1025 rows
    (around k_ref_optimize's kOptT), each with row 0 in the more diverse and in the more uniform group, so the merge
    runs in both orientations; one two-row case inside the shared-memory window;
  * the edge cases: widths the call accepts and rejects, and a realignment that outgrows the limit inside the loop.

Every alignment has a residue in every row and in every column, and a gap run of length 1 wherever it has gaps (the
reference's CalculateTotalScore is undefined without one, see test_refine_host.test_missing_length1_run_is_defined_as_zero).
"""
from __future__ import annotations

import numpy as np

from famsa_b200 import profiles

# refine.cu constants the cases are built on (test_refine_shapes_host.py reads them from the source and compares)
K_RT = 256                         # threads of the per-column / per-row block loops
K_OPT_T = 512                      # threads of k_ref_optimize's block, one block per side
K_SCAN_T = 1024                    # threads of the single-block scans (k_ref_scan, k_ref_path_index)
K_MAX_HIST_BYTES = 200 << 10       # k_ref_score_runs' largest histogram
DEFAULT_DYN_SMEM = 48 << 10        # a kernel's dynamic shared-memory budget without the opt-in attribute ...
SCORE_RUNS_STATIC_SMEM = 32 * 4 + 32 * 8   # ... less its static shared memory: sh[32] int + shl[32] long long
MAX_WIDTH = K_MAX_HIST_BYTES // 4 - 1      # 51 199 columns
GAP = 30

# widths whose histogram needs more than the default budget but not the opt-in the code made before: 12 192 .. 12 287
WINDOW = ((DEFAULT_DYN_SMEM - SCORE_RUNS_STATIC_SMEM) // 4, DEFAULT_DYN_SMEM // 4 - 1)

SCORE_WIDTHS = [1, 2, 255, 256, 257, 1023, 1024, 1025, 2049, 12191, 12192, 12287, 12288, 12289, MAX_WIDTH]
SCORE_ROWS = [2, 255, 256, 257, 1023, 1024, 1025]
SIDE_ROWS = [511, 512, 513, 1023, 1024, 1025]


def hist_bytes(w: int) -> int:
    return (w + 1) * 4


# ------------------------------------------------------------------ alignments
def gap_runs(row: np.ndarray) -> list[tuple[int, int]]:
    """(first, last) column, 1-based, of every gap run of a row."""
    g = np.concatenate([[0], (row == GAP).astype(np.int8), [0]])
    d = np.diff(g)
    return list(zip((np.flatnonzero(d == 1) + 1).tolist(), np.flatnonzero(d == -1).tolist()))


def run_lengths(a: np.ndarray) -> list[int]:
    return [e - s + 1 for row in a for s, e in gap_runs(row)]


def well_formed(a: np.ndarray) -> bool:
    g = a == GAP
    lens = run_lengths(a)
    return bool((~g).any(axis=1).all() and (~g).any(axis=0).all() and (not lens or 1 in lens))


def consensus_rows(n: int, w: int, rng, sub: float = 0.25, cons=None) -> np.ndarray:
    cons = rng.integers(0, 20, size=w) if cons is None else cons
    return np.where(rng.random((n, w)) < sub, rng.integers(0, 20, size=(n, w)), cons[None, :]).astype(np.uint8)


def alignment(n: int, w: int, seed: int, gap_p: float = 0.08, runs=()) -> np.ndarray:
    """n x w codes around a consensus with random gaps (probability gap_p per cell, not on row 0 nor on the rows of
    `runs`) and the exact gap runs `runs` = [(row, first, last), 1-based columns]; then every column gets a residue
    in row 0 and, without a run of length 1 (w > 1), the last row gets one in its middle column."""
    rng = np.random.default_rng(seed)
    a = consensus_rows(n, w, rng)
    fixed = {r for r, _, _ in runs}
    if w > 1:
        free = np.array([r not in fixed and r > 0 for r in range(n)])
        a[(rng.random((n, w)) < gap_p) & free[:, None]] = GAP
    for r, s, e in runs:
        a[r, s - 1:e] = GAP
    for r in range(n):
        if (a[r] == GAP).all():
            a[r, rng.integers(0, w)] = rng.integers(0, 20)
    if w > 1 and 1 not in run_lengths(a):
        r = n - 1 if n - 1 not in fixed else 0
        a[r, :] = np.where(a[r] == GAP, rng.integers(0, 20, size=w), a[r]).astype(np.uint8)
        a[r, w // 2] = GAP
    for r, s, e in runs:                                         # the runs are exact: residues on both sides
        assert (a[r, s - 1:e] == GAP).all() and (s == 1 or a[r, s - 2] != GAP) and (e == w or a[r, e] != GAP)
    assert well_formed(a)
    return a


def score_cases() -> list[dict]:
    """dict(name, rows, claims) for famsa_prof_refine with n_refinements = 0."""
    out = []
    for w in SCORE_WIDTHS:
        for n in ((2, 5) if w > 4096 else (2, 5, 33)):
            out.append(dict(name=f"w{w}_n{n}", rows=alignment(n, w, seed=w * 7 + n), claims=dict(width=w, n=n)))
    for n in SCORE_ROWS:
        out.append(dict(name=f"n{n}_w300", rows=alignment(n, 300, seed=n), claims=dict(width=300, n=n)))
    long_runs = [("run257", 5, 600, [(1, 10, 266)], 257), ("run1025", 7, 2000, [(1, 100, 1124)], 1025),
                 ("run_from_col1", 3, 1500, [(1, 1, 1499)], 1499), ("run_to_colW", 3, 1500, [(1, 2, 1500)], 1499),
                 ("runs_both_ends", 40, 777, [(1, 1, 300), (2, 478, 777), (3, 1, 9), (4, 769, 777)], 300),
                 ("run257_wide", 4, 12250, [(1, 5000, 5256), (2, 1, 1025), (3, 11226, 12250)], 1025)]
    for name, n, w, runs, longest in long_runs:
        out.append(dict(name=name, rows=alignment(n, w, seed=len(out), runs=runs),
                        claims=dict(width=w, n=n, longest=longest, runs=runs)))
    return out


def two_group(big: int, small: int, row0_diverse: bool, seed: int, shared: int = 260, only_big: int = 24,
              only_small: int = 9) -> np.ndarray:
    """An alignment of two groups whose gap patterns are the same within each group: `shared` columns where both have
    residues, `only_big` (`only_small`) columns where only the first (second) group has them, in a shuffled order, so
    every partially gapped column splits the rows into exactly these two groups.  Row 0 is in the first group.  One group
    is diverse (many residues per column), the other near-uniform; row0_diverse picks which, and with it the orientation
    of the realignment.  Single columns of one group give the runs of length 1."""
    rng = np.random.default_rng(seed)
    w = shared + only_big + only_small
    kind = rng.permutation(np.repeat([0, 1, 2], [shared, only_big, only_small]))
    cons = rng.integers(0, 20, size=w)
    a = consensus_rows(big, w, rng, sub=0.6 if row0_diverse else 0.02, cons=cons)
    b = consensus_rows(small, w, rng, sub=0.02 if row0_diverse else 0.6, cons=cons)
    a[:, kind == 2] = GAP
    b[:, kind == 1] = GAP
    rows = np.vstack([a, b])
    assert well_formed(rows)
    return rows


def sides(rows: np.ndarray):
    """The two sides of the split every partially gapped column makes (RefineMostEmptyAndFullColumn): (profile1 =
    rows whose gap state equals row 0's, profile2), each condensed (all-gap columns removed)."""
    g = rows == GAP
    col = int(np.flatnonzero(g.any(axis=0) & ~g.all(axis=0))[0])
    d1 = g[:, col] == g[0, col]
    out = []
    for m in (d1, ~d1):
        s = rows[m]
        out.append(s[:, ~(s == GAP).all(axis=0)])
    return out


def refine_cases() -> list[dict]:
    """dict(name, rows, ids, n_refinements, claims) for the whole loop, compared with the reference's."""
    out = []
    for w in (1023, 1024, 1025, 2049):
        out.append(dict(name=f"w{w}_n128", rows=alignment(128, w, seed=w, gap_p=0.03), n_refinements=4,
                        claims=dict(width=w, n=128)))
    for n in (1023, 1024, 1025):
        out.append(dict(name=f"n{n}_w150", rows=alignment(n, 150, seed=n, gap_p=0.03), n_refinements=3,
                        claims=dict(width=150, n=n)))
    for s in SIDE_ROWS:
        other = 64 if s < 1000 else 40
        for diverse in (True, False):
            out.append(dict(name=f"sides{s}_{other}_{'diverse' if diverse else 'uniform'}",
                            rows=two_group(s, other, diverse, seed=s + diverse), n_refinements=100,
                            claims=dict(sides=(s, other), row0_diverse=diverse)))
    rng = np.random.default_rng(12250)
    two = consensus_rows(2, 12250, rng, sub=0.1)
    two[0, 4] = GAP
    two[1, 9000] = GAP
    out.append(dict(name="window_two_rows", rows=two, n_refinements=100, claims=dict(width=12250, n=2)))
    for c in out:
        c.setdefault("ids", [f"s{i:05d}" for i in range(c["rows"].shape[0])])
    n = 1025
    out.append(dict(name="ids_not_padded", rows=alignment(n, 130, seed=99, gap_p=0.03), n_refinements=3,
                    ids=[f"s{i}" for i in range(n)], claims=dict(width=130, n=n)))
    return out


# ------------------------------------------------------------------ edge cases
def too_wide() -> np.ndarray:
    """MAX_WIDTH + 1 columns: rejected before the loop."""
    return alignment(2, MAX_WIDTH + 1, seed=3)


def growing_realignment(length: int = 26000):
    """Two gap-free rows of `length` residues, a score matrix with every entry negative and gap costs 0: every diagonal
    step of the realignment loses to a pair of gaps, so the realignment is close to 2 x length > MAX_WIDTH columns wide
    (51 998 for 26 000 residues).
    Returns (rows, score matrix, gaps)."""
    rng = np.random.default_rng(26000)
    rows = rng.integers(0, 20, size=(2, length)).astype(np.uint8)
    sm = -rng.integers(1, 5000, size=(24, 24)).astype(np.int64)
    sm = (sm + sm.T) // 2
    return rows, sm, np.zeros(4, dtype=np.int64)


def tables(rows: np.ndarray, sm, gaps):
    """Profile tables of an alignment (profiles.tables_from_rows, gaps as -1)."""
    return profiles.tables_from_rows(np.where(rows == GAP, -1, rows).astype(np.int8), sm, gaps)
