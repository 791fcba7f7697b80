"""Host-side construction of profile tables from aligned rows -- the input format of HP-2.

Mirrors CProfile::CalculateCounters / CalculateScores (reference src/core/profile.cpp:101-217) for a block
of already aligned sequences: `counters` (width+1, 32) int32 and `scores` (width+1, 32) int64, column-major
as CProfileValues stores them (column c = 32 consecutive values; rows 0..23 residues, 25 GAP_OPEN, 26 GAP_EXT,
27 GAP_TERM_EXT, 28 GAP_TERM_OPEN; src/core/defs.h:62-74).  Used by bench.py to synthesise DP workloads and by
the tests as the host mirror of that reference routine; the merged-profile construction after a DP
(ConstructProfile) is not reproduced here -- it stays the reference's host code (see INTEGRATION.md).
"""
from __future__ import annotations

import numpy as np

GAP = -1                      # gap marker inside aligned rows (any negative code)
GO, GE, TE, TO = 25, 26, 27, 28
N_AA = 24


def tables_from_rows(rows: np.ndarray, score_matrix: np.ndarray, gaps) -> tuple[np.ndarray, np.ndarray, int]:
    """rows: (card, width) int8 residue codes 0..23 with negative = gap.  score_matrix: (24, 24) int64.
    gaps = (gap_open, gap_ext, gap_term_open, gap_term_ext).  Returns (scores, counters, card)."""
    rows = np.asarray(rows)
    card, width = rows.shape
    go, ge, to, te = (int(x) for x in gaps)
    cnt = np.zeros((width + 1, 32), dtype=np.int64)
    isgap = rows < 0
    for r in range(card):
        g = isgap[r]
        nz = np.flatnonzero(~g)
        if nz.size == 0:
            raise ValueError("all-gap row")
        first, last = nz[0], nz[-1]              # 0-based columns of the first / last residue
        # terminal gaps at the front: column 1 is TERM_OPEN, the rest TERM_EXT (profile.cpp:113-120)
        if first > 0:
            cnt[1, TO] += 1
            cnt[2:first + 1, TE] += 1
        # terminal gaps at the back: first gap column TERM_OPEN, the rest TERM_EXT (profile.cpp:122-129)
        if last < width - 1:
            cnt[last + 2, TO] += 1
            cnt[last + 3:width + 1, TE] += 1
        # residues
        np.add.at(cnt, (nz + 1, rows[r, nz].astype(np.int64)), 1)
        # internal gap runs: first column OPEN, following columns EXT (profile.cpp:140-153)
        inner = g.copy()
        inner[:first] = False
        inner[last + 1:] = False
        if inner.any():
            start = inner & ~np.concatenate([[False], inner[:-1]])
            cnt[np.flatnonzero(start) + 1, GO] += 1
            cnt[np.flatnonzero(inner & ~start) + 1, GE] += 1
    scores = np.zeros((width + 1, 32), dtype=np.int64)
    # column 0: card x gap costs (profile.cpp:170-173)
    scores[0, GO] = card * go; scores[0, GE] = card * ge; scores[0, TE] = card * te; scores[0, TO] = card * to
    sm = np.asarray(score_matrix, dtype=np.int64)
    c = cnt[1:]
    gap_cost = c[:, GO] * go + c[:, TO] * to + c[:, GE] * ge + c[:, TE] * te          # profile.cpp:183-194
    scores[1:, :N_AA] = c[:, :N_AA] @ sm + gap_cost[:, None]                            # profile.cpp:196-209
    tot = c[:, :N_AA].sum(axis=1)
    scores[1:, GO] += tot * go; scores[1:, TO] += tot * to; scores[1:, GE] += tot * ge; scores[1:, TE] += tot * te
    return scores, cnt.astype(np.int32), card


def rows_after_merge(rows1: list[str], rows2: list[str], path, swapped: bool, from_text: bool = False) -> tuple[list[int], list[str]]:
    """The rows of the profile a merge of two alignments builds: ConstructProfile ends with data = profile2->data;
    append(profile1->data) (profile.cpp:992-993), profile2 being the DP's column profile, so the column side's rows come
    first, each side in its input order.  swapped: famsa_dp_result.swapped (the DP's rows are rows2).  A merged row is its
    input row with the path's gap columns inserted: H (1) inserts a gap column into the row side, V (2) into the column
    side (FinalizeGaps, profile.cpp:1053-1104).  Letters are kept as given, so lower case and non-standard letters
    survive as CGappedSequence::uppercase / extra_symbols make them survive.
    from_text: the profiles were built from rows read as text (famsa_prof_put_rows' FAMSA_PUT_ROWS_FROM_TEXT, what
    famsa in1 in2 out does): the path covers all but the last column of each side, and that column ends every merged row.
    Returns (order, rows): output row k is input row order[k] of rows1 + rows2."""
    if from_text:
        order, rows = rows_after_merge([r[:-1] for r in rows1], [r[:-1] for r in rows2], path, swapped)
        return order, [r + (rows1[k] if k < len(rows1) else rows2[k - len(rows1)])[-1] for k, r in zip(order, rows)]
    p = np.asarray(path, dtype=np.uint8)
    n1 = len(rows1)
    row_side, col_side = (1, 0) if swapped else (0, 1)

    def insert(rows: list[str], skip: int) -> list[str]:
        if not rows:
            return []
        a = np.frombuffer("".join(rows).encode("latin-1"), dtype=np.uint8).reshape(len(rows), -1)
        take = p != skip
        if int(take.sum()) != a.shape[1]:
            raise ValueError(f"the path consumes {int(take.sum())} columns of a side {a.shape[1]} wide")
        out = np.full((a.shape[0], len(p)), ord("-"), dtype=np.uint8)
        out[:, take] = a
        return [r.tobytes().decode("latin-1") for r in out]

    sides = (rows1, rows2)
    merged = {row_side: insert(sides[row_side], 1), col_side: insert(sides[col_side], 2)}
    base = (0, n1)
    order = [base[col_side] + i for i in range(len(sides[col_side]))] + [base[row_side] + i for i in range(len(sides[row_side]))]
    return order, merged[col_side] + merged[row_side]


def synth_alignment(card: int, width: int, rng, gap_frac: float = 0.12) -> np.ndarray:
    """A plausible aligned block: a consensus with per-row substitutions and random gap runs; every column
    keeps at least one residue (as any real profile does)."""
    cons = rng.integers(0, 20, size=width)
    rows = np.where(rng.random((card, width)) < 0.35, rng.integers(0, 20, size=(card, width)), cons[None, :]).astype(np.int8)
    n_runs = max(1, int(gap_frac * width / 4))
    for r in range(card):
        for _ in range(n_runs):
            a = int(rng.integers(0, width)); ln = int(rng.integers(1, 9))
            rows[r, a:a + ln] = GAP
        if (rows[r] < 0).all():
            rows[r, width // 2] = cons[width // 2]
    empty = (rows < 0).all(axis=0)
    rows[0, empty] = cons[empty]
    return rows


def synth_score_matrix(rng) -> np.ndarray:
    """Random symmetric integer substitution matrix with PFASUM-like magnitudes (x1000 fixed point)."""
    m = rng.integers(-4000, 3000, size=(24, 24))
    m = (m + m.T) // 2
    m[np.arange(24), np.arange(24)] = rng.integers(3000, 11000, size=24)
    return m.astype(np.int64)
