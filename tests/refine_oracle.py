"""Checkers of famsa_prof_refine.

* numpy restatements of CProfile::CalculateTotalScore (profile.cpp:1368-1542, with its inclusion-exclusion table
  gap_ranges) and CProfile::OptimizeGaps (profile.cpp:436-689, with CGappedSequence::InsertGap / RemoveGap as string
  edits): the independent check of the device's k_ref_score_* and k_ref_optimize, which use other formulations;
* the reference behind oracle/ref_refine_harness.cpp (oracle/_ref/libfamsa_ref_refine.so, opened by oracle/pyoracle.py):
  its own CalculateTotalScore and OptimizeGaps on given rows, and its progressive alignment followed by the restated
  RefineAlignment loop, with the per-try trace and the final profile's tables; and its RefineAlignment loop on a given
  alignment;
* total_score_rows: CalculateTotalScore vectorised, with a third formulation of the gap-open count, for widths the
  reference's (width+1)^2 / 2 tables and the restatement above cannot reach."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle


def _strs(xs):
    return (C.c_char_p * len(xs))(*[x.encode("ascii") for x in xs])


class RefRefine:
    """A CParams with the given 24 x 24 scores, gaps {open, ext, term_open, term_ext} and famsa_prof_refine flags;
    no_threads is what RefineAlignment passes to Align (> 1: the unbanded paths)."""

    def __init__(self, score_matrix, gaps, flags: int = 0, no_threads: int = 2):
        self.lib = pyoracle.lib("ref_refine")
        self.sm = np.ascontiguousarray(score_matrix, dtype=np.int64)
        self.g = np.ascontiguousarray(gaps, dtype=np.int64)
        self.h = C.c_void_p(self.lib.rr_create(self.sm.ctypes.data, self.g.ctypes.data, flags, no_threads))

    def close(self):
        if self.h:
            self.lib.rr_destroy(self.h)
            self.h = None

    def total_score(self, rows: list[str]) -> int:
        return int(self.lib.rr_total_score(self.h, _strs(rows), len(rows)))

    def optimize_gaps(self, rows: list[str]) -> list[str]:
        w = len(rows[0])
        buf = C.create_string_buffer(len(rows) * (w + 1))
        self.lib.rr_optimize_gaps(self.h, _strs(rows), len(rows), buf)
        return [buf.raw[i * (w + 1):(i + 1) * (w + 1)].split(b"\0")[0].decode() for i in range(len(rows))]

    def align_refine(self, seqs: list[str], merges, n_refinements: int = 100, ids: list[str] | None = None) -> dict:
        n = len(seqs)
        ids = ids or [f"s{i}" for i in range(n)]
        m = np.ascontiguousarray(merges, dtype=np.int32).reshape(-1, 2)
        stride = sum(len(s) for s in seqs) + 1
        unref = C.create_string_buffer(n * stride)
        ref = C.create_string_buffer(n * stride)
        widths = np.zeros(2, dtype=np.uint32)
        totals = np.zeros(2, dtype=np.int64)
        counts = np.zeros(4, dtype=np.uint32)
        max_trace = 20 * max(100, min(n_refinements, 2 * n))
        trace = np.zeros((max_trace, 6), dtype=np.int64)
        scores = np.zeros((stride + 1, 32), dtype=np.int64)
        counters = np.zeros((stride + 1, 32), dtype=np.int32)
        self.lib.rr_align_refine(self.h, _strs(seqs), _strs(ids), n, m.ctypes.data, n_refinements, unref, ref, stride,
                                 widths.ctypes.data, totals.ctypes.data, counts.ctypes.data, trace.ctypes.data, max_trace,
                                 scores.ctypes.data, counters.ctypes.data)

        return _result(n, stride, unref, ref, widths, totals, counts, trace, scores, counters)

    def refine_rows(self, rows: list[str], ids: list[str], n_refinements: int = 100) -> dict:
        """RefineAlignment of a given alignment (rows of letters, '-' for a gap; row i is sequence i with FASTA id ids[i]).
        Returns align_refine's dict, with 'unrefined' the rows given.  The refined width must stay below 2 W + 2 (room
        the rows are given); a refinement that grows wider raises."""
        n, w = len(rows), len(rows[0])
        stride = 2 * w + 2
        ref = C.create_string_buffer(n * stride)
        widths = np.zeros(2, dtype=np.uint32)
        totals = np.zeros(2, dtype=np.int64)
        counts = np.zeros(4, dtype=np.uint32)
        max_trace = 20 * max(100, min(n_refinements, 2 * n))
        trace = np.zeros((max_trace, 6), dtype=np.int64)
        scores = np.zeros((stride + 1, 32), dtype=np.int64)
        counters = np.zeros((stride + 1, 32), dtype=np.int32)
        self.lib.rr_refine_rows(self.h, _strs(rows), _strs(ids), n, n_refinements, ref, stride, widths.ctypes.data,
                                totals.ctypes.data, counts.ctypes.data, trace.ctypes.data, max_trace, scores.ctypes.data,
                                counters.ctypes.data)
        if widths[1] >= stride:
            raise RuntimeError(f"refined width {int(widths[1])} leaves no room in rows of {stride} bytes")
        out = _result(n, stride, None, ref, widths, totals, counts, trace, scores, counters)
        out["unrefined"] = list(rows)
        return out


def _result(n, stride, unref, ref, widths, totals, counts, trace, scores, counters) -> dict:
    def rows(buf, w):
        return [buf.raw[i * stride:i * stride + w].decode() for i in range(n)]
    return dict(unrefined=rows(unref, int(widths[0])) if unref is not None else None, refined=rows(ref, int(widths[1])),
                width=int(widths[1]), prev_total=int(totals[0]), total=int(totals[1]),
                counts=dict(n_tries=int(counts[0]), n_realigned=int(counts[1]), n_accepted=int(counts[2]),
                            n_identical=int(counts[3])),
                trace=trace[:int(counts[0])], scores=scores[:int(widths[1]) + 1], counters=counters[:int(widths[1]) + 1])


# ------------------------------------------------------------------------------------------------ numpy restatements
GAP = 30
GO, GE, TE, TO = 25, 26, 27, 28           # defs.h:62-74


def gap_runs(row: np.ndarray) -> list[tuple[int, int]]:
    """(length, first column, 1-based) of every gap run of one row (CGappedSequence::n_gaps)."""
    runs, c, w = [], 0, len(row)
    while c < w:
        if row[c] == GAP:
            e = c
            while e + 1 < w and row[e + 1] == GAP:
                e += 1
            runs.append((e - c + 1, c + 1))
            c = e + 1
        else:
            c += 1
    return runs


def total_score(rows: np.ndarray, counters: np.ndarray, sm: np.ndarray, gaps) -> int:
    """CalculateTotalScore (profile.cpp:1368-1542) of an alignment (n x W codes, GAP = 30) with counters (W+1) x 32.
    gap_ranges[L][s] = gap runs of all rows inside [s, s+L-1], built by the reference's recurrence; the row
    gap_matrix[1] that the reference reads unzeroed when no run has length 1 (:1475-1480) is zero here."""
    go, ge, to, te = (int(x) for x in gaps)
    n, W = rows.shape
    score = 0
    n_ext = n_text = 0
    for i in range(1, W + 1):
        col = [int(x) for x in counters[i]]
        for c1 in range(24):
            if col[c1]:
                for c2 in range(c1 + 1, 24):
                    if col[c2]:
                        score += int(sm[c1][c2]) * col[c1] * col[c2]
                score += int(sm[c1][c1]) * col[c1] * (col[c1] - 1) // 2
        ng, nt = col[GO] + col[GE], col[TO] + col[TE]
        ns = n - ng - nt
        n_ext += ns * ng
        n_text += ns * nt
    gm = np.zeros((W + 2, W + 2), dtype=np.int64)           # gap_matrix[len][start]
    positions = []
    for row in rows:
        for ln, st in gap_runs(row):
            if gm[ln][st] == 0:
                positions.append((ln, st))
            gm[ln][st] += 1
    gr = np.zeros((W + 2, W + 2), dtype=np.int64)           # gap_ranges[len][start]
    for i in range(1, W + 1):
        gr[1][i] = gm[1][i]
    for i in range(1, W):
        gr[2][i] = gm[1][i] + gm[1][i + 1] + gm[2][i]
    for ln in range(3, W + 1):
        for i in range(1, W - ln + 2):
            gr[ln][i] = gr[ln - 1][i] + gr[ln - 1][i + 1] - gr[ln - 2][i + 1] + gm[ln][i]
    n_open = n_topen = 0
    for ln, i in positions:
        inside = int(gr[W][1])
        if ln > 2:
            inside += int(gr[ln - 2][i + 1])
        if i + ln - 2 > 0:
            inside -= int(gr[i + ln - 2][1])
        if i + 1 <= W:
            inside -= int(gr[W - i][i + 1])
        cur = int(gm[ln][i])
        inside -= cur
        if i == 1 or i + ln - 1 == W:
            n_topen += (n - cur - inside) * cur
        else:
            n_open += (n - cur - inside) * cur
    n_ext -= n_open
    n_text -= n_topen
    return score + n_ext * ge + n_open * go + n_text * te + n_topen * to


def run_bounds(rows: np.ndarray):
    """(row, first column, last column) of every gap run of an n x W alignment, 1-based columns, as three int64 arrays."""
    g = np.zeros((rows.shape[0], rows.shape[1] + 2), dtype=np.int8)
    g[:, 1:-1] = rows == GAP
    d = np.diff(g, axis=1)
    r0, s = np.nonzero(d == 1)                                # a run starts in column s + 1 (1-based)
    r1, e = np.nonzero(d == -1)                               # ... and ends in column e
    assert np.array_equal(r0, r1)
    return r0.astype(np.int64), s.astype(np.int64) + 1, e.astype(np.int64)


def total_score_rows(rows: np.ndarray, counters: np.ndarray, sm: np.ndarray, gaps, chunk: int = 1 << 12) -> int:
    """CalculateTotalScore (profile.cpp:1368-1542) of an n x W alignment with counters (W+1) x 32, vectorised and in
    O(W + runs x n) for any width.  Column terms from the counters in exact int64: symbol pairs (upper triangle of sm,
    and the diagonal x C(n_k, 2)), residue x internal-gap and residue x terminal-gap pairs.  Gap opens by a third
    formulation: a run [s, e] of one row opens against every row that has a residue somewhere in [s, e] (the rows
    without one are exactly those whose run through s contains [s, e]); per-row prefix sums of residues answer that.
    The run is terminal when s == 1 or e == W."""
    go, ge, to, te = (int(x) for x in gaps)
    rows = np.asarray(rows)
    n, W = rows.shape
    cnt = np.asarray(counters, dtype=np.int64)[1:W + 1]
    s64 = np.asarray(sm, dtype=np.int64)[:24, :24]
    k = cnt[:, :24]
    pair = int(((k @ np.triu(s64, 1)) * k).sum()) + int(((k * (k - 1) // 2) @ np.diag(s64)).sum())
    ng, nt = cnt[:, GO] + cnt[:, GE], cnt[:, TO] + cnt[:, TE]
    ns = n - ng - nt
    n_ext, n_text = int((ns * ng).sum()), int((ns * nt).sum())
    pre = np.zeros((n, W + 1), dtype=np.int32)                # pre[r, c]: residues of row r in columns 1..c
    np.cumsum(rows != GAP, axis=1, out=pre[:, 1:])
    _, s, e = run_bounds(rows)
    n_open = n_topen = 0
    for lo in range(0, len(s), chunk):
        ss, ee = s[lo:lo + chunk], e[lo:lo + chunk]
        v = (pre[:, ee] > pre[:, ss - 1]).sum(axis=0).astype(np.int64)
        term = (ss == 1) | (ee == W)
        n_topen += int(v[term].sum())
        n_open += int(v[~term].sum())
    n_ext -= n_open
    n_text -= n_topen
    return pair + n_ext * ge + n_open * go + n_text * te + n_topen * to


def containing_runs_brute(rows: np.ndarray) -> int:
    """sum over the gap runs [s, e] of all rows of the runs [s', e'] with s' <= s and e' >= e: what the inclusion-exclusion
    table of total_score and the histogram of the device both count, by brute force."""
    runs = [(st, st + ln - 1) for row in rows for ln, st in gap_runs(row)]
    return sum(sum(1 for s2, e2 in runs if s2 <= s and e2 >= e) for s, e in runs)


def containing_runs_table(rows: np.ndarray) -> int:
    """the same sum from total_score's gap_ranges recurrence"""
    n, W = rows.shape
    gm = np.zeros((W + 2, W + 2), dtype=np.int64)
    for row in rows:
        for ln, st in gap_runs(row):
            gm[ln][st] += 1
    gr = np.zeros((W + 2, W + 2), dtype=np.int64)
    gr[1, 1:W + 1] = gm[1, 1:W + 1]
    for i in range(1, W):
        gr[2][i] = gm[1][i] + gm[1][i + 1] + gm[2][i]
    for ln in range(3, W + 1):
        for i in range(1, W - ln + 2):
            gr[ln][i] = gr[ln - 1][i] + gr[ln - 1][i + 1] - gr[ln - 2][i + 1] + gm[ln][i]
    tot = 0
    for ln in range(1, W + 1):
        for i in range(1, W - ln + 2):
            if gm[ln][i]:
                c = int(gr[W][1]) + (int(gr[ln - 2][i + 1]) if ln > 2 else 0)
                c -= int(gr[i + ln - 2][1]) if i + ln - 2 > 0 else 0
                c -= int(gr[W - i][i + 1]) if i + 1 <= W else 0
                tot += int(gm[ln][i]) * c
    return tot


def optimize_gaps(rows: np.ndarray) -> np.ndarray:
    """OptimizeGaps (profile.cpp:436-689) on n x W codes: exchanges decided on the gap pattern decoded once (:453-481),
    applied with InsertGap(pos) / RemoveGap(pos) as edits of the 1-based gapped row."""
    n, W = rows.shape
    g = np.ones((W + 1, n), dtype=bool)                     # trans_gap_sequences (column 0: gap)
    g[1:, :] = (rows == GAP).T
    bound = np.ones(W + 1, dtype=bool)                      # gap_sym_broundaries
    for c in range(1, W):
        bound[c] = not np.any(~g[c] & ~g[c + 1])
    bound[W] = not np.any(~g[W])
    out = [list(r) for r in rows]
    maxp = W
    for curr in [c for c in range(1, W) if bound[c]][::-1]:
        if curr + 2 > maxp:
            continue
        rng = [[0, 0] for _ in range(n)]
        typ = []
        for j in range(n):
            if g[curr][j] and g[curr + 1][j]:
                typ.append("both"); rng[j] = [1, 1]
            elif g[curr][j]:
                typ.append("left"); rng[j][0] = 1
            elif g[curr + 1][j]:
                typ.append("right"); rng[j][1] = 1
        L = 2
        while curr + 1 - L > 0:
            col = g[curr + 1 - L]
            stop = False
            for j in range(n):
                if typ[j] == "left":
                    if col[j]: rng[j][0] = L
                    else: stop = True
                elif typ[j] == "both":
                    if col[j]: rng[j][0] = L
                    else: typ[j] = "both_ne"
            if stop:
                break
            L += 1
        typ = ["both" if t == "both_ne" else t for t in typ]
        R = 2
        while curr + R < maxp:
            col = g[curr + R]
            stop = False
            for j in range(n):
                if typ[j] == "right":
                    if col[j]: rng[j][1] = R
                    else: stop = True
                elif typ[j] == "both":
                    if col[j]: rng[j][1] = R
                    else: typ[j] = "both_ne"
            if stop:
                break
            R += 1
        typ = ["both" if t == "both_ne" else t for t in typ]
        ok = True
        for j in range(n):
            if typ[j] == "both":
                a, b = rng[j][0] >= L - 1, rng[j][1] >= R - 1
                if not a and not b:
                    ok = False
                elif a and b:
                    pass
                elif a:
                    typ[j] = "to_left"
                else:
                    typ[j] = "to_right"
        if not ok or curr - L <= 0 or curr + R >= W:
            continue
        lc, rc = curr - (L - 1), curr + R
        bal = 0
        for j in range(n):
            if typ[j] == "left":
                bal += (not g[rc][j]) - (not g[lc][j])
            elif typ[j] == "right":
                bal += (not g[lc][j]) - (not g[rc][j])
            elif typ[j] == "to_left":
                bal += not g[rc][j]
            elif typ[j] == "to_right":
                bal += not g[lc][j]
        if bal >= 0:
            continue
        for j in range(n):
            r = out[j]
            if typ[j] in ("left", "to_left"):
                for _ in range(L - 1):
                    r.insert(rc - 1, GAP)                  # InsertGap(right_col)
                for _ in range(L - 1):
                    assert r[lc] == GAP
                    del r[lc]                               # RemoveGap(left_col + 1)
            elif typ[j] in ("right", "to_right"):
                for _ in range(R - 1):
                    assert r[curr] == GAP
                    del r[curr]                             # RemoveGap(curr + 1)
                for _ in range(R - 1):
                    r.insert(lc, GAP)                       # InsertGap(left_col + 1)
        maxp = lc
    return np.array(out, dtype=np.uint8)
