"""CPU tests of tests/refine_shapes.py: the generator is built on refine.cu's constants, every case has the property it
is named for (width, rows, longest run, a run of length 1, the side of each shared-memory limit its histogram is on, the
side sizes and orientation of the first split), and the vectorised total score the GPU tests rely on equals the
reference's CalculateTotalScore and the numpy restatement of its table."""
import os
import re

import numpy as np
import pytest

import dp_shapes
import refine_cases as rc
import refine_oracle as ro
import refine_shapes as S
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "famsa_b200", "csrc", "refine.cu")).read()
need_ref = pytest.mark.skipif(not pyoracle.have("ref_refine"), reason="oracle/_ref/libfamsa_ref_refine.so not built")


def test_constants_match_refine_cu():
    for name, value in (("kRT", S.K_RT), ("kScanT", S.K_SCAN_T), ("kOptT", S.K_OPT_T)):
        m = re.search(rf"constexpr int {name} = (\d+);", SRC)
        assert m and int(m.group(1)) == value, name
    m = re.search(r"constexpr size_t kMaxHistBytes = (\d+)u << (\d+);", SRC)
    assert m and int(m.group(1)) << int(m.group(2)) == S.K_MAX_HIST_BYTES
    assert S.MAX_WIDTH == 51199 and "wider than 51 199 columns" in SRC
    # k_ref_score_runs' static shared memory, which the default dynamic budget is shared with
    body = re.search(r"k_ref_score_runs\(.*?\n\{(.*?)\n\}", SRC, re.S).group(1)
    assert re.findall(r"__shared__ (int|long long) (\w+)\[32\];", body) == [("int", "sh"), ("long long", "shl")]
    assert S.SCORE_RUNS_STATIC_SMEM == 384
    assert S.WINDOW == (12192, 12287)
    assert S.hist_bytes(S.WINDOW[0] - 1) == S.DEFAULT_DYN_SMEM - S.SCORE_RUNS_STATIC_SMEM
    assert S.hist_bytes(S.WINDOW[1]) == S.DEFAULT_DYN_SMEM
    # the transposes' 32 x 32 tiles
    assert "__shared__ uint8_t t[32][33];" in SRC


def runs_of(a):
    return [(r, s, e) for r, row in enumerate(a) for s, e in S.gap_runs(row)]


def test_score_cases_reach_every_boundary():
    cases = S.score_cases()
    assert len({c["name"] for c in cases}) == len(cases)
    widths, rows, longest = set(), set(), 0
    for c in cases:
        a, cl = c["rows"], c["claims"]
        assert a.dtype == np.uint8 and a.shape == (cl["n"], cl["width"]), c["name"]
        assert S.well_formed(a), c["name"]
        lens = S.run_lengths(a)
        if a.shape[1] > 1:
            assert 1 in lens, c["name"]
        for r, s, e in cl.get("runs", []):
            assert (r, s, e) in runs_of(a), c["name"]
        if "longest" in cl:
            assert max(lens) == cl["longest"], c["name"]
        widths.add(a.shape[1]); rows.add(a.shape[0]); longest = max(longest, max(lens, default=0))
    assert widths >= set(S.SCORE_WIDTHS) and rows >= set(S.SCORE_ROWS)
    # the histogram on each side of each limit: default budget, 48 KiB, the largest histogram
    hb = {w: S.hist_bytes(w) for w in widths}
    limit = S.DEFAULT_DYN_SMEM - S.SCORE_RUNS_STATIC_SMEM
    assert any(b == limit for b in hb.values())                                           # 12 191: fits by default
    assert any(limit < b <= S.DEFAULT_DYN_SMEM for b in hb.values())                      # the window
    assert {w for w in widths if S.WINDOW[0] <= w <= S.WINDOW[1]} >= {12192, 12250, 12287}
    assert any(b > S.DEFAULT_DYN_SMEM for b in hb.values())                               # the opt-in
    assert max(hb.values()) == S.K_MAX_HIST_BYTES                                          # 51 199 columns
    # block-loop boundaries: widths and rows around kRT and kScanT, not multiples of 32 for the transposes
    for k in (S.K_RT, S.K_SCAN_T):
        assert {k - 1, k, k + 1} <= widths and {k - 1, k, k + 1} <= rows
    assert any(w % 32 for w in widths) and any(n % 32 for n in rows)
    # gap runs: past one and four passes of the suffix scan, from column 1 and to column W
    lens = {c["name"]: S.run_lengths(c["rows"]) for c in cases}
    assert max(lens["run257"]) == S.K_RT + 1 and max(lens["run1025"]) == S.K_SCAN_T + 1 and longest > 4 * S.K_RT
    for c in cases:
        if c["name"] in ("run_from_col1", "run_to_colW"):
            assert max(S.run_lengths(c["rows"])) == c["rows"].shape[1] - 1
    assert any(s == 1 for c in cases for _, s, _ in runs_of(c["rows"]) if c["name"] == "run_from_col1")
    assert any(e == c["rows"].shape[1] for c in cases for _, _, e in runs_of(c["rows"]) if c["name"] == "run_to_colW")


def test_refine_cases_reach_every_boundary():
    cases = S.refine_cases()
    assert len({c["name"] for c in cases}) == len(cases)
    widths = {c["rows"].shape[1] for c in cases}
    rows = {c["rows"].shape[0] for c in cases}
    assert {1023, 1024, 1025, 2049} <= widths and {1023, 1024, 1025} <= rows
    assert any(S.WINDOW[0] <= w <= S.WINDOW[1] for w in widths)
    for c in cases:
        assert S.well_formed(c["rows"]), c["name"]
        assert len(c["ids"]) == c["rows"].shape[0] and len(set(c["ids"])) == len(c["ids"])
    ids = next(c["ids"] for c in cases if c["name"] == "ids_not_padded")
    assert rc.id_order(ids) != list(range(len(ids)))                       # s10 sorts before s2


def test_two_group_sides_and_orientations():
    """Every partially gapped column splits off row 0's group; the first split's sides have the claimed rows; and the
    prep kernel's orientation rule (dp_shapes.label) on the condensed sides' tables differs between the two variants
    of each side size."""
    g, sm = rc.scoring(100)
    seen = {}
    for c in S.refine_cases():
        if "sides" not in c["claims"]:
            continue
        a = c["rows"]
        big, small = c["claims"]["sides"]
        gp = a == S.GAP
        part = [gp[:, k] == gp[0, k] for k in np.flatnonzero(gp.any(axis=0) & ~gp.all(axis=0))]
        assert all(np.array_equal(p, part[0]) for p in part), c["name"]
        p1, p2 = S.sides(a)
        assert (p1.shape[0], p2.shape[0]) == (big, small), c["name"]
        assert S.well_formed(p1) and S.well_formed(p2)
        lab = dp_shapes.label((*S.tables(p1, sm, g), *S.tables(p2, sm, g)))
        assert lab["var"] == 2
        seen.setdefault(big, {})[c["claims"]["row0_diverse"]] = lab["sw"]
    assert set(seen) == set(S.SIDE_ROWS)
    for s, o in seen.items():
        assert set(o) == {True, False} and o[True] != o[False], s
    assert {s for s in seen if s > S.K_OPT_T} and {s for s in seen if s < S.K_OPT_T} and S.K_OPT_T in seen


def test_edge_cases():
    a = S.too_wide()
    assert a.shape[1] == S.MAX_WIDTH + 1 and S.hist_bytes(a.shape[1]) > S.K_MAX_HIST_BYTES and S.well_formed(a)
    rows, sm, gaps = S.growing_realignment()
    assert not (rows == S.GAP).any() and (sm < 0).all() and not gaps.any()
    assert 2 * rows.shape[1] > S.MAX_WIDTH >= rows.shape[1]


@need_ref
def test_total_score_rows_equals_reference_on_small_score_cases():
    n_checked = 0
    for c in S.score_cases():
        a = c["rows"]
        if a.shape[1] * a.shape[0] > 400_000 or a.shape[1] > 2100:
            continue
        g, sm = rc.scoring(a.shape[0])
        ref = ro.RefRefine(sm, g)
        want = ref.total_score([rc.to_letters(r) for r in a])
        ref.close()
        assert ro.total_score_rows(a, S.tables(a, sm, g)[1], sm, g) == want, c["name"]
        n_checked += 1
    assert n_checked >= 20
