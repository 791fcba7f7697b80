"""CPU tests of tests/lcs_shapes.py: its limb-count table follows the kernel's, its sets reach every tile-kernel
instantiation at both ends of its length range, and its data can tell a correct kernel from a subtly wrong one."""
import os
import re

import numpy as np
import pytest

from famsa_b200 import seqio
from lcs_shapes import (INSTANTIATED, carry_set, group_nls, lcs_dropped_limb_carry, nl_range, quirk_set, quirky,
                        sweep_set, tile_nl, true_lcs)
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_instantiated_matches_launch_switch():
    """INSTANTIATED is the FB_CASE list of launch_tile_nl, and every length the tile kernel takes maps onto it."""
    src = open(os.path.join(ROOT, "famsa_b200", "csrc", "lcs.cu")).read()
    body = re.search(r"static int launch_tile_nl\(.*?\n}\n", src, re.S).group(0)
    cases = [int(x) for x in re.findall(r"FB_CASE\((\d+)\)\s", body)]
    assert tuple(cases) == INSTANTIATED
    assert {tile_nl(L) for L in range(1, 2049)} == set(INSTANTIATED)
    assert tile_nl(0) == 1 and tile_nl(2049) == 0
    for nl in INSTANTIATED:
        lo, hi = nl_range(nl)
        assert tile_nl(lo) == tile_nl(hi) == nl and tile_nl(hi + 1) != nl
        assert lo == 1 or tile_nl(lo - 1) != nl


@pytest.mark.parametrize("nl", INSTANTIATED)
def test_sweep_set_shape(nl):
    """Groups with nl limbs led by both ends of nl's range, a partial last group, every length residue mod 16, empty
    sequences, B/Z/X/*, and no row that the exact kernels would take over."""
    s = sweep_set(nl)
    lo, hi = nl_range(nl)
    for order in ("unsorted", "sorted"):
        lens = np.array([len(c) for c in s[order]])
        assert len(lens) % 32 != 0
        srt = np.sort(lens)[::-1]
        leads = srt[::32]
        assert hi in leads and lo in leads
        assert group_nls(lens)[:2] == [nl, nl]
        assert set(lens % 16) == set(range(16))
        assert lens.min() == 0
    assert [len(c) for c in s["sorted"]] == sorted((len(c) for c in s["unsorted"]), reverse=True)
    allc = np.concatenate(s["unsorted"])
    assert set(range(20, 24)) <= set(allc.tolist())
    assert not any(quirky(c) for c in s["unsorted"])


def test_sweep_sets_reach_every_instantiation():
    reached = set()
    for nl in INSTANTIATED:
        reached.update(group_nls([len(c) for c in sweep_set(nl)["unsorted"]]))
    assert reached == set(INSTANTIATED)


@pytest.mark.parametrize("nl", [n for n in INSTANTIATED if n >= 2])
def test_carry_set_detects_every_dropped_limb_carry(nl):
    """For every limb boundary b of nl limbs, dropping the carry into limb b changes the LCS of some (carry row, streamed
    sequence) pair that the GPU tests compute with the carry row as the mask side of an nl-limb group."""
    s = carry_set(nl)
    cl = s["unsorted"]
    r = s["row"]["unsorted"]
    row = cl[r]
    assert not quirky(row) and not any(quirky(c) for c in cl)
    lens = np.array([len(c) for c in s["sorted"]])
    g = s["row"]["sorted"] // 32
    assert tile_nl(lens[32 * g]) == nl
    codes, offsets, lens_u = seqio.pack(cl)
    want = pyoracle.lcs_rows(codes, offsets, lens_u, [r])[0]
    cols = sorted((k for k in range(len(cl)) if k != r), key=lambda k: len(cl[k]))
    for k in cols[:4] + cols[-2:]:
        assert lcs_dropped_limb_carry(row, cl[k], nl, 0) == want[k] == true_lcs(row, cl[k])
    for b in range(1, nl):
        assert any(lcs_dropped_limb_carry(row, cl[k], nl, b) != want[k] for k in cols), f"boundary {b} of {nl} limbs"


def test_quirk_rows_are_live_and_near_misses_are_not():
    """Flagged rows (an aligned 64-run) reach the dropped-carry corner: some column's reference LCS differs from the true
    LCS.  The exception is a run in word 0, which no carry enters -- flagged all the same, and equal to the true LCS.
    Near misses are not flagged and equal the true LCS in every column."""
    s = quirk_set()
    cl = s["unsorted"]
    n = len(cl)
    codes, offsets, lens = seqio.pack(cl)
    flagged, near, word0 = s["flagged"]["unsorted"], s["near"]["unsorted"], s["word0"]["unsorted"]
    assert [k for k in range(n) if quirky(cl[k])] == flagged
    assert [k for k in range(n) if quirky(s["sorted"][k])] == s["flagged"]["sorted"]
    assert not set(near) & set(flagged) and word0 in flagged
    rows = flagged + near
    got = pyoracle.lcs_rows(codes, offsets, lens, rows)
    for r, k in enumerate(rows):
        differs = [j for j in range(n) if got[r, j] != true_lcs(cl[k], cl[j])]
        if k in near or k == word0:
            assert not differs, f"row {k}"
        else:
            assert differs, f"flagged row {k} never reaches the dropped-carry corner"


def test_oracle_equals_true_lcs_across_nl_range():
    """Without a flagged row the reference's recurrence is the true LCS: 8 pairs per instantiation (320 pairs), rows of
    every limb count against streamed sequences of every length class, checked with the plain DP."""
    rng = np.random.default_rng(77)
    checked = 0
    for nl in INSTANTIATED:
        cl = sweep_set(nl)["unsorted"]
        codes, offsets, lens = seqio.pack(cl)
        rows = rng.choice(len(cl), size=4, replace=False)
        cols = rng.choice(len(cl), size=2, replace=False)
        got = pyoracle.lcs_rows(codes, offsets, lens, rows, cols)
        for a, r in enumerate(rows):
            for b, c in enumerate(cols):
                assert got[a, b] == true_lcs(cl[r], cl[c]), (nl, r, c)
                checked += 1
    assert checked >= 300
