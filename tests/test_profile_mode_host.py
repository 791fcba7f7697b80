"""CPU tests of FAMSA's profile-profile mode (famsa in1 in2 out): the order-and-rows rule (profiles.rows_after_merge), the
host tables of gapped alignments with all-gap columns (profiles.tables_from_rows) and the gapped encoding, against the
reference's CProfile (oracle/_ref; those tests skip without it)."""
import os

import numpy as np
import pytest

from conftest import ROOT
from famsa_b200 import profiles, seqio
from oracle import pyoracle
import profile_mode_cases as pmc
from cpp_build import build_cpp

need_ref = pytest.mark.skipif(not pyoracle.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")


def test_encode_gapped():
    row = "-aRn*-XbJu--z"
    codes = seqio.encode_gapped(row)
    assert codes.dtype == np.uint8 and len(codes) == len(row)
    assert list(np.flatnonzero(codes == seqio.GAP)) == [i for i, c in enumerate(row) if c == "-"]
    res = codes[codes != seqio.GAP]
    assert np.array_equal(res, seqio.encode(row).astype(np.uint8))
    assert seqio.decode(seqio.encode_gapped("ARNDCQEGHILKMFPSTWYVBZX*")) == "ARNDCQEGHILKMFPSTWYVBZX*"
    assert list(seqio.encode_gapped("jou?")) == [seqio.UNKNOWN] * 4


def test_rows_after_merge_rule():
    rows1 = ["aC-d", "-xYz"]                  # 4 columns
    rows2 = ["MNp", "uv-", "k-L"]             # 3 columns
    path = np.array([0, 2, 1, 0, 2], dtype=np.uint8)
    # swapped False: rows1 is the DP's row side (D and V consume it), rows2 the column side (D and H)
    order, rows = profiles.rows_after_merge(rows1, rows2, path, False)
    assert order == [2, 3, 4, 0, 1]
    col = lambda r: r[0] + "-" + r[1] + r[2] + "-"          # V at 2 and 5 insert gap columns into the column side
    row = lambda r: r[0] + r[1] + "-" + r[2] + r[3]         # H at 3 inserts a gap column into the row side
    assert rows == [col(r) for r in rows2] + [row(r) for r in rows1]
    # swapped True: rows2 is the row side
    path2 = np.array([0, 1, 2, 0, 1], dtype=np.uint8)       # row side rows2: D V D = 3; column side rows1: D H D H = 4
    order, rows = profiles.rows_after_merge(rows1, rows2, path2, True)
    assert order == [0, 1, 2, 3, 4]
    assert rows == [r[0] + r[1] + "-" + r[2] + r[3] for r in rows1] + [r[0] + "-" + r[1] + r[2] + "-" for r in rows2]
    with pytest.raises(ValueError):
        profiles.rows_after_merge(rows1, rows2, path2[:-1], True)
    # from text: the last column of every row stays apart and ends the merged row
    order, rows = profiles.rows_after_merge([r + "q" for r in rows1], [r + "-" for r in rows2], path2, True, from_text=True)
    assert rows == [r[0] + r[1] + "-" + r[2] + r[3] + "q" for r in rows1] + [r[0] + "-" + r[1] + r[2] + "-" + "-" for r in rows2]


@need_ref
@pytest.mark.parametrize("case", pmc.case_matrix(), ids=lambda c: c[0])
def test_rows_after_merge_equals_reference(case):
    """rows_after_merge driven by the C restatement's path and orientation gives the reference's merged rows and order."""
    _, rows1, rows2 = case
    ref = pmc.reference_merge(rows1, rows2)
    (s1, c1, k1), (s2, c2, k2) = ref["t1"], ref["t2"]
    o = pyoracle.dp_align(s1, c1, k1, s2, c2, k2, ref["gaps"], ref["score_matrix"])
    assert o["total"] == ref["total"]
    order, rows = profiles.rows_after_merge(rows1, rows2, o["path"], o["swapped"], from_text=True)
    assert order == ref["order"]
    assert [pmc.normalise(r) for r in rows] == ref["rows"]
    inputs = rows1 + rows2
    assert [r.replace("-", "") for r in rows] == [inputs[k].replace("-", "") for k in order]   # letters kept as given


@need_ref
@pytest.mark.parametrize("case", pmc.case_matrix(), ids=lambda c: c[0])
def test_tables_from_rows_equal_reference(case):
    """The host tables of gapped rows with all-gap columns are the reference's; CFAMSA::alignProfiles' profile of rows
    read as text is the same without its last column."""
    _, rows1, rows2 = case
    ref = pmc.reference_merge(rows1, rows2)
    for rows, (s, c, k) in ((rows1, ref["t1"]), (rows2, ref["t2"])):
        hs, hc, hk = profiles.tables_from_rows(pmc.as_gap_neg(pmc.encode(rows)), ref["score_matrix"], ref["gaps"])
        assert hk == k == len(rows)
        assert np.array_equal(hs[:-1], s) and np.array_equal(hc[:-1], c)


@need_ref
def test_case_matrix_orientations():
    """The reference's order pins both ProfProf orientations among the case matrix, and the restated text rule gives it."""
    seen = set()
    for name, rows1, rows2 in pmc.case_matrix():
        ref = pmc.reference_merge(rows1, rows2)
        sw = pmc.reference_swapped(ref, len(rows1))
        if len(rows1) > 1 and len(rows2) > 1:
            assert sw == pmc.text_orientation(rows1, rows2), name
            seen.add(sw)
    assert seen == {False, True}


@need_ref
def test_orientation_cases_turn_on_the_set_aside_column():
    """Each orientation case is decided by the set-aside column: the reference's orientation is the restated text rule's,
    and not the one its tables cut at width - 1 give."""
    seen = set()
    for name, rows1, rows2 in pmc.orientation_cases():
        ref = pmc.reference_merge(rows1, rows2)
        sw = pmc.reference_swapped(ref, len(rows1))
        assert sw == pmc.text_orientation(rows1, rows2), name
        (s1, c1, k1), (s2, c2, k2) = ref["t1"], ref["t2"]
        assert pyoracle.dp_align(s1, c1, k1, s2, c2, k2, ref["gaps"], ref["score_matrix"])["swapped"] != sw, name
        seen.add(sw)
    assert seen == {False, True}


def test_golden_fixture_rule():
    """adeno_pp_rows.npz: the fixture's path and orientation give upgma.pp.fasta's rows, order and letter case."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "adeno_pp_rows.npz"))
    rows1, rows2 = [str(x) for x in z["rows1"]], [str(x) for x in z["rows2"]]
    names = [str(x) for x in z["ids1"]] + [str(x) for x in z["ids2"]]
    order, rows = profiles.rows_after_merge(rows1, rows2, z["path"], bool(z["swapped"]), from_text=True)
    assert [names[k] for k in order] == [str(x) for x in z["gold_ids"]]
    assert rows == [str(x) for x in z["gold_rows"]]
    assert order[:len(rows2)] == list(range(len(rows1), len(rows1) + len(rows2)))      # part2's rows first
    assert any(c.islower() for r in rows for c in r)
    pp = np.load(os.path.join(ROOT, "tests", "golden", "adeno_pp.npz"))
    for rows, key in ((rows1, "1"), (rows2, "2")):
        s, c, k = profiles.tables_from_rows(pmc.as_gap_neg(pmc.encode(rows)), z["score_matrix"], z["gaps"])
        assert np.array_equal(s[:-1], pp["s" + key]) and np.array_equal(c[:-1], pp["c" + key])
    assert np.array_equal(z["path"], pp["path"]) and int(z["total"]) == int(pp["total"])


def test_host_mirror_compiles(tmp_path):
    build_cpp("test_host_profiles", tmp_path, famsa=True)
    pmc.host_mirror_input(tmp_path / "pp.txt")
