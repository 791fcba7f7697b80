"""FAMSA's profile-profile mode (famsa in1 in2 out) on the device: famsa_prof_put_rows twice, famsa_prof_merge_batch once,
profiles.rows_after_merge.  Checked bit for bit against the golden upgma.pp.fasta (without the reference) and against the
reference's own CProfile (oracle/_ref) on alignments with all-gap columns: the put tables, total, width, path,
orientation, variant, the merged resident profile's tables, and the rows and their order."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import profile_mode_cases as pmc
from cpp_build import build_cpp
import refine_cases as rc
import refine_oracle as ro
import refine_shapes as S
from conftest import ROOT
from famsa_b200 import profiles, seqio
from famsa_b200.binding import FamsaError
from oracle import pyoracle

pytestmark = pytest.mark.gpu
need_ref = pytest.mark.skipif(not pyoracle.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def eng():
    import famsa_b200
    e = famsa_b200.Engine(0)
    yield e
    e.close()


def device_mode(eng, rows1, rows2, gaps, sm, from_text=True):
    """put, put, merge: (tables of the two puts, merge result dict, merged id, order, rows)."""
    eng.prof_set_scoring(sm)
    ids = [eng.prof_put_rows(pmc.encode(r), gaps, from_text=from_text) for r in (rows1, rows2)]
    puts = [eng.prof_get(i) for i in ids]
    w = [p[0].shape[0] - 1 for p in puts]
    (merged,), (res,) = eng.prof_merge_batch([tuple(ids)], gaps, [tuple(w)])
    order, rows = profiles.rows_after_merge(rows1, rows2, res["path"], res["swapped"], from_text=from_text)
    return puts, res, merged, order, rows


def test_golden_upgma_pp(eng):
    """upgma.no_refine.part{1,2}.fasta -> upgma.pp.fasta, without the reference."""
    z = np.load(os.path.join(GOLDEN, "adeno_pp_rows.npz"))
    pp = np.load(os.path.join(GOLDEN, "adeno_pp.npz"))
    rows1, rows2 = [str(x) for x in z["rows1"]], [str(x) for x in z["rows2"]]
    g, sm = z["gaps"], z["score_matrix"]
    puts, res, merged, order, rows = device_mode(eng, rows1, rows2, g, sm)
    for (s, c, k), key in zip(puts, "12"):
        assert np.array_equal(s, pp["s" + key]) and np.array_equal(c, pp["c" + key]) and k == int(pp["k" + key])
    assert res["total"] == int(pp["total"]) and np.array_equal(res["path"], pp["path"]) and res["swapped"] == bool(pp["swapped"])
    eng.prof_drop([merged])
    out = eng.align_profiles(rows1, rows2, g)
    names = [str(x) for x in z["ids1"]] + [str(x) for x in z["ids2"]]
    assert [names[k] for k in out["order"]] == [str(x) for x in z["gold_ids"]]
    assert out["rows"] == [str(x) for x in z["gold_rows"]]
    assert out["width"] == len(out["rows"][0]) == 261 and out["total"] == int(pp["total"])
    eng.prof_drop([out["merged_id"]])
    assert eng.prof_stats()[0] == 0


def check_against_reference(eng, rows1, rows2, gaps=None, matrix_type=2):
    ref = pmc.reference_merge(rows1, rows2, gaps, matrix_type)
    g, sm = ref["gaps"], ref["score_matrix"]
    puts, res, merged, order, rows = device_mode(eng, rows1, rows2, g, sm)
    for (s, c, k), (rs, rcn, rk) in zip(puts, (ref["t1"], ref["t2"])):
        assert k == rk and np.array_equal(c, rcn) and np.array_equal(s, rs)
    assert res["total"] == ref["total"] and res["swapped"] == pmc.reference_swapped(ref, len(rows1))
    (s1, c1, k1), (s2, c2, k2) = ref["t1"], ref["t2"]
    o = pyoracle.dp_align(s1, c1, k1, s2, c2, k2, g, sm)
    # the C restatement reads the tables cut at width - 1 and so misses the set-aside column in ProfProf's orientation;
    # where that decides, the merged tables, order and rows below pin the device against the reference
    if o["swapped"] == res["swapped"]:
        assert np.array_equal(res["path"], o["path"]) and res["variant"] == o["variant"] and o["total"] == res["total"]
    ms, mc, mk = eng.prof_get(merged)
    assert mk == len(rows1) + len(rows2) and ms.shape == ref["merged"][0].shape
    assert np.array_equal(mc, ref["merged"][1]) and np.array_equal(ms, ref["merged"][0])
    assert order == ref["order"]
    assert [pmc.normalise(r) for r in rows] == ref["rows"]
    eng.prof_drop([merged])
    return res


@need_ref
@pytest.mark.parametrize("case", pmc.case_matrix(), ids=lambda c: c[0])
def test_case_matrix(eng, case):
    _, rows1, rows2 = case
    check_against_reference(eng, rows1, rows2)


@need_ref
@pytest.mark.parametrize("case", pmc.orientation_cases(), ids=lambda c: c[0])
def test_orientation_boundary(eng, case):
    """ProfProf orientations that the set-aside last column of rows read as text decides."""
    _, rows1, rows2 = case
    res = check_against_reference(eng, rows1, rows2)
    assert res["swapped"] == pmc.text_orientation(rows1, rows2)


def test_one_row_with_the_last_column_gapped(eng):
    """With FAMSA_PUT_ROWS_FROM_TEXT a one-row alignment may have a gap in the set-aside column: its profile is the
    ungapped rest.  Without the flag that gap is in the profile and the row is rejected."""
    z = np.load(os.path.join(GOLDEN, "adeno_pp_rows.npz"))
    g, sm = z["gaps"], z["score_matrix"]
    eng.prof_set_scoring(sm)
    row = pmc.encode(["ARNDC-"])
    pid = eng.prof_put_rows(row, g, from_text=True)
    s, c, k = eng.prof_get(pid)
    hs, hc, _ = profiles.tables_from_rows(pmc.as_gap_neg(pmc.encode(["ARNDC"])), sm, g)
    assert k == 1 and np.array_equal(s, hs) and np.array_equal(c, hc)
    eng.prof_drop([pid])
    with pytest.raises(FamsaError, match=r"^\[1\]"):
        eng.prof_put_rows(row, g)
    rows1, rows2 = ["ARNDC-"], pmc.alignment(6, 9, np.random.default_rng(80), (0, -1))
    if pyoracle.have_ref():
        check_against_reference(eng, rows1, rows2)


def test_one_by_one(eng):
    """Two one-row inputs (AlignSeqSeq), against the C restatement on the host tables."""
    rows1, rows2 = pmc.one_by_one()
    z = np.load(os.path.join(GOLDEN, "adeno_pp_rows.npz"))
    g, sm = z["gaps"], z["score_matrix"]
    puts, res, merged, order, rows = device_mode(eng, rows1, rows2, g, sm)
    for (s, c, k), r in zip(puts, (rows1, rows2)):
        hs, hc, hk = profiles.tables_from_rows(pmc.as_gap_neg(pmc.encode(r)), sm, g)
        assert k == hk == 1 and np.array_equal(s, hs[:-1]) and np.array_equal(c, hc[:-1])
    o = pyoracle.dp_align(*puts[0], *puts[1], g, sm)
    assert res["variant"] == o["variant"] == 0 and res["total"] == o["total"] and np.array_equal(res["path"], o["path"])
    assert [r.replace("-", "") for r in rows] == [(rows1 + rows2)[k] for k in order]
    eng.prof_drop([merged])


def sized_cases():
    rng = np.random.default_rng(77)
    out = []
    for n in (127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025):
        out.append((f"rows{n}", pmc.alignment(n, 60, rng, (0, 30, -1), gap_frac=0.2), pmc.alignment(40, 50, rng, (-2,))))
    for w in (255, 256, 257):
        out.append((f"width{w}", pmc.alignment(20, w, rng, (1, w // 2, -1)), pmc.alignment(15, w - 40, rng, (0,))))
    out.append(("width4200", pmc.alignment(6, 4200, rng, (0, 2100, 2101, -1), gap_frac=0.1), pmc.alignment(5, 4150, rng, (7,), gap_frac=0.1)))
    return out


@need_ref
@pytest.mark.parametrize("case", sized_cases(), ids=lambda c: c[0])
def test_sizes(eng, case):
    _, rows1, rows2 = case
    check_against_reference(eng, rows1, rows2)


@need_ref
def test_gap_costs_and_matrix(eng):
    rng = np.random.default_rng(78)
    rows1, rows2 = pmc.alignment(30, 70, rng, (0, 33, -1), lower=0.2), pmc.alignment(22, 64, rng, (5, 6, 7))
    check_against_reference(eng, rows1, rows2, gaps=(-9000, -700, -300, -100))
    check_against_reference(eng, rows1, rows2, gaps=(-20000, -2000, -2500, -900))
    check_against_reference(eng, rows1, rows2, matrix_type=0)


@need_ref
def test_large(eng):
    """About 20 000 + 15 000 rows of about 1 200 columns with all-gap columns."""
    rng = np.random.default_rng(79)
    rows1 = pmc.alignment(20000, 1200, rng, (0, 400, 401, 402, 900, -2, -1), gap_frac=0.1)
    rows2 = pmc.alignment(15000, 1180, rng, (3, 600, -1), gap_frac=0.1)
    ref = pmc.reference_merge(rows1, rows2)
    g, sm = ref["gaps"], ref["score_matrix"]
    eng.prof_set_scoring(sm)
    for rows in (rows1, rows2):                                          # the whole rows, without the text rule
        pid = eng.prof_put_rows(pmc.encode(rows), g)
        s, c, k = eng.prof_get(pid)
        hs, hc, hk = profiles.tables_from_rows(pmc.as_gap_neg(pmc.encode(rows)), sm, g)
        assert k == hk and np.array_equal(c, hc) and np.array_equal(s, hs)
        eng.prof_drop([pid])
    check_against_reference(eng, rows1, rows2)


def test_errors(eng):
    import famsa_b200
    e = famsa_b200.Engine(0)
    z = np.load(os.path.join(GOLDEN, "adeno_pp_rows.npz"))
    g, sm = z["gaps"], z["score_matrix"]
    good = pmc.encode(["AR-N", "-RDN"])
    with pytest.raises(FamsaError, match=r"^\[4\]"):
        e.prof_put_rows(good, g)                                           # no famsa_prof_set_scoring
    e.prof_set_scoring(sm)
    bad = {
        "no rows": np.zeros((0, 4), np.uint8),
        "no columns": np.zeros((2, 0), np.uint8),
        "code 24": np.array([[0, 24, 30]], np.uint8).repeat(2, 0),
        "code 31": np.array([[0, 1, 31], [1, 2, 3]], np.uint8),
        "row without residue": np.array([[0, 1, 2], [30, 30, 30]], np.uint8),
        "one gapped row": np.array([[0, 30, 2]], np.uint8),
    }
    for name, rows in bad.items():
        with pytest.raises(FamsaError, match=r"^\[1\]"):
            e.prof_put_rows(rows, g)
        assert e.prof_stats() == (0, 0), name
    with pytest.raises(FamsaError, match=r"^\[1\]"):
        e.prof_put_rows(np.array([[0], [1]], np.uint8), g, from_text=True)  # no column left
    gg = np.ascontiguousarray(g, dtype=np.int64)
    pid = C.c_uint32()
    for args in [(None, gg.ctypes.data, 0, C.byref(pid)), (good.ctypes.data, None, 0, C.byref(pid)),
                 (good.ctypes.data, gg.ctypes.data, 0, None), (good.ctypes.data, gg.ctypes.data, 2, C.byref(pid))]:
        rows_p, gaps_p, flags, out = args                                 # NULL pointers, unknown flags
        assert e.lib.famsa_prof_put_rows(e.h, rows_p, 2, 4, gaps_p, flags, out) == 1
    assert e.prof_stats() == (0, 0)
    with pytest.raises(ValueError):
        e.align_profiles([], ["AR"], g)
    with pytest.raises(ValueError):
        e.align_profiles(["AR-", "A"], ["AR"], g)
    ok = e.prof_put_rows(good, g)
    assert e.prof_get(ok, tables=False) == (4, 2)
    e.prof_drop([ok])
    assert e.prof_stats() == (0, 0)
    e.close()


def refine_root_case():
    return next(c for c in S.refine_cases() if c["name"] == "ids_not_padded")


@pytest.mark.skipif(not pyoracle.have("ref_refine", "rr_refine_rows"),
                    reason="oracle/_ref/libfamsa_ref_refine.so not built, or built without rr_refine_rows")
def test_refine_root_and_refine_state(eng):
    """A user's alignment as a refine root: famsa_prof_put_rows -> famsa_prof_refine is RefineAlignment of those rows.  A
    later famsa_prof_put_rows leaves famsa_prof_refined_rows alone."""
    c = refine_root_case()
    rows, ids = c["rows"], c["ids"]
    n = rows.shape[0]
    g, sm = rc.scoring(n)
    order = rc.id_order(ids)
    arr = np.ascontiguousarray(rows[order])
    eng.prof_set_scoring(sm)
    root = eng.prof_put_rows(arr, g)
    out, width, total, stats, rid = eng.refine(root, arr, g, c["n_refinements"])
    ref = ro.RefRefine(sm, g)
    want = ref.refine_rows([rc.to_letters(r) for r in rows], ids, c["n_refinements"])
    ref.close()
    got = [None] * n
    for k, i in enumerate(order):
        got[i] = rc.to_letters(out[k])
    assert width == want["width"] and total == want["total"] and got == want["refined"]
    other = eng.prof_put_rows(pmc.encode(["AR-N", "-RDN", "WW-W"]), g)
    again = np.zeros_like(out)
    eng._check(eng.lib.famsa_prof_refined_rows(eng.h, again.ctypes.data, again.size))
    assert np.array_equal(again, out)
    eng.prof_drop([rid, other])


def test_host_mirror_runs(tmp_path):
    """famsa_b200::AlignProfiles reproduces upgma.pp.fasta through FinalizeGaps' runs and the output order."""
    import subprocess
    exe = build_cpp("test_host_profiles", tmp_path, famsa=True)
    pmc.host_mirror_input(tmp_path / "pp.txt")
    out = subprocess.run([exe, str(tmp_path / "pp.txt")], capture_output=True, text=True)
    assert out.returncode == 0 and "host mirror profiles ok" in out.stdout, out.stdout + out.stderr
