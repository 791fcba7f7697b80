"""famsa_prof_refine at the boundaries of refine.cu's kernels (cases: tests/refine_shapes.py), on hand-built alignments
put resident with prof_put:

* the input's total score (n_refinements = 0) at widths and row counts around the block loops and scans, at every side
  of k_ref_score_runs' shared-memory limits (the widths just past the default budget once in a fresh process, so no
  earlier opt-in in the process can hide a launch failure), with long and terminal gap runs, against the vectorised
  total_score_rows and, where it is affordable, the reference's CalculateTotalScore;
* the whole loop against the reference's RefineAlignment of the same rows (oracle/ref_refine_harness.cpp
  rr_refine_rows): rows, width, total, loop counts and the refined profile's tables;
* the width limit before and inside the loop, and the release of every profile the failing call held;
* FAMSA's own refined adeno_fiber alignments (tests/golden/adeno_refined.npz) through align_tree -> refine."""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np
import pytest

import refine_cases as rc
import refine_oracle as ro
import refine_shapes as S
from famsa_b200.binding import REFINE_NO_TOTAL_SCORE, FamsaError
from oracle import pyoracle

pytestmark = pytest.mark.gpu
need_ref = pytest.mark.skipif(not pyoracle.have("ref_refine", "rr_refine_rows"),
                              reason="oracle/_ref/libfamsa_ref_refine.so not built, or built without rr_refine_rows")
HERE = os.path.dirname(os.path.abspath(__file__))
SCORE = {c["name"]: c for c in S.score_cases()}
REFINE = {c["name"]: c for c in S.refine_cases()}
WINDOW_CASES = ["w12191_n2", "w12192_n2", "w12287_n5"]


@pytest.fixture(scope="module")
def eng():
    import famsa_b200
    e = famsa_b200.Engine(0)
    yield e
    e.close()


def put_root(eng, rows, sm, g) -> int:
    eng.prof_set_scoring(sm)
    return eng.prof_put([S.tables(rows, sm, g)])[0]


def score_on_device(eng, rows, sm, g, flags=0):
    root = put_root(eng, rows, sm, g)
    out, width, total, stats, rid = eng.refine(root, rows, g, 0, flags)
    eng.prof_drop([rid])
    assert rid == root and stats["n_tries"] == 0
    return out, width, total


def _window_child():
    """Run in a fresh process: the totals of the cases at the default shared-memory limit, narrowest first, before any
    wider call could have raised k_ref_score_runs' limit."""
    import famsa_b200
    e = famsa_b200.Engine(0)
    res = {}
    for name in WINDOW_CASES:
        a = SCORE[name]["rows"]
        g, sm = rc.scoring(a.shape[0])
        try:
            res[name] = dict(total=int(score_on_device(e, a, sm, g)[2]))
        except FamsaError as err:
            res[name] = dict(error=str(err))
    e.close()
    print(json.dumps(res))


def test_score_at_the_default_shared_memory_limit_in_a_fresh_process():
    code = (f"import sys; sys.path[:0] = [{HERE!r}, {os.path.dirname(HERE)!r}]; "
            "import test_refine_shapes_gpu as t; t._window_child()")
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    for name in WINDOW_CASES:
        a = SCORE[name]["rows"]
        g, sm = rc.scoring(a.shape[0])
        assert "error" not in got[name], f"{name}: {got[name]}"
        assert got[name]["total"] == ro.total_score_rows(a, S.tables(a, sm, g)[1], sm, g), name


@pytest.mark.parametrize("name", list(SCORE))
def test_score(eng, name):
    a = SCORE[name]["rows"]
    n, w = a.shape
    g, sm = rc.scoring(n)
    out, width, total = score_on_device(eng, a, sm, g)
    assert width == w and np.array_equal(out, a), "n_refinements = 0 must return the rows unchanged"
    want = ro.total_score_rows(a, S.tables(a, sm, g)[1], sm, g)
    assert total == want
    if w <= 4096 and pyoracle.have("ref_refine"):
        ref = ro.RefRefine(sm, g)
        assert total == ref.total_score([rc.to_letters(r) for r in a])
        ref.close()
    assert score_on_device(eng, a, sm, g, REFINE_NO_TOTAL_SCORE)[2] == 0


def check_refine(eng, rows, ids, n_refinements, sm=None, g=None):
    n = rows.shape[0]
    if sm is None:
        g, sm = rc.scoring(n)
    order = rc.id_order(ids)
    arr = np.ascontiguousarray(rows[order])
    root = put_root(eng, arr, sm, g)
    out, width, total, stats, rid = eng.refine(root, arr, g, n_refinements)
    got = [None] * n
    for k, i in enumerate(order):
        got[i] = rc.to_letters(out[k])
    ref = ro.RefRefine(sm, g)
    want = ref.refine_rows([rc.to_letters(r) for r in rows], ids, n_refinements)
    ref.close()
    assert want["prev_total"] == ro.total_score_rows(rows, S.tables(rows, sm, g)[1], sm, g)
    assert width == want["width"] and total == want["total"], \
        f"width {width} vs {want['width']}, total {total} vs {want['total']}, device {stats}, reference {want['counts']}"
    assert got == want["refined"]
    for k, v in want["counts"].items():
        assert stats[k] == v, f"{k}: {stats[k]} != {v}"
    sc, cn, card = eng.prof_get(rid)
    assert card == n and np.array_equal(cn, want["counters"]) and np.array_equal(sc, want["scores"])
    eng.prof_drop([rid])
    return stats, want


@need_ref
@pytest.mark.parametrize("name", list(REFINE))
def test_refine(eng, name):
    c = REFINE[name]
    stats, want = check_refine(eng, c["rows"], c["ids"], c["n_refinements"])
    assert stats["n_realigned"] >= 1
    print(f"{name}: {c['rows'].shape}, width -> {want['width']}, {want['counts']}")


def test_width_over_the_limit_is_rejected_before_the_loop(eng):
    a = S.too_wide()
    g, sm = rc.scoring(a.shape[0])
    root = put_root(eng, a, sm, g)
    with pytest.raises(FamsaError, match="51 199"):
        eng.refine(root, a, g, 0)
    assert eng.prof_get(root, tables=False) == (a.shape[1], a.shape[0])      # still resident
    eng.prof_drop([root])


@need_ref
def test_realignment_over_the_limit_releases_every_profile(eng):
    import ctypes as C
    rows, sm, gaps = S.growing_realignment()
    live0 = eng.prof_stats()[0]
    root = put_root(eng, rows, sm, gaps)
    assert eng.prof_stats()[0] == live0 + 1
    with pytest.raises(FamsaError, match=r"a realignment is \d+ columns wide") as err:
        eng.refine(root, rows, gaps, 100)
    assert int(str(err.value).split("a realignment is ")[1].split()[0]) > S.MAX_WIDTH
    assert eng.prof_stats()[0] == live0, "profiles of the failed call stay resident"
    with pytest.raises(FamsaError):
        eng.prof_get(root, tables=False)
    buf = np.zeros(rows.size, dtype=np.uint8)
    assert eng.lib.famsa_prof_refined_rows(eng.h, C.c_void_p(buf.ctypes.data), buf.size) == 4        # FAMSA_E_STATE
    c = REFINE["w1023_n128"]
    check_refine(eng, c["rows"], c["ids"], c["n_refinements"])


@pytest.mark.parametrize("name", ["upgma", "sl"])
def test_famsa_refined_golden(eng, name):
    """The progressive alignment along the golden's guide tree, then the refinement: FAMSA's own refined output."""
    z = np.load(os.path.join(HERE, "golden", "adeno_refined.npz"))
    t = np.load(os.path.join(HERE, "golden", "adeno_upgma_merges.npz"))
    g, sm = t["gaps"], t["score_matrix"]                                     # 242 sequences either way
    if name == "upgma":
        seqs, merges = [str(s) for s in t["seqs"]], t["merges"]
    else:
        t = np.load(os.path.join(HERE, "golden", "adeno_sl_tree.npz"))
        seqs, merges = [str(s) for s in t["seqs"]], t["tree"][len(t["seqs"]):]
    ids = [str(i) for i in z[f"{name}_ids"]]
    gold = z[f"{name}_rows"]
    rows, width, total, stats, rid = rc.device_refine(eng, seqs, merges, g, sm, 100, ids=ids)
    eng.prof_drop([rid])
    assert width == gold.shape[1]
    assert all(rows[i] == rc.to_letters(gold[i]) for i in range(len(seqs)))
