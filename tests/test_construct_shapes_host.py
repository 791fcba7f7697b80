"""CPU tests of tests/construct_shapes.py: the constants it is built on are the kernel's, every case reaches the classes it
claims and the cases together reach every class of construct_tile's derivation; the C restatement of the reference's walk
(dp_construct) equals the reference's own ConstructProfile on every case; and the numpy restatement of construct_tile's
independent-column formulas equals dp_construct on every case and on thousands of random monotone paths, paths no DP
would choose included."""
import os
import re

import numpy as np
import pytest

import construct_shapes as S
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
need_ref = pytest.mark.skipif(not pyoracle.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")
CASES = S.cases()


def _src(name):
    return open(os.path.join(ROOT, "famsa_b200", "csrc", name)).read()


def test_constants_match_the_sources():
    dev = _src("prof_dev.cuh")
    assert re.search(r"constexpr int kConThreads = 256, kConTile = (\d+);", dev).group(1) == str(S.TILE)
    m = re.search(r"constexpr int kGO = (\d+), kGE = (\d+), kTE = (\d+), kTO = (\d+), kGAP = (\d+), kNAA = (\d+);", dev)
    assert tuple(int(x) for x in m.groups()) == (S.GO, S.GE, S.TE, S.TO, S.GAP_LANE, S.N_AA)
    plan = _src("tree_plan.h")
    assert int(re.search(r"kFusedMaxHostRows = (\d+);", plan).group(1)) == S.FUSED_MAX_HOST_ROWS
    assert int(re.search(r"kFusedMaxWidth = (\d+);", plan).group(1)) == S.FUSED_MAX_WIDTH


def test_cases_reach_their_classes_and_together_every_class():
    assert len({c["name"] for c in CASES}) == len(CASES)
    union = set()
    for c in CASES:
        t1, t2 = S.tables_of(c)
        res, _, _ = S.oracle_merge(c, t1, t2)
        got = S.case_classes(c, t1, t2, res)
        assert c["claims"] <= got, f"{c['name']} misses {sorted(c['claims'] - got)}"
        assert res["swapped"] == S.orientation(t1, t2), c["name"]
        union |= got
    assert union == set(S.ALL_CLASSES), f"not reached: {sorted(set(S.ALL_CLASSES) - union)}"


def test_fixture_matches_the_cases():
    """The fixture holds the cases as they are generated now (and the restatement's path, total and tables equal it)."""
    z = np.load(S.FIXTURE)
    assert [str(x) for x in z["names"]] == [c["name"] for c in CASES]
    for c, crcs, total, sw in zip(CASES, z["crcs"], z["totals"], z["swapped"]):
        res, s, cn = S.oracle_merge(c)
        t1, t2 = S.tables_of(c)
        assert [S.crc(s), S.crc(cn), S.crc(res["path"]), t1[2] + t2[2]] == [int(x) for x in crcs], c["name"]
        assert res["total"] == int(total) and int(res["swapped"]) == int(sw), c["name"]


@need_ref
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_restated_walk_equals_the_reference(name):
    c = next(x for x in CASES if x["name"] == name)
    if S.crafted(c) and not pyoracle.have_ref_set_scores():
        pytest.skip("oracle/_ref/libfamsa_ref.so has no ref_profile_set_scores "
                    "(test_fixture_matches_the_cases covers the case)")
    t1, t2 = S.tables_of(c)
    ref = S.reference_merge(c)
    for mine, theirs in zip((t1, t2), ref["kids"]):
        assert np.array_equal(mine[0], theirs[0]) and np.array_equal(mine[1], theirs[1]) and mine[2] == theirs[2]
    res, s, cn = S.oracle_merge(c, t1, t2)
    assert res["total"] == ref["total"]
    assert np.array_equal(cn, ref["counters"]), S.first_difference(cn, ref["counters"], res["path"])
    assert np.array_equal(s, ref["scores"]), S.first_difference(s, ref["scores"], res["path"])


def _check_np(rt, ct, path, gaps, what):
    want_s, want_c, _, _ = pyoracle.dp_construct(rt, ct, path, gaps)
    got_s, got_c = S.construct_np(rt, ct, path, gaps)
    assert np.array_equal(got_c, want_c), (what, S.first_difference(got_c, want_c, path))
    assert np.array_equal(got_s, want_s), (what, S.first_difference(got_s, want_s, path))


def test_independent_columns_equal_the_walk_on_every_case():
    for c in CASES:
        t1, t2 = S.tables_of(c)
        res = pyoracle.dp_align(t1[0], t1[1], t1[2], t2[0], t2[1], t2[2], c["gaps"])
        rt, ct = (t2, t1) if res["swapped"] else (t1, t2)
        _check_np(rt, ct, res["path"], c["gaps"], c["name"])


def test_go_at_column1_cases():
    for c in S.go_at_column1_cases():
        t1, t2 = S.tables_of(c)
        res = pyoracle.dp_align(t1[0], t1[1], t1[2], t2[0], t2[1], t2[2], c["gaps"])
        assert not res["swapped"] and c["claims"] <= S.case_classes(c, t1, t2, res), c["name"]
        assert (t1 if "R_transfer_col1" in c["claims"] else t2)[1][1, S.GO] > 0
        _check_np(t1, t2, res["path"], c["gaps"], c["name"])


def test_independent_columns_equal_the_walk_on_random_paths():
    """Random gapped children (all-gap columns, cards 1 .. 6) and random monotone paths, with runs longer than a tile
    and paths without a D (W = w1 + w2, which the DP never picks)."""
    rng = np.random.default_rng(4242)
    sm = S.score_matrix()
    seen = set()
    for it in range(3000):
        wr, wc = (int(x) for x in rng.integers(1, 90 if it % 10 == 0 else 30, size=2))
        gaps = tuple(int(x) for x in -rng.integers(1, 20000, size=4))
        tabs = []
        for w in (wr, wc):
            card = int(rng.choice([1, 1, 2, 3, 6]))
            rows = S.random_child(rng, w, card, gap_p=0.0 if card == 1 else float(rng.choice([0.1, 0.3, 0.6])))
            s, c, k = S.profiles.tables_from_rows(rows, sm, gaps)
            if it % 5 == 0:                              # column 1 counts opens, which no rows give (go_at_column1_cases)
                c[1, S.GO], c[1, S.TO] = c[1, S.TO], 0
            tabs.append((s, c, k))
        path = S.random_path(rng, wr, wc)
        if it % 7 == 0:                                  # no D at all
            path = rng.permutation(np.array([1] * wc + [2] * wr, dtype=np.uint8))
        _check_np(tabs[0], tabs[1], path, gaps, f"random path {it}")
        seen |= S.path_classes(path, tabs[0], tabs[1])
        if len(path) == wr + wc:
            seen.add("no_D")
    path_only = {c for c in S.ALL_CLASSES if not c.startswith(("cards", "card_", "rows_at", "width_", "all_24", "swapped",
                                                              "not_swapped", "W1_mod", "W_"))}
    assert path_only <= seen, sorted(path_only - seen)
    assert "no_D" in seen
