"""CPU tests of the progressive-alignment scheduling policy (famsa_b200/csrc/tree_plan.h), compiled alone with g++ into
tests/cpp/tree_plan_check.cpp.

famsa_prof_align_tree builds its dependency levels with tree_levels: they must be famsa_b200.schedule.ready_levels on
every committed tree and on random ones, and a malformed tree must be rejected at the node the check names.  The
named limits keep their values, and every predicate flips exactly one past its limit."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
from cpp_build import build_cpp
from dp_cases import random_tree
from famsa_b200.schedule import ready_levels

# the dependency levels of the fixtures test_tree_gpu.py aligns
FIXTURE_LEVELS = {"hemopexin_sl": 451, "hemopexin_medoid_sl": 94, "hemopexin_dups": 103, "adeno_upgma_merges": 22}
# other committed guide trees in tree_structure order: (fixture, key)
TREES = [("adeno_slink_tree", "tree"), ("adeno_nj_tree", "tree0"), ("adeno_nj_tree", "tree1"), ("hemopexin_nj", "tree0"),
         ("hemopexin_nj", "tree1")]


@pytest.fixture(scope="module")
def check(tmp_path_factory):
    exe = build_cpp("tree_plan_check", tmp_path_factory.mktemp("tree_plan"))

    def run(*args, stdin="", fused=None):
        env = {k: v for k, v in os.environ.items() if k != "FAMSA_PROF_FUSED"}
        if fused is not None:
            env["FAMSA_PROF_FUSED"] = fused
        return subprocess.run([exe] + [str(a) for a in args], input=stdin, env=env, capture_output=True, text=True,
                              check=True).stdout
    return run


def tree_levels(check, n_leaves, merges):
    """tree_levels on the tree: its levels, or the node it rejects."""
    out = check("levels", stdin="%d\n" % n_leaves + "".join("%d %d\n" % (a, b) for a, b in merges)).splitlines()
    if out and out[0].startswith("bad "):
        return int(out[0].split()[1])
    return [[int(k) for k in line.split()] for line in out]


def first_invalid(n_leaves, merges):
    """The first node famsa_prof_align_tree names in "node N has invalid children": a child that is negative, not
    yet made, the other child, or already used."""
    used = set()
    for k, (a, b) in enumerate(merges):
        if a < 0 or b < 0 or a >= n_leaves + k or b >= n_leaves + k or a == b or a in used or b in used:
            return n_leaves + k
        used |= {a, b}
    return None


def merges_of(z, key):
    return [(int(a), int(b)) for a, b in z[key]]


@pytest.mark.parametrize("fixture", sorted(FIXTURE_LEVELS))
def test_levels_fixtures(check, fixture):
    merges = merges_of(np.load(os.path.join(GOLDEN, fixture + ".npz")), "merges")
    levels = tree_levels(check, len(merges) + 1, merges)
    assert levels == ready_levels(len(merges) + 1, merges)
    assert len(levels) == FIXTURE_LEVELS[fixture]


@pytest.mark.parametrize("fixture,key", TREES)
def test_levels_guide_trees(check, fixture, key):
    merges = merges_of(np.load(os.path.join(GOLDEN, fixture + ".npz")), key)
    assert tree_levels(check, len(merges) + 1, merges) == ready_levels(len(merges) + 1, merges)


@pytest.mark.parametrize("seed,n,caterpillar", [(1, 2, 0.0), (2, 3, 0.5), (3, 50, 0.0), (4, 300, 0.3), (5, 700, 0.95), (6, 128, 1.0)])
def test_levels_random(check, seed, n, caterpillar):
    merges = random_tree(n, np.random.default_rng(seed), caterpillar)
    assert first_invalid(n, merges) is None
    assert tree_levels(check, n, merges) == ready_levels(n, merges)


# (n_leaves, merges, the node rejected)
INVALID = [
    (6, [(0, 1), (2, 3), (4, 5), (6, 6), (8, 9)], 9),                 # test_tree_gpu.py::test_tree_errors: self-merge
    (6, [(0, 1), (2, 3), (4, 5), (6, 9), (7, 8)], 9),                 # test_tree_errors: a child that comes later
    (6, [(0, 0), (1, 2), (3, 4), (5, 6), (7, 8)], 6),                 # self-merge of a leaf
    (6, [(0, 1), (0, 2), (3, 4), (5, 6), (7, 8)], 7),                 # a leaf used twice
    (6, [(0, 1), (2, 3), (6, 4), (6, 5), (8, 9)], 9),                 # a merged profile used twice
    (6, [(0, 1), (2, 7), (3, 4), (5, 6), (8, 9)], 7),                 # the node itself as its child
    (6, [(0, 1), (2, 8), (3, 4), (5, 6), (7, 9)], 7),                 # a forward reference
    (6, [(0, 1), (2, 3), (4, 5), (6, 7), (8, 11)], 10),               # beyond the last node
    (6, [(0, 1), (-1, 2), (3, 4), (5, 6), (7, 8)], 7),                # a negative id
    (6, [(0, 1), (2, 3), (4, -2**31), (5, 6), (7, 8)], 8),
    (6, [(0, 1), (1, 2), (3, 3), (4, 5), (7, 8)], 7),                 # two faults: the first one counts
]


@pytest.mark.parametrize("n_leaves,merges,node", INVALID)
def test_invalid_trees(check, n_leaves, merges, node):
    assert first_invalid(n_leaves, merges) == node
    assert tree_levels(check, n_leaves, merges) == node


def test_invalid_random(check):
    """One child of a random tree replaced by a random id: rejected exactly where the check names it."""
    rng = np.random.default_rng(7)
    n_rejected = 0
    for _ in range(60):
        n = int(rng.integers(2, 40))
        merges = [list(m) for m in random_tree(n, rng, 0.3)]
        merges[int(rng.integers(n - 1))][int(rng.integers(2))] = int(rng.integers(-3, 2 * n + 2))
        merges = [tuple(m) for m in merges]
        want = first_invalid(n, merges)
        n_rejected += want is not None
        assert tree_levels(check, n, merges) == (ready_levels(n, merges) if want is None else want)
    assert n_rejected > 30


def test_leaf_count_mismatch_is_a_tree(check):
    """test_tree_errors' first call announces 3 leaves with 6 uploaded: famsa_prof_align_tree rejects it for the count
    before it builds levels, and as a tree of 3 leaves it is valid."""
    assert tree_levels(check, 3, [(0, 1), (2, 3)]) == [[0], [1]]


def test_limits(check):
    got = dict(line.split() for line in check("limits").splitlines())
    assert {k: int(v) for k, v in got.items()} == {
        "max_in_flight": 8, "max_fused_uncollected": 2, "max_fused_levels": 32, "max_fused_jobs": 8192,
        "drift_slack": 1024, "heavy_cells": 64 << 20, "fused_max_jobs": 4096, "fused_max_host_rows": 512,
        "fused_max_width": 8192}


def eligible(check, batch, fused=None):
    return check("eligible", stdin="".join("%d %d %d %d\n" % m for m in batch), fused=fused) == "1\n"


@pytest.mark.parametrize("fused,allowed", [(None, True), ("1", True), ("0", False), ("7", True)])
def test_fused_eligible(check, fused, allowed):
    small = (40, 1, 300, 6)
    assert eligible(check, [small] * 4096, fused) == allowed
    assert not eligible(check, [small] * 4097, fused)
    # rows as the host sees them: a sequence side gives its width, two profiles the narrower one
    assert eligible(check, [small, (512, 1, 600, 3)], fused) == allowed
    assert not eligible(check, [small, (513, 1, 600, 3)], fused)
    assert eligible(check, [(600, 3, 512, 1)], fused) == allowed
    assert not eligible(check, [(600, 3, 513, 1)], fused)
    assert eligible(check, [(512, 2, 700, 9)], fused) == allowed
    assert not eligible(check, [(513, 2, 700, 9)], fused)
    # the wider child, whatever the rows
    assert eligible(check, [(8192, 4, 100, 4), small], fused) == allowed
    assert not eligible(check, [(8193, 4, 100, 4), small], fused)
    assert eligible(check, [(100, 4, 8192, 4)], fused) == allowed
    assert not eligible(check, [(100, 4, 8193, 4)], fused)


def test_fused_joins(check):
    def joins(levels, acc_jobs, level_jobs):
        return check("joins", levels, acc_jobs, level_jobs) == "1\n"
    assert joins(0, 0, 8192) and not joins(0, 0, 8193)
    assert joins(31, 8000, 192) and not joins(31, 8000, 193)
    assert joins(31, 1, 1) and not joins(32, 1, 1)


def test_drift(check):
    def drifted(bound, max_exact):
        return check("drifted", bound, max_exact) == "1\n"
    for max_exact in (0, 1, 350, 6668):
        limit = 1024 + 2 * max_exact
        assert not drifted(limit, max_exact) and drifted(limit + 1, max_exact)


def test_level_keep(check):
    """Before a level that goes launch by launch: drain everything when a child pends and the level is heavy, or when its
    paths do not fit the arena (even with nothing in flight: the arena grows then); otherwise keep at most 7 of 8."""
    def keep(pending, cells, path_end, path_cap, in_flight):
        return int(check("keep", int(pending), cells, path_end, path_cap, in_flight))
    heavy = 64 << 20
    for n in (0, 3, 8, 9):
        full = 7 if n >= 8 else -1
        assert keep(True, heavy, 10, 10, n) == full and keep(True, heavy + 1, 10, 10, n) == 0
        assert keep(False, heavy + 1, 10, 10, n) == full              # bounds of finished children are exact
        assert keep(False, 0, 1000, 1000, n) == full and keep(False, 0, 1001, 1000, n) == 0
    assert keep(False, 0, 0, 1, 7) == -1 and keep(False, 0, 0, 1, 8) == 7
