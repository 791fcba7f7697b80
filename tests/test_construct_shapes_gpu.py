"""construct_tile on the device at its tile, gap-run, orientation and card edges (cases: tests/construct_shapes.py), through
famsa_prof_merge_batch in both kernels that run it:

* k_prof_construct (FAMSA_PROF_FUSED=0): every case alone, and mixed batches of 1-tile jobs next to jobs of very different
  tile counts, so that the blocks' binary search over tile0 meets every job boundary;
* k_merge_fused (default settings) for the cases it takes, with the launch count of the call showing that it ran;
* align_tree on a chain of near-identical sequences (queued bounds twice the real widths) and on a caterpillar whose
  levels run in one fused launch.

Path, total, orientation and the merged tables are compared bit for bit with the reference (the fixture's CRC32s of its
tables, and the live reference where oracle/_ref is built) and with the C restatement of its walk (dp_construct); a
mismatch names the first differing (column, lane) and what that column is."""
from __future__ import annotations

import numpy as np
import pytest

import construct_shapes as S
import dp_cases
from famsa_b200 import seqio
from famsa_b200.binding import PROF_LEAF
from oracle import pyoracle

pytestmark = pytest.mark.gpu
CASES = {c["name"]: c for c in S.cases()}
FIX = np.load(S.FIXTURE)
WANT = {str(n): (tuple(int(x) for x in crcs), int(t), bool(sw))
        for n, crcs, t, sw in zip(FIX["names"], FIX["crcs"], FIX["totals"], FIX["swapped"])}
DEFAULT_GAPS = CASES["leaves_all_letters"]["gaps"]


@pytest.fixture(scope="module")
def eng():
    import famsa_b200
    e = famsa_b200.Engine(0)
    yield e
    e.close()


def merge_on_device(eng, jobs, gaps):
    """jobs: list of (child a, child b) as construct_shapes writes them; one famsa_prof_merge_batch with `gaps`.
    Returns ([(result, scores, counters, card)], kernel launches of the call)."""
    leaves = [ch[1] for a, b in jobs for ch in (a, b) if ch[0] == "leaf"]
    if leaves:
        eng.upload(*seqio.pack([seqio.encode(x) for x in leaves]))
    eng.prof_set_scoring(S.score_matrix())
    merges, widths, n_leaf = [], [], 0
    for a, b in jobs:
        ids, ws = [], []
        for ch in (a, b):
            if ch[0] == "leaf":
                ids.append(PROF_LEAF | n_leaf)
                n_leaf += 1
                ws.append(len(ch[1]))
            else:
                t = S.child_tables(ch, gaps)
                ids.append(eng.prof_put([t])[0])
                ws.append(t[0].shape[0] - 1)
        merges.append(tuple(ids))
        widths.append(tuple(ws))
    l0 = eng.kernel_launches()
    mids, res = eng.prof_merge_batch(merges, np.asarray(gaps, dtype=np.int64), widths)
    launches = eng.kernel_launches() - l0
    out = []
    for mid, r in zip(mids, res):
        s, c, k = eng.prof_get(mid)
        out.append((r, s, c, k))
    eng.prof_drop(mids)
    assert eng.prof_stats() == (0, 0)
    return out, launches


def check(name, got, case=None):
    """One merge's outcome against the restatement and the reference (fixture CRCs; live where built)."""
    r, s, c, k = got
    case = CASES[name] if case is None else case
    want_r, want_s, want_c = S.oracle_merge(case)
    assert np.array_equal(r["path"], want_r["path"]), f"{name}: path differs from the restatement's"
    assert r["total"] == want_r["total"] and r["swapped"] == want_r["swapped"], name
    assert np.array_equal(c, want_c), f"{name}: counters, first difference (column, lane, class) {S.first_difference(c, want_c, r['path'])}"
    assert np.array_equal(s, want_s), f"{name}: scores, first difference (column, lane, class) {S.first_difference(s, want_s, r['path'])}"
    if name in WANT:
        crcs, total, sw = WANT[name]
        assert (S.crc(s), S.crc(c), S.crc(r["path"]), k) == crcs and r["total"] == total and r["swapped"] == sw, \
            f"{name}: differs from the reference's recorded merge"


def fused_names():
    out = []
    for name, c in CASES.items():
        t1, t2 = S.tables_of(c)
        if S.fused_eligible(t1, t2):
            out.append(name)
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_batch_kernel(eng, monkeypatch, name):
    monkeypatch.setenv("FAMSA_PROF_FUSED", "0")
    c = CASES[name]
    (got,), launches = merge_on_device(eng, [(c["a"], c["b"])], c["gaps"])
    assert launches >= 2, "the batch path runs the DP and k_prof_construct"
    check(name, got)


@pytest.mark.parametrize("name", fused_names())
def test_fused_kernel(eng, monkeypatch, name):
    monkeypatch.delenv("FAMSA_PROF_FUSED", raising=False)
    c = CASES[name]
    (got,), launches = merge_on_device(eng, [(c["a"], c["b"])], c["gaps"])
    assert launches == 1, f"{launches} launches: the merge did not run whole in k_merge_fused"
    check(name, got)


@pytest.mark.parametrize("fused", ["0", "1"])
def test_go_at_column1(eng, monkeypatch, fused):
    """Uploaded tables with a gap open in column 1: the consumed column takes no open transfer (the reference's walk)."""
    monkeypatch.setenv("FAMSA_PROF_FUSED", fused)
    for c in S.go_at_column1_cases():
        (got,), launches = merge_on_device(eng, [(c["a"], c["b"])], c["gaps"])
        assert (launches == 1) == (fused == "1")
        check(c["name"], got, c)


def test_fused_takes_the_cases_it_should():
    names = set(fused_names())
    assert {"profiles_at_fused_row_limit", "rows_65536", "forced_alternating"} <= names
    assert "wide_8300" not in names


def _tiny_jobs(rng, n):
    """Leaf pairs whose merges are one tile (w1 + w2 + 1 <= 64), with an insertion or a deletion."""
    out = []
    for a in range(n):
        base = "".join(S.LETTERS[x] for x in rng.integers(0, 20, size=int(rng.integers(3, 28))))
        p = int(rng.integers(0, len(base)))
        other = base[:p] + "W" + base[p:] if a % 2 else base[:p] + base[p + 1:] or "A"
        out.append(dict(name=f"tiny{a}", a=("leaf", base), b=("leaf", other), gaps=DEFAULT_GAPS, claims=set()))
    return out


@pytest.mark.parametrize("order", ["tiny_between", "tiny_first", "reversed"])
def test_mixed_batch_through_the_tile_search(eng, monkeypatch, order):
    """All cases with the default gap costs in one launch of k_prof_construct, 1-tile jobs next to each other and next to
    jobs of up to 130 tiles."""
    monkeypatch.setenv("FAMSA_PROF_FUSED", "0")
    rng = np.random.default_rng(len(order))
    big = [c for c in CASES.values() if tuple(c["gaps"]) == tuple(DEFAULT_GAPS)]
    tiny = _tiny_jobs(rng, 3 * len(big))
    if order == "tiny_between":
        jobs = [x for k, c in enumerate(big) for x in [c] + tiny[3 * k:3 * k + 3]]
    elif order == "tiny_first":
        jobs = tiny + big
    else:
        jobs = (big + tiny)[::-1]
    tiles = [(S.tables_of(c)[0][0].shape[0] + S.tables_of(c)[1][0].shape[0] - 2 + S.TILE) // S.TILE for c in jobs]
    assert 1 in tiles and max(tiles) > 100
    assert any(a == b == 1 for a, b in zip(tiles, tiles[1:]))
    got, _ = merge_on_device(eng, [(c["a"], c["b"]) for c in jobs], DEFAULT_GAPS)
    for c, g in zip(jobs, got):
        check(c["name"], g, c)


@pytest.mark.parametrize("fused", ["0", "1"])
@pytest.mark.parametrize("tree", [t["name"] for t in S.tree_cases()])
def test_tree_root_equals_the_reference(eng, monkeypatch, tree, fused):
    monkeypatch.setenv("FAMSA_PROF_FUSED", fused)
    t = next(x for x in S.tree_cases() if x["name"] == tree)
    g = FIX[f"tree_{tree}_gaps"]
    eng.upload(*seqio.pack([seqio.encode(x) for x in t["seqs"]]))
    eng.prof_set_scoring(S.score_matrix())
    root, res, stats = eng.align_tree(t["merges"], g)
    s, c, k = eng.prof_get(root)
    eng.prof_drop([root])
    assert [r["total"] for r in res] == [int(x) for x in FIX[f"tree_{tree}_totals"]]
    assert (S.crc(s), S.crc(c), k) == tuple(int(x) for x in FIX[f"tree_{tree}_root"]), "root tables differ from the reference's"
    if fused == "1":
        assert stats["n_batches"] < len(t["merges"]), "no level of the tree joined a fused launch"
    if pyoracle.have_ref():
        g_ref, recs = dp_cases.reference_merges(t["seqs"], t["merges"], threads=(1,), want_merged=True)
        assert np.array_equal(g_ref, g)
        ws, wc, wk = recs[-1]["merged"]
        assert np.array_equal(s, ws) and np.array_equal(c, wc) and k == wk
    if tree == "chain_identical":
        assert max(r["cols_width"] + r["rows_width"] - len(r["path"]) for r in res) > 100, \
            "no merge whose bound w1 + w2 is far above its real width"
