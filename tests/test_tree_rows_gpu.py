"""famsa_prof_tree_rows: the final alignment of famsa_prof_align_tree built on the device (FinalizeGaps of every merge,
profile.cpp:1053-1104).  The rows must be exactly what dp_cases.assemble_rows builds on the host from the same paths, the
reference's alignment where a fixture or oracle/_ref has it, and refine(root, rows=None) on them must be today's
host-rows refinement."""
from __future__ import annotations

import ctypes as C
import os
import zlib

import numpy as np
import pytest

import dp_cases
import refine_cases as rc
from conftest import GOLDEN
from famsa_b200 import seqio
from famsa_b200.binding import Engine, FamsaError, _ptr
from oracle import pyoracle

pytestmark = pytest.mark.gpu

GAP = 30
TILE = 512                      # path steps per iteration of k_tree_rows (kTRTile)
E_INVALID, E_STATE = 1, 4


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def _golden_scoring():
    z = np.load(os.path.join(GOLDEN, "adeno_upgma_merges.npz"))
    return z["gaps"], z["score_matrix"]


def _upload(eng, seqs, sm):
    eng.upload(*seqio.pack([seqio.encode(s) for s in seqs]))
    eng.prof_set_scoring(sm)


def _family(n, length, seed):
    codes, off, lens = seqio.synth_family(n, length, seed, sort_desc=False)
    return [seqio.decode(codes[int(o):int(o) + int(l)]) for o, l in zip(off, lens)]


def _as_codes(rows: dict, order) -> np.ndarray:
    return np.stack([rc.to_codes(rows[i]) for i in order])


def check_tree(eng, seqs, merges, gaps=None, sm=None, order=None):
    """align_tree, then tree_rows: equal to assemble_rows on the same paths, every row its sequence, no empty column."""
    g0, sm0 = _golden_scoring()
    gaps = g0 if gaps is None else gaps
    _upload(eng, seqs, sm0 if sm is None else sm)
    root, res, _ = eng.align_tree(merges, gaps)
    n = len(seqs)
    order = list(range(n)) if order is None else list(order)
    got = eng.tree_rows(order)
    want = _as_codes(dp_cases.assemble_rows(seqs, merges, res), order)
    assert got.shape == want.shape == (n, len(res[-1]["path"]))
    assert np.array_equal(got, want), f"rows differ from assemble_rows at {np.argwhere(got != want)[:5].tolist()}"
    for k, leaf in enumerate(order):
        assert np.array_equal(got[k][got[k] != GAP], seqio.encode(seqs[leaf])), f"row {k} is not sequence {leaf}"
    assert (got != GAP).any(axis=0).all(), "a column holds no residue"
    eng.prof_drop([root])
    return got, res


# ---------------------------------------------------------------- the reference's alignments

@pytest.mark.parametrize("fixture", ["hemopexin_sl", "hemopexin_dups"])
def test_hemopexin_rows_crc(eng, fixture):
    """test/hemopexin under the default single-linkage tree, and hemopexin_duplicates: the CRC of the reference's rows."""
    z = np.load(os.path.join(GOLDEN, fixture + ".npz"))
    seqs = [str(s) for s in z["seqs"]]
    merges = [tuple(int(x) for x in m) for m in z["merges"]]
    _upload(eng, seqs, _golden_scoring()[1])
    root, res, _ = eng.align_tree(merges, z["gaps"], want_paths=False)
    rows = eng.tree_rows()
    eng.prof_drop([root])
    text = "\n".join(rc.to_letters(r) for r in rows)
    assert zlib.crc32(text.encode()) == int(z["rows_crc"])


def test_hemopexin_medoid_sl(eng):
    z = np.load(os.path.join(GOLDEN, "hemopexin_medoid_sl.npz"))
    check_tree(eng, [str(s) for s in z["seqs"]], [tuple(int(x) for x in m) for m in z["merges"]], z["gaps"])


def test_adeno_upgma(eng):
    z = np.load(os.path.join(GOLDEN, "adeno_upgma_merges.npz"))
    check_tree(eng, [str(s) for s in z["seqs"]], [tuple(int(x) for x in m) for m in z["merges"]], z["gaps"], z["score_matrix"])


@pytest.mark.skipif(not pyoracle.have("ref", "ref_align_tree_mt"), reason="oracle/_ref not built")
def test_reference_rows(eng):
    """The rows of the reference's own ComputeAlignment (ref_align_tree_mt), its guard column left out."""
    seqs = _family(120, 70, 31)
    merges = dp_cases.random_tree(120, np.random.default_rng(31), caterpillar=0.5)
    dp = pyoracle.RefDp(len(seqs))
    g, sm = dp.gaps(), dp.score_matrix()
    *_, width, ref_rows = dp.align_tree_mt(seqs, merges, 1, want_rows=True)
    dp.close()
    got, _ = check_tree(eng, seqs, merges, g, sm)
    for i in range(len(seqs)):
        r = ref_rows[i]
        r = r[len(r) - got.shape[1]:]                           # without the guard column
        assert rc.to_letters(got[i]) == r.upper(), f"row {i} differs from the reference's"


# ---------------------------------------------------------------- shapes

@pytest.mark.parametrize("cat", [0.0, 0.5, 0.9])
def test_random_trees(eng, cat):
    seqs = _family(300, 80, int(cat * 10) + 40)
    check_tree(eng, seqs, dp_cases.random_tree(300, np.random.default_rng(int(cat * 10)), caterpillar=cat))


def _chain(n, left=True):
    m = [(0, 1)]
    for k in range(2, n):
        m.append((n + k - 2, k) if left else (k, n + k - 2))
    return m


def _balanced(n):
    alive, merges = list(range(n)), []
    while len(alive) > 1:
        nxt = []
        for a in range(0, len(alive) - 1, 2):
            merges.append((alive[a], alive[a + 1]))
            nxt.append(n + len(merges) - 1)
        if len(alive) % 2:
            nxt.append(alive[-1])
        alive = nxt
    return merges


@pytest.mark.parametrize("shape", ["left_chain", "right_chain", "balanced"])
def test_chains_and_balanced(eng, shape):
    n = 150
    seqs = _family(n, 60, 7)
    merges = {"left_chain": _chain(n, True), "right_chain": _chain(n, False), "balanced": _balanced(n)}[shape]
    check_tree(eng, seqs, merges)


@pytest.mark.parametrize("n", [2, 3])
def test_smallest_trees(eng, n):
    seqs = _family(n, 50, 3)
    check_tree(eng, seqs, [(0, 1)] if n == 2 else [(0, 1), (2, 3)])
    if n == 3:
        check_tree(eng, seqs, [(1, 2), (3, 0)])


def test_length_one_sequence(eng):
    seqs = _family(20, 40, 9)
    seqs[5] = "W"
    seqs[11] = seqs[11][:1]
    check_tree(eng, seqs, dp_cases.random_tree(20, np.random.default_rng(9), caterpillar=0.5))


def test_all_d_merge(eng):
    """Identical sequences: every path is one run of D steps."""
    s = _family(1, 90, 2)[0]
    got, res = check_tree(eng, [s] * 5, [(0, 1), (2, 5), (3, 4), (6, 7)])
    assert all(not r["path"].any() for r in res)
    assert (got != GAP).all()


@pytest.mark.parametrize("width", [TILE - 1, TILE, TILE + 1])
def test_root_width_at_the_tile(eng, width):
    """W_root (and every path) at the kernel's tile size - 1, tile size, + 1; a gapped family of that length too."""
    s = _family(1, width, 5)[0][:width].ljust(width, "A")
    got, res = check_tree(eng, [s] * 4, _balanced(4))
    assert got.shape[1] == width
    fam = _family(40, width - 40, width)
    check_tree(eng, fam, dp_cases.random_tree(40, np.random.default_rng(width), caterpillar=0.5))


def test_deep_chain_wraps_the_grid(eng):
    """A chain of 3000 merges: every merge waits on the one before it, and the ticket passes the resident grid
    (132 SMs x 4 blocks on an H100) several times."""
    n = 3001
    seqs = _family(n, 18, 13)
    check_tree(eng, seqs, _chain(n, True))


# ---------------------------------------------------------------- order and state

def test_orders(eng):
    seqs = _family(60, 50, 21)
    merges = dp_cases.random_tree(60, np.random.default_rng(21), caterpillar=0.3)
    ids = [f"seq{(i * 37) % 101}" for i in range(60)]
    for order in (list(range(60)), list(range(59, -1, -1)), rc.id_order(ids)):
        check_tree(eng, seqs, merges, order=order)


def _raw(eng, order, n, buf, cap):
    w = C.c_uint32()
    o = None if order is None else np.ascontiguousarray(order, dtype=np.uint32)
    return eng.lib.famsa_prof_tree_rows(eng.h, _ptr(o), n, None if buf is None else _ptr(buf), cap, C.byref(w)), w.value


def test_errors_and_state(eng):
    g, sm = _golden_scoring()
    seqs = _family(12, 40, 2)
    merges = dp_cases.random_tree(12, np.random.default_rng(2))
    fresh = Engine(0)
    assert _raw(fresh, None, 12, None, 0)[0] == E_STATE                     # no tree yet
    fresh.close()
    _upload(eng, seqs, sm)
    root, res, _ = eng.align_tree(merges, g)
    W = len(res[-1]["path"])
    stats = eng.prof_stats()
    buf = np.zeros(12 * W, dtype=np.uint8)
    assert _raw(eng, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10], 12, buf, buf.size)[0] == E_INVALID   # duplicate
    assert _raw(eng, list(range(11)) + [12], 12, buf, buf.size)[0] == E_INVALID                  # out of range
    assert _raw(eng, None, 12, buf, buf.size - 1)[0] == E_INVALID                                  # cap one byte short
    assert _raw(eng, None, 11, buf, buf.size)[0] == E_INVALID                                      # n_rows
    assert eng.lib.famsa_prof_tree_rows(eng.h, None, 12, None, 0, None) == E_INVALID               # width_out
    rc0, w = _raw(eng, None, 12, buf, buf.size)
    assert rc0 == 0 and w == W
    first = buf.copy()
    assert _raw(eng, None, 12, buf, buf.size)[0] == 0 and np.array_equal(buf, first)             # two calls, same bytes
    assert eng.prof_stats() == stats                                                               # nothing resident added
    assert np.array_equal(first.reshape(12, W), _as_codes(dp_cases.assemble_rows(seqs, merges, res), range(12)))
    eng.prof_drop([root])
    # a re-upload after the tree
    _upload(eng, seqs, sm)
    assert _raw(eng, None, 12, buf, buf.size)[0] == E_STATE
    # a failed tree call, after a good one
    root, res, _ = eng.align_tree(merges, g)
    eng.prof_drop([root])
    with pytest.raises(FamsaError):
        eng.align_tree([(0, 1)] * 11, g)
    assert _raw(eng, None, 12, buf, buf.size)[0] == E_STATE
    assert eng.prof_stats() == (0, 0)
    check_tree(eng, seqs, merges)                                                                  # still usable


def test_binding_sizes_rows_from_the_latest_tree(eng):
    """Engine.tree_rows sizes its rows from the tree that was run last, also by align_tree_buffers or behind the
    binding's back through the C call."""
    g, sm = _golden_scoring()
    seqs = _family(30, 50, 6)
    _upload(eng, seqs, sm)
    chain, bal = _chain(30, True), _balanced(30)
    root, res, _ = eng.align_tree(chain, g)
    eng.prof_drop([root])
    b = eng.align_tree_buffers(bal, g, None)                        # runs (and drops) the balanced tree
    root2, res2, _ = eng.align_tree(bal, g)
    eng.prof_drop([root2])
    rows = eng.tree_rows()
    assert rows.shape == (30, len(res2[-1]["path"]))
    for other in (chain, bal):                                      # a tree run through the C ABI directly
        t = np.ascontiguousarray(other, dtype=np.int32)
        r, nb, st = C.c_uint32(), C.c_uint64(), b["res"]
        assert eng.lib.famsa_prof_align_tree(eng.h, _ptr(t), 30, _ptr(b["gaps"]), C.byref(st), C.byref(r), C.byref(nb), None) == 0
        eng.prof_drop([r.value])
        want = int(st[28].path_len)
        rows = eng.tree_rows()
        assert rows.shape == (30, want)
        for i in range(30):
            assert np.array_equal(rows[i][rows[i] != GAP], seqio.encode(seqs[i]))


# ---------------------------------------------------------------- refinement from the kept rows

def _refine_both(eng, seqs, merges, g, sm, ids, n_refinements=100):
    """Today's host-rows path and the kept-rows path on the same tree: (rows, width, total, stats) of each."""
    order = rc.id_order(ids)
    out = []
    for kept in (False, True):
        _upload(eng, seqs, sm)
        root, res, _ = eng.align_tree(merges, g)
        if kept:
            eng.tree_rows(order, download=False)
            rows, width, total, stats, rid = eng.refine(root, None, g, n_refinements)
        else:
            arr = _as_codes(dp_cases.assemble_rows(seqs, merges, res), order)
            rows, width, total, stats, rid = eng.refine(root, arr, g, n_refinements)
        eng.prof_drop([rid])
        out.append((rows, width, total, stats))
    (r0, w0, t0, s0), (r1, w1, t1, s1) = out
    assert w1 == w0 and t1 == t0 and np.array_equal(r1, r0)
    for k in ("n_tries", "n_realigned", "n_accepted", "n_identical", "cells"):
        assert s1[k] == s0[k], k
    return r1, w1, order


@pytest.mark.parametrize("n", [2, 5, 100, 300])
def test_refine_families(eng, n):
    seqs = rc.family(n, 60, seed=n)
    g, sm = _golden_scoring()
    _refine_both(eng, seqs, dp_cases.random_tree(n, np.random.default_rng(n)), g, sm, [f"s{i}" for i in range(n)])


@pytest.mark.parametrize("name", ["upgma", "sl"])
def test_refine_adeno(eng, name):
    """FAMSA's own refined adeno_fiber alignments (adeno_refined.npz) from the kept rows."""
    z = np.load(os.path.join(GOLDEN, "adeno_refined.npz"))
    t = np.load(os.path.join(GOLDEN, "adeno_upgma_merges.npz"))
    g, sm = t["gaps"], t["score_matrix"]
    if name == "upgma":
        seqs, merges = [str(s) for s in t["seqs"]], t["merges"]
    else:
        t = np.load(os.path.join(GOLDEN, "adeno_sl_tree.npz"))
        seqs, merges = [str(s) for s in t["seqs"]], t["tree"][len(t["seqs"]):]
    ids = [str(i) for i in z[f"{name}_ids"]]
    rows, width, order = _refine_both(eng, seqs, merges, g, sm, ids)
    gold = z[f"{name}_rows"]
    assert width == gold.shape[1]
    assert all(np.array_equal(rows[k], gold[i]) for k, i in enumerate(order))


def test_refine_kept_rows_errors(eng):
    g, sm = _golden_scoring()
    seqs = _family(10, 40, 4)
    merges = dp_cases.random_tree(10, np.random.default_rng(4))
    _upload(eng, seqs, sm)
    root, res, _ = eng.align_tree(merges, g)
    W = len(res[-1]["path"])
    eng.tree_rows(download=False)
    r = (C.c_uint32(), C.c_uint32(), C.c_int64())
    gp = np.ascontiguousarray(g, dtype=np.int64)

    def call(root_id, n, w, rows=None):
        return eng.lib.famsa_prof_refine(eng.h, root_id, rows, n, w, _ptr(gp), 10, 4, *(C.byref(x) for x in r), None)
    assert call(root + 1000, 10, W) == E_INVALID                    # not the tree's root
    assert call(root, 9, W) == E_INVALID                            # n_rows
    assert call(root, 10, W + 1) == E_INVALID                       # width
    assert call(root, 10, W, C.c_void_p(1)) == E_INVALID            # rows given with the flag
    assert eng.prof_get(root, tables=False) == (W, 10)              # the root is still resident
    rows, width, total, stats, rid = eng.refine(root, None, g, 10)  # and the kept rows still serve
    eng.prof_drop([rid])
    # the kept rows name their root: a new tree's root does not take them
    root2, _, _ = eng.align_tree(merges, g)
    assert call(root2, 10, W) == E_INVALID
    eng.prof_drop([root2])
    assert eng.prof_stats() == (0, 0)
