"""The cooperative guide-tree kernels where a thread owns more than one sequence, and the distance triangles past 2^32
elements.

FAMSA_TREE_MAX_BLOCKS=<cap> shrinks the grids of k_prim, k_upgma and k_nj to `cap` blocks, so the sizes of
tree_coop_cases.sizes(cap) run the loop over a thread's second and later sequences (st[], visited[], the owner block of
a visited vertex) that otherwise only sets above ~135 k sequences reach.  Every capped run is compared with an
independent restatement and, bit for bit, with the uncapped call; its `[coop]` line (FAMSA_TREE_DEBUG) shows the grid it
ran on.  The restatements: tree_coop_cases.prim_vectorised (MSTPrim's loop), mst.kruskal_total_order + prim_replay and
mst.slink_tree (the unique MST), upgma_oracle.c (computeTree), nj_oracle.c (NJ's computeTree), each on the oracle's LCS
triangle for small sets and on the device's own triangle (checked by test_lcs_gpu.py) for large ones.

Past 2^32: UPGMA on a planted u16 triangle of 93 000 rows built on the device, and the Boruvka rounds and SLINK on
synth_family(93 000, 60) against the sequential loop.  Each skips when the device has too little free memory."""
import ctypes as C
import functools
import os
import re

import numpy as np
import pytest
import torch

import famsa_b200
from conftest import GOLDEN
from famsa_b200 import mst, seqio
from oracle import pyoracle as P
import tree_coop_cases as T
import upgma_cases as U
from test_nj_gpu import boundary_set, check_against_restatement
from test_upgma_gpu import device_triangle, tree_from_triangle, upload_lens

pytestmark = pytest.mark.gpu

SMALL = 3000                    # above this many sequences the restatements read the device's own triangle


def coop_lines(text):
    return [(k, int(n), int(b)) for k, n, b in re.findall(r"\[coop\] (\S+) n=(\d+) blocks=(\d+)", text)]


def set_cap(monkeypatch, cap):
    monkeypatch.setenv("FAMSA_TREE_DEBUG", "1")
    if cap:
        monkeypatch.setenv("FAMSA_TREE_MAX_BLOCKS", str(cap))
    else:
        monkeypatch.delenv("FAMSA_TREE_MAX_BLOCKS", raising=False)


def assert_capped(capfd, kernel, n, cap):
    """The call just made ran `kernel` once, on `cap` blocks, with every thread of the grid owning a sequence and, past
    exact fit, some owning a second one."""
    lines = coop_lines(capfd.readouterr().err)
    assert lines == [(kernel, n, cap)], lines
    assert n >= T.COOP_THREADS * cap


@functools.lru_cache(maxsize=None)
def sequence_set(name, n, cap):
    return T.sequence_set(name, n, cap)


def lcs_triangle(engine, codes, offsets, lens, dtype=np.uint32):
    """The LCS triangle (row = seq0) of the uploaded set: the oracle's for small sets, the device's for large ones."""
    if len(lens) <= SMALL:
        return P.lcs_triangle(codes, offsets, lens).astype(dtype)
    return engine.triangle(dtype=dtype)


_prim_cache = {}


def restated_prim(engine, name, n, cap, kind):
    key = (name, n, cap, kind)
    if key not in _prim_cache:
        codes, offsets, lens, exact = sequence_set(name, n, cap)
        rows = T.LcsRows(lcs_triangle(engine, codes, offsets, lens), codes, offsets, lens, exact)
        _prim_cache[key] = T.prim_vectorised(rows, lens, kind)
    return _prim_cache[key]


def same(got, want, what):
    for g, w in zip(got, want):
        assert np.array_equal(g, w), what


@pytest.mark.parametrize("cap,n,name", T.CASES, ids=[f"{s}-{n}-cap{c}" for c, n, s in T.CASES])
def test_prim(engine, monkeypatch, capfd, cap, n, name):
    """famsa_lcs_prim: the sequential loop k_prim<false> on `cap` blocks and uncapped, and (sets without flagged
    sequences) the Boruvka rounds, all against the vectorised restatement; at the smallest sizes also the Kruskal MST."""
    codes, offsets, lens, exact = sequence_set(name, n, cap)
    engine.upload(codes, offsets, lens)
    for kind in (0, 1):
        want = restated_prim(engine, name, n, cap, kind)
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
        set_cap(monkeypatch, cap)
        capfd.readouterr()
        got = engine.prim(kind)
        assert_capped(capfd, "k_prim<0>", n, cap)
        same(got, want, f"capped, kind {kind}")
        set_cap(monkeypatch, 0)
        same(engine.prim(kind), got, f"uncapped, kind {kind}")
        monkeypatch.delenv("FAMSA_PRIM_SEQUENTIAL")
        capfd.readouterr()
        got = engine.prim(kind)
        lines = coop_lines(capfd.readouterr().err)
        if exact:                               # flagged sequences: the sequential loop, uncapped
            assert [k for k, _, _ in lines] == ["k_prim<0>"]
            same(got, want, f"default engine, kind {kind}")
            continue
        assert lines == [], "the Boruvka rounds did not run"
        same(got, want, f"Boruvka, kind {kind}")
        if n <= 1025:
            tri = lcs_triangle(engine, codes, offsets, lens)
            same(got, mst.prim_replay(n, mst.kruskal_total_order(n, T.distance_triangle_f64(kind, tri, lens))),
                 f"Kruskal, kind {kind}")


@pytest.mark.parametrize("cap,n,name", T.CASES, ids=[f"{s}-{n}-cap{c}" for c, n, s in T.CASES])
def test_slink(engine, monkeypatch, capfd, cap, n, name):
    """famsa_lcs_slink: the sequential loop k_prim<true> on `cap` blocks against the uncapped Boruvka tree (pinned to the
    reference by test_slink_gpu.py) and, for sets without flagged sequences, against mst.slink_tree of the restated MST."""
    codes, offsets, lens, exact = sequence_set(name, n, cap)
    engine.upload(codes, offsets, lens)
    for kind in (0, 1):
        set_cap(monkeypatch, 0)
        capfd.readouterr()
        boruvka = engine.slink(kind)
        assert coop_lines(capfd.readouterr().err) == [], "the Boruvka rounds did not run"
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
        set_cap(monkeypatch, cap)
        got = engine.slink(kind)
        assert_capped(capfd, "k_prim<1>", n, cap)
        monkeypatch.delenv("FAMSA_PRIM_SEQUENTIAL")
        assert np.array_equal(got, boruvka), f"kind {kind}"
        if not exact:
            ef, et, ed, _ = restated_prim(engine, name, n, cap, kind)
            assert np.array_equal(got, mst.slink_tree(n, list(zip(ef.tolist(), et.tolist(), ed.tolist())))), f"kind {kind}"


@pytest.mark.parametrize("cap,n,name", T.CASES, ids=[f"{s}-{n}-cap{c}" for c, n, s in T.CASES])
def test_upgma(engine, monkeypatch, capfd, cap, n, name):
    """famsa_lcs_upgma and _from_triangle at 2 and 4 bytes, both averaging rules, on `cap` blocks: the restated
    computeTree and the uncapped call."""
    codes, offsets, lens, _ = sequence_set(name, n, cap)
    engine.upload(codes, offsets, lens)
    lcs = lcs_triangle(engine, codes, offsets, lens)
    for modified in (False, True):
        kinds = (0, 1) if modified else (0,)
        for kind in kinds:
            want = U.expected_tree(kind, modified, lcs, lens)
            set_cap(monkeypatch, cap)
            capfd.readouterr()
            got = engine.upgma(kind, modified)
            assert_capped(capfd, f"k_upgma<{int(modified)}>", n, cap)
            assert np.array_equal(got, want), (kind, modified)
            set_cap(monkeypatch, 0)
            assert np.array_equal(engine.upgma(kind, modified), got), (kind, modified, "uncapped")
        set_cap(monkeypatch, cap)
        want = U.expected_tree(0, modified, lcs, lens)
        for eb in (2, 4):
            t = torch.empty(n * (n - 1) // 2, dtype=torch.int16 if eb == 2 else torch.int32, device="cuda")
            engine.triangle_device(0, n, t.data_ptr(), eb)
            assert np.array_equal(tree_from_triangle(engine, 0, modified, t), want), (modified, eb)
            del t
    capfd.readouterr()


@pytest.mark.parametrize("cap,n,case", T.CRAFT_CASES, ids=[f"{c}-{n}-cap{k}" for k, n, c in T.CRAFT_CASES])
def test_upgma_crafted(engine, monkeypatch, capfd, cap, n, case):
    """Crafted triangles through _from_triangle at 2 and 4 bytes, both rules, on `cap` blocks: equal minima in a thread's
    first and second row, a stale cache relabelled on a row a thread owns second, the unique minimum in the last row."""
    lcs, lens = T.craft_coop(n, case, cap)
    upload_lens(engine, lens)
    first = T.craft_first_merges(n, case, cap)
    for modified in (False, True):
        want = U.expected_tree(0, modified, lcs, lens)
        assert [tuple(m) for m in want[:len(first)].tolist()] == first
        for eb in (2, 4):
            t = device_triangle(lcs, eb)
            set_cap(monkeypatch, cap)
            capfd.readouterr()
            got = tree_from_triangle(engine, 0, modified, t)
            assert_capped(capfd, f"k_upgma<{int(modified)}>", n, cap)
            assert np.array_equal(got, want), (modified, eb)
            set_cap(monkeypatch, 0)
            assert np.array_equal(tree_from_triangle(engine, 0, modified, t), got), (modified, eb, "uncapped")
            del t


def nj_raw(engine, kind, n):
    """(status, merges buffer) of famsa_lcs_nj: a late step without a candidate returns FAMSA_E_INVALID after the same
    merges, capped or not."""
    out = np.zeros((n - 1, 2), dtype=np.int32)
    return engine.lib.famsa_lcs_nj(engine.h, kind, out.ctypes.data_as(C.c_void_p)), out


@pytest.mark.parametrize("cap,n", T.NJ_CASES, ids=[f"{n}-cap{c}" for c, n in T.NJ_CASES])
def test_nj(engine, monkeypatch, capfd, cap, n):
    """famsa_lcs_nj on `cap` blocks: up to ~70 scan rows per warp, against the restated computeTree and the uncapped call."""
    codes, offsets, lens = boundary_set(n, 3, 2000 + n)
    engine.upload(codes, offsets, lens)
    for kind in (0, 1):
        set_cap(monkeypatch, cap)
        capfd.readouterr()
        check_against_restatement(engine, kind, lens)
        lines = coop_lines(capfd.readouterr().err)
        assert lines == [("k_nj", n, cap)], lines
        got = nj_raw(engine, kind, n)
        set_cap(monkeypatch, 0)
        full = nj_raw(engine, kind, n)
        assert got[0] == full[0] and np.array_equal(got[1], full[1]), f"kind {kind}"
    capfd.readouterr()


def test_hemopexin_one_block(engine, monkeypatch, capfd):
    """The hemopexin set (4 188 sequences) on one block, up to five sequences per thread: every engine equals its
    uncapped run, and NJ the reference's tree (hemopexin_nj.npz)."""
    z = np.load(os.path.join(GOLDEN, "hemopexin_nj.npz"))
    engine.upload(*seqio.pack([seqio.encode(str(s)) for s in z["seqs"]]))
    n = len(z["seqs"])
    set_cap(monkeypatch, 0)
    full = dict(prim=engine.prim(0), slink=engine.slink(0), upgma0=engine.upgma(0, False), upgma1=engine.upgma(0, True))
    monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
    full_seq = dict(prim=engine.prim(0), slink=engine.slink(0))
    set_cap(monkeypatch, 1)
    capfd.readouterr()
    got = engine.prim(0)
    same(got, full["prim"], "prim")
    same(got, full_seq["prim"], "prim")
    assert np.array_equal(engine.slink(0), full["slink"])
    assert np.array_equal(full_seq["slink"], full["slink"])
    monkeypatch.delenv("FAMSA_PRIM_SEQUENTIAL")
    assert np.array_equal(engine.upgma(0, False), full["upgma0"])
    assert np.array_equal(engine.upgma(0, True), full["upgma1"])
    assert np.array_equal(engine.nj(0), z["tree0"])
    lines = coop_lines(capfd.readouterr().err)
    assert [k for k, _, _ in lines] == ["k_prim<0>", "k_prim<1>", "k_upgma<0>", "k_upgma<1>", "k_nj"]
    assert all(nn == n and b == 1 for _, nn, b in lines)


# ------------------------------------------------------------------ past 2^32 elements
def need_free(gb):
    free = torch.cuda.mem_get_info()[0]
    if free < gb * 1e9:
        pytest.skip(f"needs {gb} GB of free device memory, {free / 1e9:.1f} GB free")


@pytest.mark.parametrize("modified", [False, True])
def test_upgma_past_2_32(modified):
    """UPGMA on a u16 triangle of 93 000 rows (4 324 453 500 elements, 8.6 GB) built on the device, plus its 17.3 GB of
    float distances: every LCS 50 but planted pairs past 2^32 (one at the first cell of row 92 682 that is) and a triple
    whose second merge reads the averaged row k_upgma wrote past 2^32.  The first merges are derived by hand
    (tree_coop_cases.big_upgma_expected, checked on a small analogue by the host tests), and the tree is whole."""
    need_free(30)
    n = T.BIG_N
    eng = famsa_b200.Engine()
    try:
        upload_lens(eng, np.full(n, T.BIG_LEN))
        t = torch.full((n * (n - 1) // 2,), T.BIG_BG, dtype=torch.int16, device="cuda")
        for off, v in T.big_cells():
            t[off] = v
        torch.cuda.synchronize()
        got = tree_from_triangle(eng, 0, modified, t)
        del t
    finally:
        eng.close()
        torch.cuda.empty_cache()
    want = T.big_upgma_expected(n, T.BIG_PAIRS, T.BIG_TRIPLE, modified)
    assert [tuple(m) for m in got[:len(want)].tolist()] == want
    assert T.valid_tree(got, n)


def test_boruvka_and_slink_past_2_32(monkeypatch, capfd):
    """synth_family(93 000, 60): 8.6 GB of LCS triangle and 34.6 GB of float64 distances.  famsa_lcs_prim and
    famsa_lcs_slink with the Boruvka rounds (no k_prim line: they ran) equal the sequential loop, whose reads past 2^32
    test/LRR already covers, edge for edge."""
    need_free(48)
    codes, offsets, lens = seqio.synth_family(T.BIG_N, 60, seed=91)
    eng = famsa_b200.Engine()
    monkeypatch.setenv("FAMSA_TREE_DEBUG", "1")
    monkeypatch.delenv("FAMSA_TREE_MAX_BLOCKS", raising=False)
    try:
        eng.upload(codes, offsets, lens)
        capfd.readouterr()
        prim, slink = eng.prim(0), eng.slink(0)
        assert coop_lines(capfd.readouterr().err) == [], "the Boruvka rounds did not run"
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
        same(eng.prim(0), prim, "prim")
        assert np.array_equal(eng.slink(0), slink)
        assert [k for k, _, _ in coop_lines(capfd.readouterr().err)] == ["k_prim<0>", "k_prim<1>"]
    finally:
        eng.close()
        torch.cuda.empty_cache()
