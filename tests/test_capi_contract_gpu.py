"""The C ABI's argument contract, through ctypes: the raw return code of every LCS entry point before an upload, of each
argument the host rejects after one, of the NULL arguments of the DP and profile entries, and of the empty calls that
succeed.  After every rejected call famsa_last_error() says something and the context still answers a valid
famsa_lcs_rows.  Then the scratch ordering of calls on two caller streams and the context stream, and the timing that
famsa_lcs_prim reports for a set with flagged sequences.  Every rejected call is refused before anything is launched."""
import ctypes as C

import numpy as np
import pytest

import famsa_b200
from famsa_b200 import seqio
from famsa_b200.binding import WRITE_FN
from conftest import QUIRK_SEQS, random_set
from oracle import pyoracle

pytestmark = pytest.mark.gpu

OK, E_INVALID, E_STATE = 0, 1, 4
NULL = None


def vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def u32(xs):
    return np.ascontiguousarray(xs, dtype=np.uint32)


def sink(_u, _p, _n):
    return 0


SINK = WRITE_FN(sink)


class Set:
    def __init__(self, code_list):
        self.codes, self.offsets, self.lens = seqio.pack(code_list)
        self.n = len(code_list)


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(5)
    return Set([seqio.encode(s) for s in QUIRK_SEQS] + random_set(rng, 36, 1, 300))


@pytest.fixture()
def ctx(data):
    """A context of its own (no earlier call has left a set, an error or queued work on it) with `data` uploaded."""
    eng = famsa_b200.Engine(0)
    eng.upload(data.codes, data.offsets, data.lens)
    yield eng
    eng.close()


def assert_usable(eng, s):
    """A rejected call leaves its message and a context that still computes."""
    assert eng.lib.famsa_last_error(), "no error message"
    refs = u32([0, s.n - 1, 1])
    out = np.zeros(len(refs) * s.n, dtype=np.uint32)
    assert eng.lib.famsa_lcs_rows(eng.h, vp(refs), len(refs), NULL, s.n, vp(out), 4) == OK
    assert np.array_equal(out.reshape(len(refs), s.n), pyoracle.lcs_rows(s.codes, s.offsets, s.lens, refs))


def export_args(n):
    ids = b"".join(b"s%d" % i for i in range(n))
    offs = np.array([0] + [len(b"".join(b"s%d" % i for i in range(k + 1))) for k in range(n)], dtype=np.uint64)
    return C.c_char_p(ids), offs


def lcs_calls(eng, n, kind=0, eb=2, row=(0, None), ref=None, col=None, seed=None, d_out=None, shard=(0, 1)):
    """One call of every LCS entry point, by name, with the given arguments (defaults: valid, whole set)."""
    lib, h = eng.lib, eng.h
    rb, re = row[0], n if row[1] is None else row[1]
    ref = u32([0]) if ref is None else ref
    seed = u32([0]) if seed is None else seed
    out = np.zeros(max(n * n, 1), dtype=np.uint32)
    f, t, d, o = (np.zeros(max(n, 1), dt) for dt in (np.int32, np.int32, np.float64, np.int32))
    a, m = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.float32)
    tree = np.zeros(2 * max(n, 1), np.int32)
    ids, offs = export_args(n)
    dptr = C.c_void_p(d_out) if d_out else None
    peer = (C.c_void_p * 1)(dptr)
    n_col = n if col is None else len(col)
    return {
        "triangle": lambda: lib.famsa_lcs_triangle(h, rb, re, vp(out), eb),
        "triangle_device": lambda: lib.famsa_lcs_triangle_device(h, rb, re, dptr, eb, NULL),
        "triangle_exchange": lambda: lib.famsa_lcs_triangle_exchange(h, rb, re, dptr, peer, 1, eb, 8, NULL),
        "rows": lambda: lib.famsa_lcs_rows(h, vp(ref), len(ref), vp(col), n_col, vp(out), eb),
        "prim": lambda: lib.famsa_lcs_prim(h, kind, vp(f), vp(t), vp(d), vp(o)),
        "assign": lambda: lib.famsa_lcs_assign(h, vp(seed), len(seed), kind, vp(a), vp(m)),
        "assign_shard": lambda: lib.famsa_lcs_assign_shard(h, vp(seed), len(seed), kind, shard[0], shard[1], dptr, NULL),
        "upgma": lambda: lib.famsa_lcs_upgma(h, kind, 0, vp(tree)),
        "upgma_from_triangle": lambda: lib.famsa_lcs_upgma_from_triangle(h, kind, 0, dptr, eb, vp(tree)),
        "dist_export": lambda: lib.famsa_dist_export(h, kind, 0, 0, ids, vp(offs), 0, SINK, NULL, NULL),
    }


def test_null_context():
    lib = famsa_b200.load_library()
    z = C.c_void_p(0)
    for rc in (lib.famsa_lcs_upload(z, NULL, NULL, NULL, 0), lib.famsa_lcs_sorted_order(z, NULL),
               lib.famsa_lcs_triangle(z, 0, 0, NULL, 2), lib.famsa_lcs_triangle_device(z, 0, 0, NULL, 2, NULL),
               lib.famsa_lcs_triangle_exchange(z, 0, 0, NULL, NULL, 0, 2, 1, NULL),
               lib.famsa_lcs_rows(z, NULL, 0, NULL, 0, NULL, 4), lib.famsa_lcs_rows_device(z, NULL, 0, NULL, 0, NULL, 4, NULL),
               lib.famsa_lcs_prim(z, 0, NULL, NULL, NULL, NULL), lib.famsa_lcs_assign(z, NULL, 0, 0, NULL, NULL),
               lib.famsa_lcs_assign_shard(z, NULL, 0, 0, 0, 1, NULL, NULL), lib.famsa_lcs_upgma(z, 0, 0, NULL),
               lib.famsa_lcs_upgma_from_triangle(z, 0, 0, NULL, 2, NULL),
               lib.famsa_dist_export(z, 0, 0, 0, NULL, NULL, 0, SINK, NULL, NULL),
               lib.famsa_dp_align_batch(z, NULL, 0, NULL, NULL, NULL, NULL),
               lib.famsa_dp_align_batch_device(z, NULL, 0, NULL, NULL, NULL, NULL, NULL),
               lib.famsa_prof_set_scoring(z, NULL), lib.famsa_prof_put(z, NULL, 0, NULL),
               lib.famsa_prof_merge_batch(z, NULL, 0, NULL, NULL, NULL, NULL, 0), lib.famsa_prof_drop(z, NULL, 0),
               lib.famsa_prof_align_tree(z, NULL, 0, NULL, NULL, NULL, NULL, NULL), lib.famsa_prof_tree_paths(z, NULL, 0)):
        assert rc == E_INVALID


def test_every_lcs_entry_before_an_upload(data):
    eng = famsa_b200.Engine(0)
    try:
        lib, h = eng.lib, eng.h
        d_buf = eng.device_alloc(1 << 16)
        try:
            calls = lcs_calls(eng, 4, d_out=d_buf, row=(0, 3))
            calls["rows_device"] = lambda: lib.famsa_lcs_rows_device(h, C.c_void_p(d_buf), 1, NULL, 1, C.c_void_p(d_buf), 4, NULL)
            got, said = {}, {}
            for name, call in calls.items():
                got[name] = call()
                said[name] = bool(lib.famsa_last_error())
            want = {name: E_STATE for name in calls}
            want["triangle"] = E_INVALID                    # its row range is checked first: row_end > n = 0
            assert got == want
            assert all(said.values()), said
            # the empty calls that succeed without a set, and the element width that is checked all the same
            got = {"triangle": lib.famsa_lcs_triangle(h, 0, 0, NULL, 2),
                   "triangle_device": lib.famsa_lcs_triangle_device(h, 0, 0, NULL, 2, NULL),
                   "sorted_order": lib.famsa_lcs_sorted_order(h, NULL),
                   "triangle eb=3": lib.famsa_lcs_triangle(h, 0, 0, NULL, 3),
                   "triangle_device eb=3": lib.famsa_lcs_triangle_device(h, 0, 0, NULL, 3, NULL)}
            assert got == {"triangle": OK, "triangle_device": OK, "sorted_order": OK, "triangle eb=3": E_INVALID,
                           "triangle_device eb=3": E_INVALID}
        finally:
            eng.device_free(d_buf)
        eng.upload(data.codes, data.offsets, data.lens)
        assert_usable(eng, data)
    finally:
        eng.close()


def rejected(eng, n):
    """(label, call) for each argument the host rejects after an upload of n sequences: all FAMSA_E_INVALID."""
    lib, h = eng.lib, eng.h
    d = eng.device_alloc(4 * n * n + 64)
    out = [("free", d)]
    big = u32([n])
    for name in ("triangle", "triangle_device", "triangle_exchange", "rows", "upgma_from_triangle"):
        out.append((f"{name} eb=3", lcs_calls(eng, n, eb=3, d_out=d)[name]))
    for name in ("triangle", "triangle_device", "triangle_exchange"):
        out.append((f"{name} begin>end", lcs_calls(eng, n, row=(5, 4), d_out=d)[name]))
        out.append((f"{name} end>n", lcs_calls(eng, n, row=(0, n + 1), d_out=d)[name]))
    out += [("triangle out NULL", lambda: lib.famsa_lcs_triangle(h, 0, n, NULL, 2)),
            ("triangle_device out NULL", lambda: lib.famsa_lcs_triangle_device(h, 0, n, NULL, 2, NULL)),
            ("exchange d_full NULL", lcs_calls(eng, n)["triangle_exchange"]),
            ("exchange peers NULL", lambda: lib.famsa_lcs_triangle_exchange(h, 0, n, C.c_void_p(d), NULL, 1, 2, 8, NULL)),
            ("rows ref NULL", lambda: lib.famsa_lcs_rows(h, NULL, 1, NULL, n, C.c_void_p(d), 4)),
            ("rows out NULL", lambda: lib.famsa_lcs_rows(h, vp(u32([0])), 1, NULL, n, NULL, 4)),
            ("rows n_col > n", lambda: lib.famsa_lcs_rows(h, vp(u32([0])), 1, NULL, n + 1, vp(np.zeros(n + 1, np.uint32)), 4)),
            ("rows ref >= n", lcs_calls(eng, n, eb=4, ref=big)["rows"]),
            ("rows col >= n", lcs_calls(eng, n, eb=4, col=u32([0, n]))["rows"]),
            ("rows_device ref NULL", lambda: lib.famsa_lcs_rows_device(h, NULL, 1, NULL, n, C.c_void_p(d), 4, NULL)),
            ("rows_device eb=3", lambda: lib.famsa_lcs_rows_device(h, C.c_void_p(d), 0, NULL, n, C.c_void_p(d), 3, NULL)),
            ("rows_device n_col > n", lambda: lib.famsa_lcs_rows_device(h, C.c_void_p(d), 0, NULL, n + 1, C.c_void_p(d), 4, NULL)),
            ("prim kind 2", lcs_calls(eng, n, kind=2)["prim"]),
            ("prim kind -1", lcs_calls(eng, n, kind=-1)["prim"]),
            ("prim order NULL", lambda: lib.famsa_lcs_prim(h, 0, vp(np.zeros(n, np.int32)), vp(np.zeros(n, np.int32)),
                                                           vp(np.zeros(n)), NULL)),
            ("assign seeds NULL", lambda: lib.famsa_lcs_assign(h, NULL, 1, 0, vp(np.zeros(n, np.uint32)), vp(np.zeros(n, np.float32)))),
            ("assign no seeds", lcs_calls(eng, n, seed=u32([]))["assign"]),
            ("assign kind 3", lcs_calls(eng, n, kind=3)["assign"]),
            ("assign kind -1", lcs_calls(eng, n, kind=-1)["assign"]),
            ("assign seed >= n", lcs_calls(eng, n, seed=u32([1, n]))["assign"]),
            ("assign_shard packed NULL", lcs_calls(eng, n)["assign_shard"]),
            ("assign_shard kind 3", lcs_calls(eng, n, kind=3, d_out=d)["assign_shard"]),
            ("assign_shard n_shards 0", lcs_calls(eng, n, d_out=d, shard=(0, 0))["assign_shard"]),
            ("assign_shard shard >= n_shards", lcs_calls(eng, n, d_out=d, shard=(2, 2))["assign_shard"]),
            ("assign_shard seed >= n", lcs_calls(eng, n, d_out=d, seed=big)["assign_shard"]),
            ("upgma tree NULL", lambda: lib.famsa_lcs_upgma(h, 0, 0, NULL)),
            ("upgma kind 3", lcs_calls(eng, n, kind=3)["upgma"]),
            ("upgma kind 2", lcs_calls(eng, n, kind=2)["upgma"]),                  # a similarity: no UPGMA instantiation
            ("upgma kind -1", lcs_calls(eng, n, kind=-1)["upgma"]),
            ("upgma_from_triangle NULL", lcs_calls(eng, n)["upgma_from_triangle"]),
            ("upgma_from_triangle kind -1", lcs_calls(eng, n, kind=-1, d_out=d)["upgma_from_triangle"]),
            ("upgma_from_triangle kind 2", lcs_calls(eng, n, kind=2, d_out=d)["upgma_from_triangle"]),
            ("upgma_from_triangle kind 3", lcs_calls(eng, n, kind=3, d_out=d)["upgma_from_triangle"]),
            ("dist_export kind 2", lcs_calls(eng, n, kind=2)["dist_export"]),
            ("dist_export ids NULL", lambda: lib.famsa_dist_export(h, 0, 0, 0, NULL, vp(export_args(n)[1]), 0, SINK, NULL, NULL)),
            ("dist_export decreasing offsets", lambda: lib.famsa_dist_export(h, 0, 0, 1, export_args(n)[0],
                                                                             vp(export_args(n)[1][::-1].copy()), 0, SINK, NULL, NULL))]
    return out


def test_rejected_arguments(ctx, data):
    import torch
    calls = rejected(ctx, data.n)
    d = calls.pop(0)[1]
    d_ref = torch.tensor([data.n], dtype=torch.int32, device="cuda")      # a reference id out of range, on the device
    calls.append(("rows_device ref >= n", lambda: ctx.lib.famsa_lcs_rows_device(
        ctx.h, C.c_void_p(d_ref.data_ptr()), 1, NULL, data.n, C.c_void_p(d), 4, NULL)))
    torch.cuda.synchronize()
    try:
        got = {}
        for label, call in calls:
            got[label] = call()
            assert_usable(ctx, data)
        assert got == {label: E_INVALID for label, _ in calls}
    finally:
        ctx.device_free(d)


def test_empty_calls_after_an_upload(ctx, data):
    lib, h = ctx.lib, ctx.h
    order = np.zeros(data.n, np.uint32)
    got = {"rows n_ref 0": lib.famsa_lcs_rows(h, NULL, 0, NULL, data.n, NULL, 4),
           "rows n_col 0": lib.famsa_lcs_rows(h, vp(u32([0])), 1, NULL, 0, NULL, 2),
           "rows_device n_ref 0": lib.famsa_lcs_rows_device(h, NULL, 0, NULL, data.n, NULL, 4, NULL),
           "triangle 3..3": lib.famsa_lcs_triangle(h, 3, 3, NULL, 4),
           "triangle 0..1": lib.famsa_lcs_triangle(h, 0, 1, NULL, 4),                  # row 0 has no pairs
           "triangle_device 0..1": lib.famsa_lcs_triangle_device(h, 0, 1, NULL, 2, NULL),
           "sorted_order NULL": lib.famsa_lcs_sorted_order(h, NULL),
           "sorted_order": lib.famsa_lcs_sorted_order(h, vp(order))}
    assert got == {"rows n_ref 0": OK, "rows n_col 0": OK, "rows_device n_ref 0": OK, "triangle 3..3": OK,
                   "triangle 0..1": OK, "triangle_device 0..1": OK, "sorted_order NULL": E_INVALID, "sorted_order": OK}
    assert np.array_equal(order, np.arange(data.n))
    assert_usable(ctx, data)


def test_element_width_of_a_long_set():
    """elem_bytes = 2 cannot hold the LCS of a sequence of 65536 residues."""
    rng = np.random.default_rng(2)
    s = Set([rng.integers(0, 20, 65536).astype(np.int8)] + random_set(rng, 5, 10, 60))
    eng = famsa_b200.Engine(0)
    try:
        eng.upload(s.codes, s.offsets, s.lens)
        d = eng.device_alloc(4 * s.n * s.n + 64)
        try:
            calls = lcs_calls(eng, s.n, eb=2, d_out=d)
            for name in ("triangle", "triangle_device", "triangle_exchange", "rows"):
                assert calls[name]() == E_INVALID, name
                assert_usable(eng, s)
            assert eng.lib.famsa_lcs_rows_device(eng.h, C.c_void_p(d), 0, NULL, s.n, C.c_void_p(d), 2, NULL) == E_INVALID
            assert_usable(eng, s)
        finally:
            eng.device_free(d)
    finally:
        eng.close()


def test_upgma_needs_two_sequences():
    s = Set([seqio.encode("ACDEFG")])
    eng = famsa_b200.Engine(0)
    try:
        eng.upload(s.codes, s.offsets, s.lens)
        d = eng.device_alloc(64)
        try:
            calls = lcs_calls(eng, 1, d_out=d)
            assert calls["upgma"]() == E_STATE
            assert calls["upgma_from_triangle"]() == E_STATE
            assert eng.lib.famsa_last_error()
        finally:
            eng.device_free(d)
    finally:
        eng.close()


def test_dp_and_profile_null_arguments(ctx, data):
    lib, h = ctx.lib, ctx.h
    g = np.zeros(4, np.int64)
    one = np.zeros(64, np.uint8)
    got = {}
    for label, rc in [("dp jobs NULL", lib.famsa_dp_align_batch(h, NULL, 1, vp(g), vp(one), vp(one), NULL)),
                      ("dp gaps NULL", lib.famsa_dp_align_batch(h, vp(one), 1, NULL, vp(one), vp(one), NULL)),
                      ("dp results NULL", lib.famsa_dp_align_batch(h, vp(one), 1, vp(g), NULL, vp(one), NULL)),
                      ("dp path NULL", lib.famsa_dp_align_batch(h, vp(one), 1, vp(g), vp(one), NULL, NULL)),
                      ("dp_device jobs NULL", lib.famsa_dp_align_batch_device(h, NULL, 1, vp(g), NULL, NULL, NULL, NULL)),
                      ("dp_device results NULL", lib.famsa_dp_align_batch_device(h, vp(one), 1, vp(g), NULL, vp(one), NULL, NULL)),
                      ("scoring NULL", lib.famsa_prof_set_scoring(h, NULL)),
                      ("put NULL", lib.famsa_prof_put(h, NULL, 1, vp(one))),
                      ("put ids NULL", lib.famsa_prof_put(h, vp(one), 1, NULL)),
                      ("merge NULL", lib.famsa_prof_merge_batch(h, NULL, 1, vp(g), vp(one), vp(one), vp(one), 64)),
                      ("merge gaps NULL", lib.famsa_prof_merge_batch(h, vp(one), 1, NULL, vp(one), vp(one), vp(one), 64)),
                      ("align_tree NULL", lib.famsa_prof_align_tree(h, NULL, 2, vp(g), vp(one), NULL, NULL, NULL)),
                      ("tree_paths NULL", lib.famsa_prof_tree_paths(h, NULL, 0)),
                      ("drop NULL", lib.famsa_prof_drop(h, NULL, 1))]:
        got[label] = rc
        assert_usable(ctx, data)
    assert got == {label: E_INVALID for label in got}
    # the empty batches succeed
    got = {"dp": lib.famsa_dp_align_batch(h, NULL, 0, NULL, NULL, NULL, NULL),
           "dp_device": lib.famsa_dp_align_batch_device(h, NULL, 0, NULL, NULL, NULL, NULL, NULL),
           "put": lib.famsa_prof_put(h, NULL, 0, NULL),
           "drop": lib.famsa_prof_drop(h, NULL, 0)}
    assert got == {"dp": OK, "dp_device": OK, "put": OK, "drop": OK}
    assert_usable(ctx, data)


def test_scratch_order_across_streams():
    """rows_device on one caller stream, triangle_device on a second, then famsa_lcs_rows on the context's stream, with
    nothing synchronised in between: every result is the oracle's."""
    import torch
    rng = np.random.default_rng(9)
    s = Set([seqio.encode(q) for q in QUIRK_SEQS] + random_set(rng, 400, 50, 600))
    eng = famsa_b200.Engine(0)
    try:
        eng.upload(s.codes, s.offsets, s.lens)
        refs = u32(rng.choice(s.n, size=40, replace=False))
        refs[:2] = [1, 3]
        cols = u32(np.concatenate([rng.choice(s.n, size=150), [0, 1, 3]]))
        d_refs = torch.from_numpy(refs.view(np.int32)).cuda()
        d_cols = torch.from_numpy(cols.view(np.int32)).cuda()
        d_rows = torch.zeros(len(refs) * len(cols), dtype=torch.int32, device="cuda")
        d_tri = torch.zeros(s.n * (s.n - 1) // 2, dtype=torch.int32, device="cuda")
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        lib, h = eng.lib, eng.h
        assert lib.famsa_lcs_rows_device(h, C.c_void_p(d_refs.data_ptr()), len(refs), C.c_void_p(d_cols.data_ptr()), len(cols),
                                         C.c_void_p(d_rows.data_ptr()), 4, C.c_void_p(s1.cuda_stream)) == OK
        assert lib.famsa_lcs_triangle_device(h, 0, s.n, C.c_void_p(d_tri.data_ptr()), 4, C.c_void_p(s2.cuda_stream)) == OK
        host_refs = u32([2, 0, s.n - 1])
        out = np.zeros(len(host_refs) * s.n, np.uint32)
        assert lib.famsa_lcs_rows(h, vp(host_refs), len(host_refs), NULL, s.n, vp(out), 4) == OK
        torch.cuda.synchronize()
        assert np.array_equal(out.reshape(-1, s.n), pyoracle.lcs_rows(s.codes, s.offsets, s.lens, host_refs))
        assert np.array_equal(d_rows.cpu().numpy().view(np.uint32).reshape(len(refs), len(cols)),
                              pyoracle.lcs_rows(s.codes, s.offsets, s.lens, refs, cols))
        assert np.array_equal(d_tri.cpu().numpy().view(np.uint32), pyoracle.lcs_triangle(s.codes, s.offsets, s.lens))
    finally:
        eng.close()


def test_prim_timing_counts_the_triangle():
    """famsa_lcs_prim on a set with two flagged sequences: the call's pairs are the triangle's, and its total covers
    the tile kernels."""
    s = Set([seqio.encode(q) for q in QUIRK_SEQS])
    eng = famsa_b200.Engine(0)
    try:
        eng.upload(s.codes, s.offsets, s.lens)
        eng.prim(0)
        total, main, pairs = eng.last_timing()
        assert pairs == 6
        assert total >= main > 0
    finally:
        eng.close()
