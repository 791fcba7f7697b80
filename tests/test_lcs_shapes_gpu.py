"""Every instantiation of the LCS tile kernel k_lcs_tile<NL> at its limb, tail and group boundaries, against the oracle.

The sets come from tests/lcs_shapes.py: per limb count a sweep set whose groups are led by both ends of the count's length
range, carry-stress sets whose carries cross every limb boundary, and a set of dropped-carry rows and near misses.  The
device entry points are checked on a caller's stream, writing into the middle of a sentinel-filled buffer."""
import numpy as np
import pytest

from famsa_b200 import seqio
from lcs_shapes import INSTANTIATED, carry_set, group_nls, quirk_set, sweep_set
from oracle import pyoracle

pytestmark = pytest.mark.gpu


def _tri(r: int) -> int:
    return r * (r - 1) // 2 if r else 0


def _cuts(n: int) -> list[tuple[int, int]]:
    """Row ranges that tile [0, n) and cut mask groups: one row, part of group 0 and 1, the rest but 3, the last 3."""
    b = [0, 1, 33, 61, n - 3, n]
    return list(zip(b[:-1], b[1:]))


@pytest.mark.parametrize("nl", INSTANTIATED)
def test_triangle_every_instantiation(engine, nl):
    """u16 and u32 triangles of the sweep set: unsorted upload (one launch per distinct group limb count), and the
    length-sorted upload in row ranges that cut groups."""
    s = sweep_set(nl)
    codes, offsets, lens = seqio.pack(s["unsorted"])
    n = len(lens)
    engine.upload(codes, offsets, lens)
    want = pyoracle.lcs_triangle(codes, offsets, lens)
    before = engine.kernel_launches()
    got = engine.triangle(dtype=np.uint32)
    assert engine.kernel_launches() - before == len(set(group_nls(lens)))
    assert np.array_equal(got, want)
    assert np.array_equal(engine.triangle(dtype=np.uint16), want)

    codes, offsets, lens = seqio.pack(s["sorted"])
    engine.upload(codes, offsets, lens)
    want = pyoracle.lcs_triangle(codes, offsets, lens)
    for k, (a, b) in enumerate(_cuts(n)):
        got = engine.triangle(a, b, dtype=np.uint16 if k % 2 else np.uint32)
        assert np.array_equal(got, want[_tri(a):_tri(b)]), (a, b)


@pytest.mark.parametrize("nl", INSTANTIATED)
def test_rows_every_instantiation(engine, nl):
    """famsa_lcs_rows with 1, 7, 31, 32 and 33 streamed rows (33: two tiles per group) against columns from every
    group, duplicates included."""
    s = sweep_set(nl)
    codes, offsets, lens = seqio.pack(s["unsorted"])
    n = len(lens)
    engine.upload(codes, offsets, lens)
    rng = np.random.default_rng(nl)
    by_len = np.argsort(-lens.astype(np.int64), kind="stable")          # caller id at each sorted position
    cols = np.concatenate([rng.choice(by_len[g:g + 32], size=min(5, len(by_len[g:g + 32])), replace=False)
                           for g in range(0, n, 32)])
    cols = np.concatenate([cols, cols[::3], [by_len[0], by_len[-1]]])
    rng.shuffle(cols)
    for k, n_ref in enumerate((1, 7, 31, 32, 33)):
        refs = rng.choice(n, size=n_ref, replace=False)
        want = pyoracle.lcs_rows(codes, offsets, lens, refs, cols)
        got = engine.rows(refs, cols, dtype=np.uint16 if k % 2 else np.uint32)
        assert np.array_equal(got, want), n_ref


@pytest.mark.parametrize("nl", [n for n in INSTANTIATED if n >= 2])
def test_carry_stress(engine, nl):
    """A row whose 'A' mask is nearly all ones in every limb, against A-rich sequences: the triangle in both upload
    orders and the full square of rows, so the row is the mask side of an nl-limb group and the streamed side of others."""
    s = carry_set(nl)
    for order in ("unsorted", "sorted"):
        codes, offsets, lens = seqio.pack(s[order])
        n = len(lens)
        engine.upload(codes, offsets, lens)
        assert np.array_equal(engine.triangle(dtype=np.uint32), pyoracle.lcs_triangle(codes, offsets, lens))
        assert np.array_equal(engine.rows(np.arange(n), dtype=np.uint16), pyoracle.lcs_rows(codes, offsets, lens, np.arange(n)))


@pytest.mark.parametrize("order", ["unsorted", "sorted"])
def test_quirk_rows_and_near_misses(engine, order):
    """Rows with an aligned 64-run (exact kernels) and near misses (tile kernel) among ordinary rows: triangles, row
    ranges with flagged rows inside and outside, and the full square of rows."""
    s = quirk_set()
    codes, offsets, lens = seqio.pack(s[order])
    n = len(lens)
    engine.upload(codes, offsets, lens)
    want = pyoracle.lcs_triangle(codes, offsets, lens)
    assert np.array_equal(engine.triangle(dtype=np.uint32), want)
    assert np.array_equal(engine.triangle(dtype=np.uint16), want)
    for a, b in _cuts(n) + [(5, n - 20), (40, 41)]:
        assert np.array_equal(engine.triangle(a, b, dtype=np.uint32), want[_tri(a):_tri(b)]), (a, b)
    assert np.array_equal(engine.rows(np.arange(n)), pyoracle.lcs_rows(codes, offsets, lens, np.arange(n)))


SENTINEL = {2: 0xA5A5, 4: 0xA5A5A5A5}
PAD = 37                                    # sentinel elements before and after the written region


def _sentinel_buffer(torch, n_elems: int, eb: int):
    dt = torch.int16 if eb == 2 else torch.int32
    npdt = np.uint16 if eb == 2 else np.uint32
    fill = np.array([SENTINEL[eb]], dtype=npdt).view(np.int16 if eb == 2 else np.int32)[0]
    return torch.full((PAD + n_elems + PAD,), int(fill), dtype=dt, device="cuda"), npdt


def _check_region(buf, npdt, want):
    got = buf.cpu().numpy().view(npdt)
    eb = np.dtype(npdt).itemsize
    assert np.all(got[:PAD] == SENTINEL[eb]), "write before the caller's region"
    assert np.all(got[PAD + len(want):] == SENTINEL[eb]), "write after the caller's region"
    assert np.array_equal(got[PAD:PAD + len(want)], want)


@pytest.mark.parametrize("case", ["quirk_unsorted", "quirk_sorted", "sweep64_sorted"])
def test_device_entry_points_on_a_caller_stream(engine, case):
    """famsa_lcs_triangle_device and famsa_lcs_rows_device, u16 and u32, on a non-default stream: the caller's region
    equals the oracle and not one element before or after it is touched -- partial row ranges with flagged rows inside
    and outside, device column ids with duplicates, and the column prefix (col_ids = NULL)."""
    import torch
    if case == "sweep64_sorted":
        cl, flagged = sweep_set(64)["sorted"], []
    else:
        order = case.split("_")[1]
        cl, flagged = quirk_set()[order], quirk_set()["flagged"][order]
    codes, offsets, lens = seqio.pack(cl)
    n = len(lens)
    engine.upload(codes, offsets, lens)
    full = pyoracle.lcs_triangle(codes, offsets, lens)
    ranges = [(0, n), (1, 33), (33, n - 3)]
    if flagged:
        f = sorted(flagged)
        ranges += [(f[0] + 1, f[-1]), (f[len(f) // 2], n)]
        for a, b in ranges[3:]:
            assert any(a <= x < b for x in f) and any(not a <= x < b for x in f)
    stream = torch.cuda.Stream()
    for eb in (2, 4):
        for a, b in ranges:
            buf, npdt = _sentinel_buffer(torch, _tri(b) - _tri(a), eb)
            torch.cuda.synchronize()
            engine.triangle_device(a, b, buf.data_ptr() + PAD * eb, eb, stream.cuda_stream)
            stream.synchronize()
            _check_region(buf, npdt, full[_tri(a):_tri(b)])

    rng = np.random.default_rng(5)
    refs = np.concatenate([rng.choice(n, size=9, replace=False), flagged[:3]]).astype(np.int32)
    cols = np.concatenate([rng.choice(n, size=40, replace=False), flagged, flagged[:2], [0, n - 1, 0]]).astype(np.int32)
    d_refs = torch.from_numpy(refs).cuda()
    d_cols = torch.from_numpy(cols).cuda()
    for eb in (2, 4):
        for d_col, n_col, want in [(d_cols, len(cols), pyoracle.lcs_rows(codes, offsets, lens, refs, cols)),
                                   (None, n - 5, pyoracle.lcs_rows(codes, offsets, lens, refs, None, n - 5))]:
            buf, npdt = _sentinel_buffer(torch, len(refs) * n_col, eb)
            torch.cuda.synchronize()
            engine.rows_device(d_refs.data_ptr(), len(refs), d_col.data_ptr() if d_col is not None else 0, n_col,
                               buf.data_ptr() + PAD * eb, eb, stream.cuda_stream)
            stream.synchronize()
            _check_region(buf, npdt, want.reshape(-1))
