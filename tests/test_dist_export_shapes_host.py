"""CPU tests of tests/dist_export_shapes.py: the generator is built on dist_export.cu's constants, the stage holds a
tile of the widest text, every case has the property it is named for, chunk_plan restates the host planner on hand-made
rows, and (where oracle/_ref is built) the restated text of every case equals the reference's DistanceCalculator."""
import os
import re

import numpy as np
import pytest

import dist_export_oracle as O
import dist_export_shapes as S
import lcs_shapes
from famsa_b200 import seqio
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "famsa_b200", "csrc", "dist_export.cu")).read()
CTX = open(os.path.join(ROOT, "famsa_b200", "csrc", "ctx.h")).read()
need_ref = pytest.mark.skipif(not pyoracle.have("ref_dist"), reason="oracle/_ref/libfamsa_ref_dist.so not built")


def test_constants_match_dist_export_cu():
    for name, value in (("kFmtThreads", S.K_FMT_THREADS), ("kFmtPerThread", S.K_FMT_PER_THREAD),
                        ("kMaxValueChars", S.K_MAX_VALUE_CHARS)):
        m = re.search(rf"constexpr int {name} = (\d+);", SRC)
        assert m and int(m.group(1)) == value, name
    assert re.search(r"constexpr int kFmtTile = kFmtThreads \* kFmtPerThread;", SRC)
    m = re.search(r"constexpr uint64_t kDefaultChunk = (\d+)ull << (\d+);", SRC)
    assert m and int(m.group(1)) << int(m.group(2)) == S.K_DEFAULT_CHUNK
    # k_dist_format's stage, and the launches of both passes with kFmtThreads threads
    body = re.search(r"k_dist_format\(.*?\n\{(.*?)\n\}", SRC, re.S).group(1)
    assert "__shared__ __align__(16) char stage[kFmtTile * kMaxValueChars + 32];" in body
    assert S.STAGE_BYTES == S.K_FMT_TILE * S.K_MAX_VALUE_CHARS + 32
    assert "k_dist_row_bytes<<<n, kFmtThreads, 0, st>>>" in SRC and "k_dist_format<<<r1 - r0, kFmtThreads, 0, st>>>" in SRC
    assert re.search(r"int elem_bytes\(\) const \{ return max_len < (\d+) \? 2 : 4; \}", CTX).group(1) == str(S.ELEM_WIDTH_LEN)


def elem_bytes(code_list) -> int:
    return 2 if max(len(c) for c in code_list) < S.ELEM_WIDTH_LEN else 4


@pytest.fixture(scope="module")
def wide_lcs():
    c = S.wide_elem()
    codes, offsets, lens = seqio.pack(c["code_list"])
    return O.lcs_square(codes, offsets, lens), lens


def test_stage_holds_a_tile_of_the_widest_text(wide_lcs):
    """+inf, NaN, FLT_MAX and the largest finite distance of wide_elem (any kind) with their ',': at most
    kMaxValueChars, and a tile of them plus the largest 16-byte phase fits the stage."""
    lcs, lens = wide_lcs
    finite = [v[np.isfinite(v)].max() for v in (O.transform_matrix(lcs, lens, lens, k, p) for k, p in ((0, 0), (1, 0), (0, 1)))]
    assert max(finite) > 30000                                    # kind 1: the 70 000-residue row's indels over an LCS of 2
    vals = np.array([np.inf, np.nan, np.finfo(np.float32).max] + finite, dtype=np.float32)
    texts = O.num2str(vals)
    assert texts[0] == texts[1] == S.INF_TEXT
    widest = max(len(t) + 1 for t in texts)
    assert widest == len(S.INF_TEXT) + 1 == 39
    assert widest <= S.K_MAX_VALUE_CHARS
    assert S.K_FMT_TILE * widest + 15 <= S.STAGE_BYTES


def test_cases_are_distinct_and_well_formed():
    cs = S.cases()
    assert len({c["name"] for c in cs}) == len(cs)
    for c in cs:
        assert len(c["ids"]) == len(c["code_list"]) and c["modes"] and set(c["modes"]) <= set(S.ALL_MODES), c["name"]
        assert not any(b"\n" in i or b"\0" in i for i in c["ids"]), c["name"]
        assert all(x.dtype == np.int8 and ((x >= 0) & (x < 24)).all() for x in c["code_list"]), c["name"]


def test_widths_tri_covers_every_width():
    c = S.widths_tri()
    n = len(c["code_list"])
    widths = set(range(n))                                        # triangle: row r has r columns
    assert n == 2050 and all(not sq for _, sq, _ in c["modes"])
    assert {k * S.K_FMT_THREADS + d for k in range(1, 9) for d in (-1, 0, 1)} <= widths           # pass 1's stride
    assert {S.K_FMT_TILE + d for d in (-1, 0, 1)} | {2 * S.K_FMT_TILE + d for d in (-1, 0, 1)} <= widths  # pass 2's tiles
    last = {(w - 1) % S.K_FMT_TILE + 1 for w in widths if w > S.K_FMT_TILE}                     # columns in the last tile
    assert {x % S.K_FMT_PER_THREAD for x in last} == set(range(S.K_FMT_PER_THREAD))
    lens = [len(x) for x in c["code_list"]]
    assert min(lens) == 5 and max(lens) == 60
    assert set(np.concatenate(c["code_list"]).tolist()) == set(range(24))                      # B/Z/X/* too


def test_widths_sq_and_the_default_chunk():
    for n in S.SQ_WIDTHS:
        c = S.widths_sq(n)
        assert len(c["code_list"]) == n and all(sq for _, sq, _ in c["modes"])
    c = S.widths_sq(2049)
    text = O.expected(c["code_list"], c["ids"], *S.SQ)
    header, rows = S.split_rows(text, True)
    assert len(rows) == 2049 and len(text) - header > S.K_DEFAULT_CHUNK
    plan = S.chunk_plan(rows, 0, header)
    assert len(plan) == 3 and plan[0] == header and sum(plan) == len(text)


def test_widest_first_tile_is_the_widest_text_at_every_phase():
    c = S.widest()
    a = c["claims"]["group_b"]
    cl, ids = c["code_list"], c["ids"]
    assert a >= S.K_FMT_TILE and set(np.concatenate(cl[:a]).tolist()) == set(range(10))
    assert set(np.concatenate(cl[a:]).tolist()) == set(range(10, 20))
    assert sorted({len(i) for i in ids[a:]}) == list(range(1, 17))
    group_b = range(a, len(cl))
    for mode in (S.TRI, S.TRI1, S.TRI_PID):
        text = O.expected(cl, ids, *mode)
        _, rows = S.split_rows(text, False)
        lines = text.split(b"\n")
        want = S.INF_TEXT if not mode[2] else b"0.000000"
        for r in group_b:
            assert lines[r].split(b",")[1:1 + S.K_FMT_TILE] == [want] * S.K_FMT_TILE, (mode, r)
        if not mode[2]:
            phases = {s % 16 for s in S.value_starts(rows, ids, group_b)}
            assert phases == set(range(16)), mode


def test_ids_lengths_and_bytes():
    ids = S.ids_case()["ids"]
    assert len(ids) == 40
    assert set(S.ID_LENGTHS) <= {len(i) for i in ids}
    assert {0, 255, 256, 257, 1000, 5000} <= {len(i) for i in ids}
    high = [i for i in ids if any(b >= 0x80 for b in i)]
    utf8 = [i for i in high if i.decode("utf-8", "replace").encode() == i]
    assert utf8 and len(utf8) < len(high)                         # UTF-8 text and bytes that are not
    assert any(b"," in i for i in ids) and b"," in ids and b"" in ids
    assert any(len(i) > S.K_FMT_THREADS for i in ids)


def test_wide_elem_widths_flags_and_order():
    c = S.wide_elem()
    cl, cm = c["code_list"], c["claims"]
    n = len(cl)
    assert elem_bytes(cl) == 4 and len(cl[cm["wide"]]) == S.WIDE_LEN
    assert S.K_FMT_TILE < cm["wide"] < n                                               # rows cross a tile, its own too
    assert [i for i in range(n) if lcs_shapes.quirky(cl[i])] == cm["flagged"]
    assert [i for i in range(n) if len(cl[i]) > 2048] == sorted(cm["long"] + [cm["wide"]])
    # flagged before and after the wide sequence; the over-long pair around it, the later one flagged
    lo, hi = cm["long"]
    assert min(cm["flagged"]) < cm["wide"] < max(cm["flagged"])
    assert lo < cm["wide"] < hi and hi in cm["flagged"] and lo not in cm["flagged"]


@pytest.mark.parametrize("max_len", [S.ELEM_WIDTH_LEN - 1, S.ELEM_WIDTH_LEN])
def test_wide_elem_threshold_sides(max_len):
    cl = S.wide_elem_edge(max_len)["code_list"]
    assert max(len(x) for x in cl) == max_len and elem_bytes(cl) == (2 if max_len < S.ELEM_WIDTH_LEN else 4)
    codes, offsets, lens = seqio.pack(cl)
    assert pyoracle.lcs_rows(codes, offsets, lens, [len(cl) - 1], col_ids=[0])[0, 0] == max_len


def test_empty_positions():
    c = S.empty()
    cl = c["code_list"]
    at = [i for i, x in enumerate(cl) if len(x) == 0]
    assert at == list(c["claims"]["empty"]) and at[0] == 0 and at[-1] == len(cl) - 1 and len(at) == 3
    assert c["modes"] == S.ALL_MODES


def test_chunk_plan_by_hand():
    rows = [10, 20, 30, 40]
    assert S.chunk_plan(rows, 30) == [30, 30, 40]                 # [10, 20] fills 30 exactly: 20 stays
    assert S.chunk_plan(rows, 29) == [10, 20, 30, 40]             # one byte less: 20 moves on; 30 > 29 alone
    assert S.chunk_plan(rows, 60) == [60, 40]
    assert S.chunk_plan([5, 100, 5, 5], 10) == [5, 100, 10]       # a row wider than chunk_bytes is a chunk of its own
    assert S.chunk_plan([100, 5], 10) == [100, 5]
    assert S.chunk_plan(rows, 1) == rows                          # one row per chunk
    assert S.chunk_plan(rows, 0) == [100] and S.chunk_plan(rows, 0, header=7) == [7, 100]
    big = [1 << 20] * 40
    assert S.chunk_plan(big, 0) == [32 << 20, 8 << 20]            # 0: kDefaultChunk
    assert S.chunk_plan([3], 1, header=9) == [9, 3]


def test_split_rows_and_value_starts():
    text = b",x,yy\nx,1.000000,0.500000\nyy,0.500000,1.000000\n"
    header, rows = S.split_rows(text, True)
    assert header == 6 and rows == [20, 21]
    assert S.value_starts(rows, [b"x", b"yy"], [0, 1]) == [2, 23]


@need_ref
def test_restatement_equals_reference():
    """The reference's DistanceCalculator on every case and mode but `empty`: on an 11-sequence set with empty
    sequences at 0, 6 and 10 the reference's export crashes (kind 0, triangle), so that case is checked against the
    restatement alone."""
    for c in S.cases():
        if c["name"] == "empty":
            continue
        codes, offsets, lens = seqio.pack(c["code_list"])
        lcs = O.lcs_square(codes, offsets, lens)
        letters = [seqio.decode(x) for x in c["code_list"]]
        for mode in c["modes"]:
            want = O.ref_dist_export(letters, c["ids"], *mode, n_threads=8)
            assert O.csv_from_lcs(lcs, lens, c["ids"], *mode) == want, (c["name"], mode)
