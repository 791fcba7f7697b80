"""famsa_dist_export past the sizes where its loops repeat (tests/dist_export_shapes.py): rows of every width up to
2 049 columns, tiles of the widest text at every 16-byte phase, ids up to 5 000 bytes, the uint32 LCS triangle and
empty sequences give the reference's DistanceCalculator text (live where oracle/_ref is built, else the restatement in
dist_export_oracle.py), and chunked exports call `write` with the sizes the host planner gives."""
import ctypes as C

import pytest

from famsa_b200 import seqio
import dist_export_oracle as O
import dist_export_shapes as S
from test_dist_export_gpu import raw_export

pytestmark = pytest.mark.gpu

E_OK = 0
CASE_MODES = [(name, mode) for name, modes in S.MODES.items() if name != "empty" for mode in modes]


def mode_id(mode) -> str:
    kind, square, pid = mode
    return ("sq" if square else "tri") + ("_pid" if pid else f"_k{kind}")


@pytest.fixture(scope="module")
def want():
    """want(name, mode): the expected text, computed once per module."""
    cache = {}

    def get(name, mode):
        if (name, mode) not in cache:
            c = S.case(name)
            cache[name, mode] = O.expected(c["code_list"], c["ids"], *mode, live=name != "empty")
        return cache[name, mode]
    return get


def first_difference(a: bytes, b: bytes) -> int:
    return next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))


def export_and_check(engine, want, name, mode):
    c = S.case(name)
    n = len(c["code_list"])
    engine.upload(*seqio.pack(c["code_list"]))
    got, text = engine.dist_export(c["ids"], *mode), want(name, mode)
    assert got == text, (name, mode, len(got), len(text), first_difference(got, text))
    assert engine.last_timing()[2] == (n * n if mode[1] else n * (n - 1) // 2)


@pytest.mark.parametrize("name,mode", CASE_MODES, ids=[f"{n}-{mode_id(m)}" for n, m in CASE_MODES])
def test_equals_reference(engine, want, name, mode):
    export_and_check(engine, want, name, mode)


@pytest.mark.parametrize("mode", S.ALL_MODES, ids=mode_id)
def test_empty_sequences(engine, want, mode):
    """Length-0 sequences first, in the middle and last, against the restatement only: on an 11-sequence set with empty
    sequences at 0, 6 and 10 the reference's DistanceCalculator crashed (kind 0, triangle; it accepted a 7-sequence set
    with empty sequences at 0 and 6).  Every cell of an empty sequence prints as +inf (kinds 0 and 1) or NaN (pid)."""
    export_and_check(engine, want, "empty", mode)


CHUNKED = [("widths_tri", S.TRI), ("widths_sq_2049", S.SQ), ("widest", S.TRI)]
CHUNK_SIZES = ("default", "one_byte", "prefix", "prefix_minus_1", "five_chunks")


@pytest.mark.parametrize("which", CHUNK_SIZES)
@pytest.mark.parametrize("name,mode", CHUNKED, ids=[n for n, _ in CHUNKED])
def test_chunks_follow_the_planner(engine, want, name, mode, which):
    """The sizes passed to `write` are chunk_plan's: a chunk that fills chunk_bytes exactly keeps its last row, one byte
    less moves that row on, 1 gives one row per chunk, 0 is 32 MiB (two chunks of widths_sq_2049), and five chunks or
    more reuse both device / pinned buffer pairs more than once.  Their concatenation is the text and *bytes_written
    its length."""
    c = S.case(name)
    text = want(name, mode)
    header, rows = S.split_rows(text, mode[1])
    k = len(rows) // 3                                            # the prefix: rows [0, k)
    chunk = {"default": 0, "one_byte": 1, "prefix": sum(rows[:k]), "prefix_minus_1": sum(rows[:k]) - 1,
             "five_chunks": sum(rows) // 6 + 1}[which]
    plan = S.chunk_plan(rows, chunk, header)
    chunks = plan[header is not None:]
    assert {"default": len(chunks) == (2 if name == "widths_sq_2049" else 1), "one_byte": chunks == rows,
            "prefix": chunks[0] == sum(rows[:k]), "prefix_minus_1": chunks[0] == sum(rows[:k - 1]),
            "five_chunks": len(chunks) >= 5}[which]
    engine.upload(*seqio.pack(c["code_list"]))
    calls = []

    def sink(_u, ptr, n):
        calls.append(C.string_at(ptr, n))
        return 0

    rc, written = raw_export(engine, c["ids"], sink, *mode, chunk=chunk)
    assert rc == E_OK
    assert [len(x) for x in calls] == plan
    assert b"".join(calls) == text
    assert written == len(text)


@pytest.mark.parametrize("mode", [S.TRI, S.SQ, S.SQ_PID], ids=mode_id)
def test_id_offsets_skip_a_prefix(engine, want, mode):
    """id_offsets[0] > 0: the export starts reading the ids there (the header of square mode and every row)."""
    c = S.case("ids")
    engine.upload(*seqio.pack(c["code_list"]))
    calls = []

    def sink(_u, ptr, n):
        calls.append(C.string_at(ptr, n))
        return 0

    rc, written = raw_export(engine, c["ids"], sink, *mode, prefix=b"not,an\nid " * 3 + b"\xff" * 7)
    assert rc == E_OK and b"".join(calls) == want("ids", mode) and written == len(want("ids", mode))
