"""famsa_dist_export on the device: byte equality with the reference's -dist_export files, its DistanceCalculator
(live where oracle/_ref is built, else the restatement in dist_export_oracle.py), the formatter alone, the sink
protocol and the argument checks."""
import ctypes as C
import io
import os

import numpy as np
import pytest

import famsa_b200
from famsa_b200 import seqio
from famsa_b200.binding import WRITE_FN
from conftest import GOLDEN, QUIRK_SEQS, random_set
import dist_export_oracle as O
from test_dist_export_host import MODES, TABLE, wrapping_floats

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE, E_SINK = 1, 4, 6
EXPORT_MODES = [(0, False, False), (1, False, False), (0, False, True), (0, True, False), (1, True, False), (0, True, True)]


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "adeno_dist_export.npz"))
    lz = np.load(os.path.join(GOLDEN, "adeno_fiber_lcs.npz"))
    return dict(ids=[str(i) for i in z["ids"]], code_list=[seqio.encode(str(s)) for s in lz["seqs"]],
                files={k: z[k].tobytes() for k, _, _ in MODES})


@pytest.mark.parametrize("chunk_bytes", [0, 1])
@pytest.mark.parametrize("name,square,pid", MODES)
def test_adeno_goldens(engine, golden, name, square, pid, chunk_bytes):
    """chunk_bytes = 1: every row is a chunk of its own."""
    engine.upload(*seqio.pack(golden["code_list"]))
    assert engine.dist_export(golden["ids"], 0, square, pid, chunk_bytes=chunk_bytes) == golden["files"][name]
    total, main, cells = engine.last_timing()
    n = len(golden["ids"])
    assert cells == (n * n if square else n * (n - 1) // 2) and total >= main > 0


def sets():
    rng = np.random.default_rng(11)
    out = {"ragged": random_set(rng, 40, 1, 2300)}
    quirk = [seqio.encode(s) for s in QUIRK_SEQS]
    for k in range(6):                                         # 64-residue runs at aligned and unaligned starts
        s = random_set(rng, 1, 100, 400)[0]
        at = 64 * int(rng.integers(0, 3)) + (k % 2)
        s[at:at + 64] = int(rng.integers(0, 20))
        quirk.append(s)
    out["quirk"] = quirk + random_set(rng, 20, 1, 300)
    out["all_x"] = [np.full(50, 22, np.int8)] + random_set(rng, 9, 1, 80) + [np.full(3, 20, np.int8)]
    base = random_set(rng, 8, 20, 200)
    out["duplicates"] = base + base[:5] + [base[0]] * 3
    for n in (1, 2, 31, 33, 200):
        out[f"n{n}"] = random_set(rng, n, 1, 500)
    # flagged sequences before and after unflagged ones, and two over-long sequences whose LCS depends on which one is
    # seq0, the flagged one second
    rng = np.random.default_rng(13)
    long_pair = random_set(rng, 2, 2100, 2400, alphabet=4)
    long_pair[1][128:192] = 1
    out["quirk_order"] = (quirk[:2] + random_set(rng, 4, 1, 300) + long_pair[:1] + quirk[2:5] + random_set(rng, 4, 1, 300)
                          + long_pair[1:] + quirk[5:8])
    return out


SETS = sets()


@pytest.mark.parametrize("kind,square,pid", EXPORT_MODES)
@pytest.mark.parametrize("case", sorted(SETS))
def test_equals_reference(engine, case, kind, square, pid):
    code_list = SETS[case]
    ids = [f"{case}_{i}|x y/{len(c)}" for i, c in enumerate(code_list)]
    engine.upload(*seqio.pack(code_list))
    assert engine.dist_export(ids, kind, square, pid, chunk_bytes=4096) == O.expected(code_list, ids, kind, square, pid)


def test_out_file_object(engine, golden):
    engine.upload(*seqio.pack(golden["code_list"]))
    buf = io.BytesIO()
    n = engine.dist_export(golden["ids"], square=True, out=buf, chunk_bytes=65536)
    assert n == len(golden["files"]["dist_sq"]) and buf.getvalue() == golden["files"]["dist_sq"]


def formatter_values():
    lens = np.arange(1, 4097, dtype=np.int64)
    # pairwise identity: lcs / m for every m <= 4096 and lcs <= m
    m = np.repeat(lens, lens + 1)
    lcs = np.concatenate([np.arange(k + 1) for k in lens])
    vals = [lcs.astype(np.float32) / m.astype(np.float32)]
    # the indel distances: every indel count <= 8192 over every lcs <= 512 (double, then rounded to float)
    ind, l = np.meshgrid(np.arange(0, 8193, dtype=np.int64), np.arange(1, 513, dtype=np.int64))
    pw = O.pow075_table(4096)
    vals.append((ind.astype(np.float64) / l).astype(np.float32).ravel())
    vals.append((pw[ind] / l).astype(np.float32).ravel())
    vals.append(np.array([np.inf, np.nan, np.float32(np.nextafter(np.finfo(np.float64).max, 0))], dtype=np.float32))
    vals.append(wrapping_floats())
    vals.append(np.array([v for v, _ in TABLE], dtype=np.float32))
    return np.unique(np.concatenate(vals))


def test_device_formatter(engine):
    v = formatter_values()
    got = engine.debug_format_f32(v).split(b",")[:-1]
    want = O.num2str(v)
    bad = [i for i in range(len(v)) if got[i] != want[i]]
    assert not bad, [(float(v[i]), got[i], want[i]) for i in bad[:5]]
    assert engine.debug_format_f32(np.array([v for v, _ in TABLE], np.float32)) == b"".join(t + b"," for _, t in TABLE)


def raw_export(engine, ids, sink, kind=0, square=0, pid=0, chunk=0, id_blob=True, prefix=b""):
    """famsa_dist_export through the C ABI; the id blob starts with `prefix`, which id_offsets[0] skips."""
    raw = [i.encode() if isinstance(i, str) else bytes(i) for i in ids]
    blob = prefix + b"".join(raw)
    offs = np.full(len(raw) + 1, len(prefix), dtype=np.uint64)
    offs[1:] += np.cumsum([len(i) for i in raw], dtype=np.uint64)
    written = C.c_uint64()
    cb = WRITE_FN(sink)
    rc = engine.lib.famsa_dist_export(engine.h, kind, square, pid, C.c_char_p(blob) if id_blob else None,
                                      offs.ctypes.data, chunk, cb, None, C.byref(written))
    return rc, written.value


def test_failing_sink_stops_and_context_survives(engine, golden):
    engine.upload(*seqio.pack(golden["code_list"]))
    calls = []

    def sink(_u, ptr, n):
        calls.append(C.string_at(ptr, n))
        return 7 if len(calls) == 3 else 0

    rc, written = raw_export(engine, golden["ids"], sink, pid=1, chunk=8192)
    assert rc == E_SINK and len(calls) == 3
    assert written == len(calls[0]) + len(calls[1])
    msg = engine.lib.famsa_last_error().decode()
    assert f"byte offset {written}" in msg, msg
    assert golden["files"]["pid"].startswith(b"".join(calls[:3]))
    # the binding: an exception in the file object's write stops the export and comes back
    class Boom(io.RawIOBase):
        def writable(self):
            return True

        def write(self, b):
            raise OSError("disk full")
    with pytest.raises(OSError, match="disk full"):
        engine.dist_export(golden["ids"], pid=True, out=Boom(), chunk_bytes=8192)
    assert engine.dist_export(golden["ids"], pid=True) == golden["files"]["pid"]


def test_state_and_invalid(engine, golden):
    fresh = famsa_b200.Engine(0)
    try:
        rc, _ = raw_export(fresh, [], lambda u, p, n: 0)
        assert rc == E_STATE
    finally:
        fresh.close()
    codes, offsets, lens = seqio.pack(golden["code_list"])
    engine.upload_sorted(codes, offsets, lens)
    assert raw_export(engine, golden["ids"], lambda u, p, n: 0)[0] == E_STATE
    engine.upload(codes, offsets, lens)
    assert raw_export(engine, golden["ids"], lambda u, p, n: 0, kind=2)[0] == E_INVALID
    assert raw_export(engine, golden["ids"], lambda u, p, n: 0, kind=-1)[0] == E_INVALID
    assert raw_export(engine, golden["ids"], lambda u, p, n: 0, id_blob=False)[0] == E_INVALID
    # kind is ignored with pid
    assert engine.dist_export(golden["ids"], kind=5, pid=True) == golden["files"]["pid"]
