"""famsa_lcs_slink on the device: the reference's single-linkage tree (SingleLinkage<d>::run, -gt slink) pair for pair,
from the committed fixtures (tests/golden/make_slink.py) and, where oracle/_ref is built, from the live reference; both
MST engines (the Boruvka rounds and the sequential loop, forced with FAMSA_PRIM_SEQUENTIAL); the 124 140-sequence LRR
set, whose float64 triangle does not fit; and the C ABI's return codes."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import famsa_b200
from famsa_b200 import seqio
from conftest import GOLDEN, random_set
from oracle import pyoracle
import slink_oracle as S
from cpp_build import build_cpp

pytestmark = pytest.mark.gpu

OK, E_INVALID, E_STATE = 0, 1, 4
need_ref = pytest.mark.skipif(not pyoracle.have("ref_slink"), reason="oracle/_ref/libfamsa_ref_slink.so not built")


def engine_kinds(monkeypatch, sequential):
    if sequential:
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")


def upload_letters(engine, letters):
    engine.upload(*seqio.pack([seqio.encode(s) for s in letters]))


@pytest.mark.parametrize("sequential", [False, True])
def test_golden_adeno_tree(engine, monkeypatch, sequential):
    """test/adeno_fiber in FAMSA's order: the reference's tree, whose clades are those of slink.dnd."""
    engine_kinds(monkeypatch, sequential)
    z = np.load(os.path.join(GOLDEN, "adeno_slink_tree.npz"))
    upload_letters(engine, [str(s) for s in z["seqs"]])
    assert np.array_equal(engine.slink(0), z["tree"])
    total, main, pairs = engine.last_timing()
    n = len(z["seqs"])
    assert pairs == n * (n - 1) // 2 and total >= main > 0


@pytest.mark.parametrize("sequential", [False, True])
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("order", ["unsorted", "sorted"])
def test_dropped_carry_case(engine, monkeypatch, sequential, kind, order):
    """slink_pruning_case.npz: flagged sequences (64-residue runs, LCS above the shorter length when they are the row)
    next to short ones.  In the unsorted order the loop with MSTPrim's lower-bound skip would lose an edge SLINK keeps."""
    engine_kinds(monkeypatch, sequential)
    z = np.load(os.path.join(GOLDEN, "slink_pruning_case.npz"))
    pre = "" if order == "unsorted" else "sorted_"
    upload_letters(engine, [str(s) for s in z[pre + "seqs"]])
    assert np.array_equal(engine.slink(kind), z[f"{pre}tree{kind}"])


def live_sets():
    out = {}
    codes, offsets, lens = seqio.synth_family(700, 130, seed=61)
    out["family700"] = [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(offsets, lens)]
    z = np.load(os.path.join(GOLDEN, "adeno_slink_tree.npz"))
    out["adeno"] = [str(s) for s in z["seqs"]]
    rng = np.random.default_rng(62)
    for alphabet in (3, 4):
        cl = random_set(rng, 150, 1, 90, alphabet=alphabet)
        cl.sort(key=lambda c: (-len(c), c.tobytes()))
        out[f"ragged{alphabet}"] = [seqio.decode(c) for c in cl]
    twice = [seqio.decode(c) for c in random_set(rng, 60, 20, 200)]
    twice = sorted(twice + twice, key=lambda s: -len(s))
    out["twice"] = twice
    for n in (1, 2, 3, 33):
        out[f"n{n}"] = [seqio.decode(c) for c in sorted(random_set(rng, n, 5, 60), key=lambda c: -len(c))]
    return out


LIVE = ["family700", "adeno", "ragged3", "ragged4", "twice", "n1", "n2", "n3", "n33"]


@need_ref
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", LIVE)
def test_against_live_reference(engine, case, kind):
    letters = live_sets()[case]
    upload_letters(engine, letters)
    got = engine.slink(kind)
    assert got.shape == (len(letters) - 1, 2)
    assert np.array_equal(got, S.ref_slink_tree(letters, kind))


@need_ref
@pytest.mark.parametrize("sequential", [False, True])
@pytest.mark.parametrize("kind", [0, 1])
def test_dropped_carry_against_live_reference(engine, monkeypatch, sequential, kind):
    """Flagged sequences in FAMSA's order and in a shuffled order, with both engines."""
    engine_kinds(monkeypatch, sequential)
    rng = np.random.default_rng(63)
    cl = random_set(rng, 50, 1, 8, alphabet=4)
    for k in range(8):
        run = np.full(64 * (1 + k % 3), k % 4, np.int8)
        cl.append(np.concatenate([random_set(rng, 1, 0, 64 * (k % 2), alphabet=4)[0], run]))
    cl.sort(key=lambda c: (-len(c), c.tobytes()))
    for letters in ([seqio.decode(c) for c in cl], [seqio.decode(cl[i]) for i in rng.permutation(len(cl))]):
        upload_letters(engine, letters)
        assert np.array_equal(engine.slink(kind), S.ref_slink_tree(letters, kind))


def test_boruvka_and_sequential_agree_at_40000(monkeypatch):
    """40 000 sequences: 1.6 GB of LCS triangle and 6.4 GB of float64 distances, many blocks per Boruvka round."""
    codes, offsets, lens = seqio.synth_family(40000, 60, seed=64)
    eng = famsa_b200.Engine()
    try:
        eng.upload(codes, offsets, lens)
        got = eng.slink(0)
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
        want = eng.slink(0)
    finally:
        eng.close()
    assert np.array_equal(got, want)


def test_lrr_falls_back_to_the_sequential_loop(monkeypatch):
    """test/LRR (124 140 sequences, lrr_sl.npz, FAMSA's order): 7.7 G pairs, 15 GB of u16 LCS triangle; the 62 GB of
    float64 distances the Boruvka rounds would need do not fit beside it in 80 GB, so the sequential loop runs: the call
    launches exactly the kernels of a call with FAMSA_PRIM_SEQUENTIAL set (the rounds would add at least four).  The
    tree's CRC is the reference's (lrr_slink.npz), the fall-back leaves no error behind, and the context still answers."""
    z = np.load(os.path.join(GOLDEN, "lrr_sl.npz"))
    seqs = bytes(z["seqs"]).decode().split("\n")
    n = len(seqs)
    eng = famsa_b200.Engine()
    try:
        eng.upload(*seqio.pack([seqio.encode(s) for s in seqs]))
        before = eng.kernel_launches()
        tree = eng.slink(0)
        launches = eng.kernel_launches() - before
        assert eng.lib.famsa_last_error() == b"", "a successful call must not report the fall-back's failed allocation"
        assert eng.last_timing()[2] == n * (n - 1) // 2
        monkeypatch.setenv("FAMSA_PRIM_SEQUENTIAL", "1")
        before = eng.kernel_launches()
        assert np.array_equal(eng.slink(0), tree)
        assert eng.kernel_launches() - before == launches
        monkeypatch.delenv("FAMSA_PRIM_SEQUENTIAL")
        small = np.load(os.path.join(GOLDEN, "adeno_slink_tree.npz"))
        upload_letters(eng, [str(s) for s in small["seqs"]])
        assert np.array_equal(eng.slink(0), small["tree"])
    finally:
        eng.close()
    path = os.path.join(GOLDEN, "lrr_slink.npz")
    if not os.path.exists(path):
        pytest.skip("lrr_slink.npz not generated")
    assert zlib.crc32(np.ascontiguousarray(tree, dtype=np.int32).tobytes()) == int(np.load(path)["tree_crc"][0])


def test_abi_contract():
    eng = famsa_b200.Engine(0)
    lib, h = eng.lib, eng.h
    out = np.zeros(64, np.int32)
    p = out.ctypes.data_as(C.c_void_p)
    try:
        assert lib.famsa_lcs_slink(h, 0, p) == E_STATE                     # nothing uploaded
        assert lib.famsa_last_error()
        assert lib.famsa_lcs_slink(None, 0, p) == E_INVALID
        upload_letters(eng, ["ACDEFG"])
        assert lib.famsa_lcs_slink(h, 0, None) == OK                       # one sequence: no merges, NULL is fine
        assert lib.famsa_lcs_slink(h, 2, p) == E_INVALID
        letters = ["ACDEFGHIK", "ACDEFGHI", "ACDFGHI", "KLMN"]
        upload_letters(eng, letters)
        for kind in (-1, 2, 3):
            assert lib.famsa_lcs_slink(h, kind, p) == E_INVALID and lib.famsa_last_error()
        assert lib.famsa_lcs_slink(h, 0, None) == E_INVALID and lib.famsa_last_error()
        assert lib.famsa_lcs_slink(h, 1, p) == OK
        assert eng.last_timing()[2] == 6
        want = eng.slink(1)
        assert np.array_equal(out[:6].reshape(3, 2), want)
    finally:
        eng.close()


def test_host_mirror_slink_runs(engine, tmp_path):
    dump = tmp_path / "slink.txt"
    r = subprocess.run([build_cpp("test_host_slink", tmp_path, famsa=True), str(dump)], capture_output=True, text=True)
    assert r.returncode == 0 and "host mirror slink ok" in r.stdout, r.stdout + r.stderr
    lines = dump.read_text().split("\n")
    n = 200
    seqs = [np.frombuffer(s.encode(), np.uint8).astype(np.int8) - ord("0") for s in lines[:n]]
    merges = np.array([[int(x) for x in ln.split()] for ln in lines[n:] if ln], dtype=np.int32)
    engine.upload(*seqio.pack(seqs))
    assert np.array_equal(engine.slink(0), merges)
