"""famsa_lcs_nj on the device: the reference's neighbour-joining tree (NeighborJoining<d>::run, -gt nj) pair for pair.

Sources of truth: the committed fixtures (tests/golden/make_nj.py, trees of the reference's own run), the live reference
where oracle/_ref is built, and the restated computeTree (oracle/nj_oracle.c) on the float Transform of the device's own
LCS triangle.

The regimes of the kernel as built (famsa_b200/csrc/tree.cu, k_nj) and the sizes that cross them:
- blocks: ceil(n / 64) blocks of 1024 threads, at most one per SM (the kernel takes 60 registers), so 1 block up to
  n = 64, 2 from n = 65, 3 from n = 129, and 66 for the 4 188-sequence fixture;
- scan rows per warp: the scan runs on all warps but the last (31 per block for one block), so n = 32 gives one row per
  warp and n = 33, 64, 65 give some warps two rows;
- compaction: at the first step with m <= R/2 live rows (R stored), so n = 4 never compacts, n = 6 compacts once at
  m = 3, and n = 2 100 compacts at m = 1 050, 525, 262, 131, 65, 32, 16, 8, 4;
- the s_a chain: one warp sums row a in chunks of 128 slots with one chunk of look-ahead while the other warps scan;
  stored widths R = 128 / 129 / 130 (n = 129, 130, and the compactions of n = 260 at R = 130) put the chain's last chunk
  at 0, 1 and 2 slots; the first step has no chain (n = 2, 3 also have none at their last scan);
- no candidate: every q NaN or >= FLT_MAX returns FAMSA_E_INVALID (n = 2 100 over 20 letters meets it at merge 2 043, the
  ragged4 set at merge 146, sets without any shared residue at the first step)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import famsa_b200
from conftest import GOLDEN, random_set
from famsa_b200 import seqio
from oracle import pyoracle as P
import nj_oracle as N
import upgma_cases as U
from test_slink_gpu import live_sets
from cpp_build import build_cpp

pytestmark = pytest.mark.gpu

OK, E_INVALID, E_STATE = 0, 1, 4
need_ref = pytest.mark.skipif(not P.have("ref_nj"), reason="oracle/_ref/libfamsa_ref_nj.so not built")


def upload_letters(engine, letters):
    engine.upload(*seqio.pack([seqio.encode(s) for s in letters]))


def check_against_restatement(engine, kind, lens):
    """The device's tree against the restatement on the float Transform of the LCS triangle the device computes for the
    uploaded set.  Where the restatement meets a step without a candidate (as random sets of short sequences can, late in
    the run), the device returns FAMSA_E_INVALID after the same merges."""
    rc, want = N.restated(P.transform_triangle(kind, engine.triangle(dtype=np.uint32), lens), len(lens))
    out = np.zeros((len(lens) - 1, 2), dtype=np.int32)
    got = engine.lib.famsa_lcs_nj(engine.h, kind, out.ctypes.data_as(C.c_void_p))
    assert got == (E_INVALID if rc else OK), f"kind {kind}: status {got}, restatement {rc}"
    assert np.array_equal(out[:len(want)], want), f"kind {kind}"


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("fixture", ["adeno_nj_tree.npz", "hemopexin_nj.npz"])
def test_fixtures(engine, fixture, kind):
    """adeno_fiber (242 sequences, 4 blocks) and the hemopexin set (4 188 sequences, 66 blocks, 10 compactions)."""
    z = np.load(os.path.join(GOLDEN, fixture))
    upload_letters(engine, [str(s) for s in z["seqs"]])
    assert np.array_equal(engine.nj(kind), z[f"tree{kind}"])
    total, main, pairs = engine.last_timing()
    n = len(z["seqs"])
    assert pairs == n * (n - 1) // 2 and total >= main > 0


def nj_live_sets():
    out = {k: v for k, v in live_sets().items() if k != "n1"}
    rng = np.random.default_rng(81)
    out["n4"] = [seqio.decode(c) for c in sorted(random_set(rng, 4, 5, 60), key=lambda c: -len(c))]
    # one sequence without a residue in common with the others: each of its distances is FLT_MAX, its sum overflows to
    # +inf, and every q of two ordinary sequences is -inf; the first such pair wins
    ordinary = [seqio.decode(c) for c in random_set(rng, 40, 20, 80, alphabet=10, with_specials=False)]
    out["minus_inf"] = sorted(ordinary + ["W" * 30], key=lambda s: -len(s))
    for name in ("carry_sorted", "carry_shuffled"):
        out[name] = U.letters_of(*U.sequence_set(name))
    return out


LIVE = ["family700", "adeno", "ragged3", "twice", "n2", "n3", "n4", "n33", "minus_inf", "carry_sorted",
        "carry_shuffled"]


@need_ref
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("case", LIVE)
def test_against_live_reference(engine, case, kind):
    letters = nj_live_sets()[case]
    upload_letters(engine, letters)
    got = engine.nj(kind)
    assert got.shape == (len(letters) - 1, 2)
    want, _ = N.ref_tree(letters, kind)
    assert np.array_equal(got, want)


@need_ref
@pytest.mark.parametrize("kind", [0, 1])
def test_late_step_without_candidate(engine, kind):
    """ragged4 of test_slink_gpu.live_sets (150 sequences of 1..90 residues over 4 letters): after 146 merges every q
    left is NaN or >= FLT_MAX, and the reference's merge 146 is a cluster joined with itself.  The device returns
    FAMSA_E_INVALID, and the context answers the next call."""
    letters = live_sets()["ragged4"]
    want, _ = N.ref_tree(letters, kind)
    assert want[146, 0] == want[146, 1]
    upload_letters(engine, letters)
    out = np.zeros((len(letters) - 1, 2), dtype=np.int32)
    assert engine.lib.famsa_lcs_nj(engine.h, kind, out.ctypes.data_as(C.c_void_p)) == E_INVALID
    assert b"famsa_lcs_nj" in engine.lib.famsa_last_error()
    assert np.array_equal(out[:146], want[:146])             # the merges before it are the reference's
    z = np.load(os.path.join(GOLDEN, "adeno_nj_tree.npz"))
    upload_letters(engine, [str(s) for s in z["seqs"]])
    assert np.array_equal(engine.nj(kind), z[f"tree{kind}"])


def boundary_set(n, alphabet, seed):
    """n sequences in FAMSA's order; a small alphabet gives many equal distances, hence equal q values."""
    rng = np.random.default_rng(seed)
    cl = U.famsa_sorted(random_set(rng, n, 8, 40, alphabet=alphabet, with_specials=False))
    return seqio.pack(cl)


BOUNDARY_N = [2, 3, 4, 5, 6, 31, 32, 33, 64, 65, 128, 129, 130, 131, 260, 2100]


@pytest.mark.parametrize("alphabet", [3, 20])
@pytest.mark.parametrize("n", BOUNDARY_N)
def test_restatement_on_device_triangle(engine, n, alphabet):
    """Every regime boundary of the module docstring, against the restatement on the device's own triangle."""
    codes, offsets, lens = boundary_set(n, alphabet, 1000 + n)
    engine.upload(codes, offsets, lens)
    for kind in (0, 1):
        check_against_restatement(engine, kind, lens)


def test_duplicates_only(engine):
    """Every sequence four times: the distance triangle is full of zeros and ties across rows and blocks."""
    rng = np.random.default_rng(82)
    base = random_set(rng, 40, 10, 50, alphabet=4, with_specials=False)
    codes, offsets, lens = seqio.pack(U.famsa_sorted([c.copy() for c in base for _ in range(4)]))
    engine.upload(codes, offsets, lens)
    for kind in (0, 1):
        check_against_restatement(engine, kind, lens)


@pytest.mark.parametrize("n", [4, 5, 20])
def test_all_residue_disjoint_then_reuse(engine, n):
    """No two sequences share a residue: the first step has no candidate (q = inf - inf = NaN everywhere).  The call
    returns FAMSA_E_INVALID with a message, and the next call on the same context succeeds."""
    upload_letters(engine, ["ACDEFGHIKLMNPQRSTVWY"[k] * (n - k) for k in range(n)])
    out = np.zeros((n - 1, 2), dtype=np.int32)
    assert engine.lib.famsa_lcs_nj(engine.h, 0, out.ctypes.data_as(C.c_void_p)) == E_INVALID
    assert b"famsa_lcs_nj" in engine.lib.famsa_last_error()
    z = np.load(os.path.join(GOLDEN, "adeno_nj_tree.npz"))
    upload_letters(engine, [str(s) for s in z["seqs"]])
    assert np.array_equal(engine.nj(1), z["tree1"])


def test_abi_contract():
    eng = famsa_b200.Engine(0)
    lib, h = eng.lib, eng.h
    out = np.zeros(64, np.int32)
    p = out.ctypes.data_as(C.c_void_p)
    try:
        assert lib.famsa_lcs_nj(h, 0, p) == E_STATE                        # nothing uploaded
        assert lib.famsa_last_error()
        assert lib.famsa_lcs_nj(None, 0, p) == E_INVALID
        upload_letters(eng, ["ACDEFG"])
        assert lib.famsa_lcs_nj(h, 0, p) == E_STATE and lib.famsa_last_error()      # one sequence
        letters = ["ACDEFGHIK", "ACDEFGHI", "ACDFGHI", "KLMN"]
        upload_letters(eng, letters)
        for kind in (-1, 2, 3):
            assert lib.famsa_lcs_nj(h, kind, p) == E_INVALID and lib.famsa_last_error()
        assert lib.famsa_lcs_nj(h, 0, None) == E_INVALID and lib.famsa_last_error()
        assert lib.famsa_lcs_nj(h, 1, p) == OK
        assert eng.last_timing()[2] == 6
        want = eng.nj(1)
        assert np.array_equal(out[:6].reshape(3, 2), want)
    finally:
        eng.close()


def test_host_mirror_nj_runs(engine, tmp_path):
    dump = tmp_path / "nj.txt"
    r = subprocess.run([build_cpp("test_host_nj", tmp_path, famsa=True), str(dump)], capture_output=True, text=True)
    assert r.returncode == 0 and "host mirror nj ok" in r.stdout, r.stdout + r.stderr
    lines = dump.read_text().split("\n")
    n = 200
    seqs = [np.frombuffer(s.encode(), np.uint8).astype(np.int8) - ord("0") for s in lines[:n]]
    merges = np.array([[int(x) for x in ln.split()] for ln in lines[n:] if ln], dtype=np.int32)
    engine.upload(*seqio.pack(seqs))
    assert np.array_equal(engine.nj(0), merges)
