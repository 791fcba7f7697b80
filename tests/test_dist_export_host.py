"""CPU tests of the -dist_export text: the restatement in dist_export_oracle.py against the reference's four
test/adeno_fiber files and against the reference's own formatter and DistanceCalculator (where oracle/_ref is built)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
import dist_export_oracle as O
from oracle import pyoracle

MODES = (("dist", False, False), ("pid", False, True), ("dist_sq", True, False), ("pid_sq", True, True))

# float value -> what Double2PChar((double) v, 6) prints on x86-64
TABLE = [
    (0.674734294, b"0.674734"),
    (12.5, b"12.500000"),
    (1.99999964, b"1.000000"),           # the fraction wraps to b = 2000000
    (0.999999702, b"0.000000"),
    (np.inf, b"9223372036854775808.223372036854775808"),    # cvttsd2si: out of range -> INT64_MIN
]


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "adeno_dist_export.npz"))
    lz = np.load(os.path.join(GOLDEN, "adeno_fiber_lcs.npz"))
    from famsa_b200 import seqio
    seqs = [str(s) for s in lz["seqs"]]
    return dict(ids=[str(i) for i in z["ids"]], seqs=seqs, lcs=lz["lcs"],
                lens=np.array([len(seqio.encode(s)) for s in seqs]),
                files={k: z[k].tobytes() for k, _, _ in MODES})


def wrapping_floats() -> np.ndarray:
    """Every float in [0, 8) whose printed fraction wraps (b = 2000000): the ones just below 1, 2, ..., 8."""
    out = []
    for m in range(1, 9):
        v = np.float32(m)
        while True:
            v = np.nextafter(v, np.float32(0))
            if O.split_values(np.array([v]))[1][0] != 2000000:
                break
            out.append(v)
    return np.array(out, dtype=np.float32)


def random_floats(n=1_000_000, seed=5) -> np.ndarray:
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 0x4b000000, size=n // 2, dtype=np.uint32).view(np.float32)     # [0, 2^23): every exponent
    small = (rng.random(n - n // 2) * 20).astype(np.float32)                                 # the range distances live in
    return np.concatenate([bits, small])


@pytest.mark.parametrize("name,square,pid", MODES)
def test_oracle_rebuilds_golden(golden, name, square, pid):
    got = O.csv_from_lcs(golden["lcs"], golden["lens"], golden["ids"], 0, square, pid)
    assert got == golden["files"][name]


def test_oracle_formatter_table():
    assert O.num2str(np.array([v for v, _ in TABLE], dtype=np.float32)) == [t for _, t in TABLE]
    assert O.num2str(np.array([np.nan], dtype=np.float32)) == [TABLE[-1][1]]


def test_wrapping_floats():
    w = wrapping_floats()
    assert len(w) == 20
    a, _ = O.split_values(w)
    assert all(s == b"%d.000000" % x for s, x in zip(O.num2str(w), a.tolist()))


needs_ref = pytest.mark.skipif(not pyoracle.have("ref_dist"), reason="oracle/_ref/libfamsa_ref_dist.so not built")


@needs_ref
def test_formatter_equals_reference_num2str():
    for vals in (np.array([v for v, _ in TABLE] + [np.nan, 0.0, 1.0, 7.9999995], dtype=np.float32), wrapping_floats(),
                 random_floats()):
        assert O.num2str(vals) == O.ref_num2str(vals)


@needs_ref
@pytest.mark.parametrize("name,square,pid", MODES)
def test_reference_distance_calculator_rebuilds_golden(golden, name, square, pid):
    assert O.ref_dist_export(golden["seqs"], golden["ids"], 0, square, pid, n_threads=4) == golden["files"][name]
