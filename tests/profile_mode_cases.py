"""Cases of FAMSA's profile-profile mode (famsa in1 in2 out): pairs of finished alignments as text, with all-gap columns,
and what the reference computes for them through oracle/_ref (RefDp: profile() of each side as CFAMSA::alignProfiles
builds it, align(..., 1), the merged profile's rows in data order and its tables)."""
from __future__ import annotations

import os

import numpy as np

from famsa_b200 import seqio

AA = "ARNDCQEGHILKMFPSTWYV"


def alignment(n: int, width: int, rng, allgap=(), gap_frac: float = 0.25, lower: float = 0.0, extra: float = 0.0) -> list[str]:
    """n text rows of `width` columns: a consensus with substitutions and gap runs; the columns in `allgap` (0-based,
    negative from the end) hold no residue; every row keeps one.  n == 1 gives an ungapped row (a one-row alignment with
    a gap is not a valid input).  lower / extra: share of residues in lower case / replaced by a non-standard letter."""
    if n == 1:
        allgap, gap_frac = (), 0.0
    gapcols = np.zeros(width, dtype=bool)
    for c in allgap:
        gapcols[c] = True
    cons = rng.integers(0, 20, size=width)
    codes = np.where(rng.random((n, width)) < 0.3, rng.integers(0, 20, size=(n, width)), cons[None, :])
    gap = rng.random((n, width)) < gap_frac
    for r in range(n):
        a = int(rng.integers(0, width)); gap[r, a:a + int(rng.integers(1, 12))] = True
    gap |= gapcols[None, :]
    if n == 1:
        gap[:] = False
    free = np.flatnonzero(~gapcols)
    for r in range(n):
        if gap[r].all():
            gap[r, free[int(rng.integers(0, len(free)))]] = False
    letters = np.frombuffer(AA.encode(), dtype=np.uint8)[codes]
    extra_at = rng.random((n, width)) < extra
    letters[extra_at] = np.frombuffer(b"JOU", dtype=np.uint8)[rng.integers(0, 3, size=int(extra_at.sum()))]
    letters[rng.random((n, width)) < lower] += 32
    letters[gap] = ord("-")
    return [r.tobytes().decode() for r in letters]


def encode(rows: list[str]) -> np.ndarray:
    return np.stack([seqio.encode_gapped(r) for r in rows])


def as_gap_neg(codes: np.ndarray) -> np.ndarray:
    """famsa_b200.profiles.tables_from_rows' input: gaps as -1."""
    a = codes.astype(np.int16)
    a[a == seqio.GAP] = -1
    return a


def normalise(row: str) -> str:
    """A text row as the reference's harness prints it: upper case, non-standard letters as X."""
    return "".join(c if c == "-" else seqio.ALPHABET[int(seqio.encode(c)[0])] for c in row)


def reference_gaps(n_seqs: int):
    """(gaps, score matrix) after the reference's adjustParams(n_seqs)."""
    from oracle import pyoracle
    dp = pyoracle.RefDp(n_seqs)
    g, sm = dp.gaps(), dp.score_matrix()
    dp.close()
    return g, sm


def reference_merge(rows1: list[str], rows2: list[str], gaps=None, matrix_type: int = 2) -> dict:
    """The reference's CFAMSA::alignProfiles merge (unbanded, one thread) of two alignments.  gaps None: adjustParams'
    rescaled costs for n1 + n2 sequences.  Returns dict(gaps, score_matrix, t1, t2 (tables of the two inputs), total,
    order (input index of each merged row), rows (upper case), merged (tables of the merged profile))."""
    from oracle import pyoracle
    n1, n2 = len(rows1), len(rows2)
    dp = pyoracle.RefDp(n1 + n2, matrix_type)
    try:
        if gaps is not None:
            dp.set_gaps(gaps)
        g, sm = dp.gaps(), dp.score_matrix()
        p1 = dp.profile([r.upper() for r in rows1], list(range(n1)))
        p2 = dp.profile([r.upper() for r in rows2], list(range(n1, n1 + n2)))
        t1, t2 = dp.tables(p1), dp.tables(p2)
        m, total = dp.align(p1, p2, 1)
        rows = dp.rows(m)
        merged = dp.tables(m)
        dp.free(m)
    finally:
        dp.close()
    return dict(gaps=g, score_matrix=sm, t1=t1, t2=t2, total=total, order=list(rows.keys()), rows=list(rows.values()),
                merged=merged)


def case_matrix(seed: int = 5):
    """(name, rows1, rows2): all-gap columns at column 1, inside, at the last column the merge sees and at the very last
    column, and in runs; one-row sides on either side and profile-profile pairs of both orientations.  Two one-row inputs
    are one_by_one(): the reference's harness aborts on them."""
    rng = np.random.default_rng(seed)
    out = []
    W1, W2 = 40, 33
    for name, ag in [("first", (0,)), ("inner", (7, 19)), ("last_seen", (-2,)), ("last", (-1,)), ("run", (10, 11, 12, 13)),
                     ("ends", (0, 1, -2, -1))]:
        out.append((f"pp_{name}", alignment(9, W1, rng, ag, lower=0.1, extra=0.05), alignment(14, W2, rng, ag, lower=0.1)))
    out.append(("pp_swap", alignment(30, 25, rng, (3,)), alignment(4, 60, rng, (0, -1))))
    out.append(("pp_wide_few", alignment(3, 80, rng, (5, 6), gap_frac=0.5), alignment(25, 20, rng, (-1,))))
    out.append(("seq_left", alignment(1, 30, rng), alignment(12, 35, rng, (0, 17, -1))))
    out.append(("seq_right", alignment(10, 35, rng, (4, -2)), alignment(1, 28, rng)))
    out.append(("two_rows", alignment(2, 12, rng, (0, 5)), alignment(2, 9, rng, (-1,))))
    return out


def one_by_one(seed: int = 6):
    """Two one-row alignments (AlignSeqSeq)."""
    rng = np.random.default_rng(seed)
    return alignment(1, 22, rng, lower=0.3), alignment(1, 26, rng)


def orientation_cases():
    """(name, rows1, rows2) whose ProfProf orientation turns on the set-aside last column: the reference counts its
    residue counters in get_num_of_non_zeros (the counters have gapped_size + 1 columns), so the orientation differs from
    the one the tables cut at width - 1 give.  Both orientations occur."""
    out = [("boundary_pair", ["AAC", "AAD"], ["ARA", "RRA"])]
    for seed in (11, 14, 17, 61, 82, 93):
        rng = np.random.default_rng(1000 + seed)
        n1, n2 = int(rng.integers(2, 6)), int(rng.integers(2, 6))
        w1, w2 = int(rng.integers(3, 9)), int(rng.integers(3, 9))
        out.append((f"boundary_{seed}", alignment(n1, w1, rng, gap_frac=0.2), alignment(n2, w2, rng, gap_frac=0.2)))
    return out


def reference_swapped(ref: dict, n1: int) -> bool:
    """famsa_dp_result.swapped of the reference's merge, from its row order: the column profile's rows come first."""
    return ref["order"][0] < n1


def text_orientation(rows1: list[str], rows2: list[str]) -> bool:
    """The reference's ProfProf orientation for two profiles of rows read as text, restated: get_num_of_non_zeros over
    all gapped_size + 1 counter columns (the set-aside last column holds its residues only) times the other's width - 1;
    True when the DP's rows are rows2 (profile.cpp:283)."""
    from famsa_b200 import profiles
    nz = []
    for rows in (rows1, rows2):
        codes = as_gap_neg(encode(rows))
        _, cnt, _ = profiles.tables_from_rows(codes, np.zeros((24, 24), np.int64), (0, 0, 0, 0))
        last = codes[:, -1]
        nz.append(int(np.count_nonzero(cnt[:-1])) + len(set(int(x) for x in last[last >= 0])))
    w1, w2 = len(rows1[0]) - 1, len(rows2[0]) - 1
    return not nz[0] * w2 < nz[1] * w1


def host_mirror_input(path) -> None:
    """The golden as the C++ mirror test (tests/cpp/test_host_profiles.cpp) reads it: gaps, score matrix, both inputs,
    upgma.pp.fasta's rows."""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adeno_pp_rows.npz"))
    lines = [" ".join(str(int(x)) for x in z["gaps"]), " ".join(str(int(x)) for x in z["score_matrix"].ravel())]
    for key in ("rows1", "rows2", "gold_rows"):
        lines += [str(len(z[key]))] + [str(r) for r in z[key]]
    open(path, "w").write("\n".join(lines) + "\n")
