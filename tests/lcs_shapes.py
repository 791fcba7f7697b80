"""Sequence sets that reach every instantiation of the LCS tile kernel, and plain references to check them against.

k_lcs_tile<NL> (famsa_b200/csrc/lcs.cu) is compiled for NL = 1..32 and 36, 40, ..., 64 32-bit limbs.  Each NL has its own
load shape (NL / 4 LDS.128 quads and a 0..3-limb tail), carry-chain length and shared-memory size, and the NL of a launch
is chosen per 32-sequence mask group from the group's longest member.  An arbitrary test set therefore reaches only a few
instantiations, by accident.  The sets here reach each one on purpose:

  sweep_set(nl)   two full groups whose longest members sit at both ends of nl's length range, and a partial third group
                  of shorter sequences down to length 0;
  carry_set(nl)   a row whose 'A' mask is nearly all ones in every limb, against A-rich sequences, so that a carry crosses
                  every limb boundary (lcs_dropped_limb_carry shows that dropping any one of them changes a result);
  quirk_set()     rows with an aligned 64-run of one residue (the reference's dropped-carry corner, recomputed by the exact
                  kernels) and near misses that must stay on the tile kernel, mixed with ordinary rows.

true_lcs is the plain O(mn) dynamic programme: an independent reference, not another bit-parallel restatement.
"""
from __future__ import annotations

import functools

import numpy as np

from famsa_b200 import seqio

A, C = 0, 4                              # residue codes of 'A' and 'C' in seqio.ALPHABET

# the limb counts launch_tile_nl instantiates k_lcs_tile for
INSTANTIATED = tuple(range(1, 33)) + tuple(range(36, 65, 4))


def tile_nl(max_len: int) -> int:
    """nl_for_len in lcs.cu: the limb count of a mask group whose longest member has max_len residues; 0 = the group is
    too long for the tile kernel (above 2048 residues) and goes to the exact kernels."""
    req = max(1, (int(max_len) + 31) // 32)
    if req <= 32:
        return req
    if req <= 64:
        return (req + 3) // 4 * 4
    return 0


def nl_range(nl: int) -> tuple[int, int]:
    """(shortest, longest) length whose group gets nl limbs, e.g. (1025, 1152) for 36."""
    lo = 32 * (nl - 1) + 1 if nl <= 32 else 32 * (nl - 4) + 1
    return lo, 32 * nl


def true_lcs(a, b) -> int:
    """LCS length by the row-wise DP, vectorised over the longer sequence.  Codes 20..23 (B Z X *) never match."""
    a = np.asarray(a, dtype=np.int64)
    b = np.asarray(b, dtype=np.int64)
    if len(a) < len(b):
        a, b = b, a
    prev = np.zeros(len(a) + 1, dtype=np.int64)
    eq = {}
    for c in b:
        c = int(c)
        if not 0 <= c < seqio.N_VALID:
            continue
        if c not in eq:
            eq[c] = a == c
        cur = np.zeros_like(prev)
        cur[1:] = np.maximum.accumulate(np.maximum(prev[1:], (prev[:-1] + 1) * eq[c]))
        prev = cur
    return int(prev[-1])


def quirky(codes) -> bool:
    """k_quirky in lcs.cu: some aligned 64-residue word is one matching residue throughout (an all-ones mask word)."""
    c = np.asarray(codes)
    k = len(c) // 64
    if k == 0:
        return False
    w = c[:64 * k].reshape(k, 64)
    return bool(np.any((w == w[:, :1]).all(axis=1) & (w[:, 0] >= 0) & (w[:, 0] < seqio.N_VALID)))


def lcs_dropped_limb_carry(row, col, nl: int, b: int) -> int:
    """The tile kernel's recurrence X' = (X + (X & M)) | (X & ~M) on 32 * nl bits with `row` supplying the masks and
    `col` streamed, except that the carry from limb b-1 into limb b is dropped (b = 0: nothing is dropped, i.e. the true
    LCS).  Python ints hold the whole bit-vector."""
    nbits = 32 * nl
    assert len(row) <= nbits and 0 <= b < nl
    full = (1 << nbits) - 1
    masks = [0] * seqio.N_VALID
    for p, c in enumerate(row):
        if 0 <= c < seqio.N_VALID:
            masks[int(c)] |= 1 << p
    sh = 32 * b
    lo = (1 << sh) - 1
    x = full
    for c in col:
        if not 0 <= c < seqio.N_VALID:
            continue
        m = masks[int(c)]
        tb = x & m
        if b:
            s = (((x & lo) + (tb & lo)) & lo) | (((x >> sh) + (tb >> sh)) << sh)
        else:
            s = x + tb
        x = (s | (x & ~m)) & full
    return nbits - x.bit_count()


def _residues(rng, length: int, alphabet: int) -> np.ndarray:
    c = rng.integers(0, alphabet, size=length).astype(np.int8)
    k = rng.random(length) < 0.03
    c[k] = rng.integers(20, 24, size=int(k.sum())).astype(np.int8)
    return c


def _shapes(code_list, seed: int) -> dict:
    """The set in a shuffled caller order (unsorted upload) and in the library's length-descending order."""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(code_list))
    unsorted = [code_list[i] for i in order]
    srt = sorted(unsorted, key=lambda c: -len(c))                       # stable, as lcs_upload orders
    return dict(unsorted=unsorted, sorted=srt)


def group_nls(lens) -> list[int]:
    """The limb count of every mask group, in group order."""
    s = np.sort(np.asarray(lens, dtype=np.int64))[::-1]
    return [tile_nl(int(s[g])) for g in range(0, len(s), 32)]


@functools.lru_cache(maxsize=None)
def sweep_set(nl: int) -> dict:
    """Two full groups with nl limbs, their longest members the longest and the shortest length nl covers, and a
    partial group of shorter sequences.  Lengths hi-1 .. hi-16 cover every residue mod 4 and mod 16; half the sequences
    use 4 residues (long common subsequences, long carry runs), half all 20; 3 % are B/Z/X/*."""
    rng = np.random.default_rng(1000 + nl)
    lo, hi = nl_range(nl)
    half = lo // 2
    g0 = [hi] + [hi - k for k in range(1, 17)] + [int(x) for x in rng.integers(lo, hi + 1, size=15)]
    g1 = [lo] + [int(x) for x in rng.integers(half, lo + 1, size=30)] + [half]
    k = int(rng.integers(1, 32))                                        # n % 32 != 0: the last group is partial
    g2 = [0] + [int(x) for x in rng.integers(0, half + 1, size=k - 1)]
    cl = [_residues(rng, ln, 4 if rng.random() < 0.5 else 20) for ln in g0 + g1 + g2]
    return _shapes(cl, 1500 + nl)


def _a_rich(rng, length: int) -> np.ndarray:
    """Mostly 'A', the rest any code (C and B/Z/X/* included), and no aligned 64-word of 'A' only."""
    c = np.where(rng.random(length) < 0.75, A, rng.integers(1, 24, size=length)).astype(np.int8)
    for w in range(length // 64):
        if np.all(c[64 * w:64 * w + 64] == A):
            c[64 * w + int(rng.integers(0, 64))] = C
    return c


def carry_row(length: int) -> np.ndarray:
    """'A' everywhere except 'C' at every 64-aligned position: the 'A' mask is all ones but for bit 0 of every 64-bit
    word, so the row is not flagged and stays on the tile kernel, and an 'A' carry runs through every limb boundary."""
    r = np.full(length, A, dtype=np.int8)
    r[::64] = C
    return r


@functools.lru_cache(maxsize=None)
def carry_set(nl: int) -> dict:
    """carry_row of nearly 32 * nl residues (its group gets nl limbs), 6 longer A-rich sequences (streamed against it in
    the triangle too), and A-rich sequences of assorted lengths including short runs of 'A' only.  `row` = the carry
    row's index in each order."""
    assert nl >= 2
    rng = np.random.default_rng(2000 + nl)
    hi = nl_range(nl)[1]
    ln = hi - 8 - int(rng.integers(0, 9))
    row = carry_row(ln)
    longer = [_a_rich(rng, int(x)) for x in [hi] + list(rng.integers(ln + 1, hi + 1, size=5))]
    pure = [np.full(x, A, dtype=np.int8) for x in (1, 2, 3, 7, 33, 63)]
    shorter = [_a_rich(rng, int(x)) for x in list(rng.integers(1, ln + 1, size=24)) + [ln // 2, min(64, ln), min(65, ln), 5]]
    cl = longer + [row] + pure + shorter
    out = _shapes(cl, 2500 + nl)
    out["row"] = {k: next(i for i, c in enumerate(v) if c is row) for k, v in out.items()}
    return out


def _run(rng, length: int, start: int, run: int, code: int, alphabet: int = 4) -> np.ndarray:
    """Random residues over `alphabet` (which includes 'A') with residues [start, start + run) set to `code`."""
    c = rng.integers(0, alphabet, size=length).astype(np.int8)
    c[start:start + run] = code
    return c


@functools.lru_cache(maxsize=None)
def quirk_set() -> dict:
    """Rows with an aligned 64-run (flagged) and near misses (not flagged), among ordinary rows of 0..1800 residues and
    A- and C-led columns that make a dropped carry show.  `flagged`, `near` and `word0` give the indices of those rows
    in each order."""
    rng = np.random.default_rng(3001)
    flagged = [
        _run(rng, 200, 0, 64, A),                         # word 0 (no carry enters word 0: flagged, but never differs)
        _run(rng, 3 * 64 + 40, 128, 64, A),               # the last full word of a 232-residue row
        _run(rng, 300, 64, 128, A),                       # a 128-run
        _run(rng, 4 * 64, 64, 64, A),                     # a row of exactly 64k residues
        _run(rng, 1500, 17 * 64, 64, A),                  # a long row: 24 words in the exact kernels
        _run(rng, 350, 128, 64, C, alphabet=6),           # another residue
    ]
    near = []
    for start in (63, 65, 127, 129):                      # runs starting at 64k +- 1
        c = _run(rng, 260, start, 64, A)
        c[start + 64 if start % 64 == 63 else start - 1] = C          # the aligned word the run overlaps is not all 'A'
        near.append(c)
    c = _run(rng, 200, 64, 63, A); c[127] = C; near.append(c)             # an aligned 63-run
    near.append(_run(rng, 3 * 64 + 40, 192, 40, A))                        # a run filling a partial last word
    for code in (20, 21, 22, 23):                                          # aligned 64-runs of B, Z, X, *
        near.append(_run(rng, 190, 64, 64, code))
    ordinary = [_residues(rng, int(x), 4) for x in rng.integers(1, 400, size=40)]
    ordinary += [_residues(rng, int(x), 20) for x in (1800, 1400, 1100, 700)]
    ordinary += [np.full(1, A, np.int8), np.array([A, C], np.int8), np.full(5, A, np.int8), np.zeros(0, np.int8)]
    ordinary += [np.concatenate([[lead], _residues(rng, int(x), 4)]).astype(np.int8) for lead in (A, C) for x in (10, 90, 250)]
    out = _shapes(flagged + near + ordinary, 3002)
    ids = {k: {id(c): i for i, c in enumerate(v)} for k, v in out.items()}
    out["flagged"] = {k: sorted(v[id(c)] for c in flagged) for k, v in ids.items()}
    out["near"] = {k: sorted(v[id(c)] for c in near) for k, v in ids.items()}
    out["word0"] = {k: v[id(flagged[0])] for k, v in ids.items()}
    return out
