"""Sequence encoding, FASTA reading and the synthetic protein-family generator.

Encoding mirrors the reference's CSequence constructor (src/core/sequence.cpp:17,53-79):
codes 0..23 index "ARNDCQEGHILKMFPSTWYVBZX*", lower case is folded to upper case, '-' is dropped,
anything else becomes UNKNOWN (22).
"""
from __future__ import annotations

import numpy as np

ALPHABET = "ARNDCQEGHILKMFPSTWYVBZX*"
UNKNOWN = 22
N_VALID = 20
GAP = 30                                 # a gap in the rows of a finished alignment (src/core/defs.h)

_LUT = np.full(256, UNKNOWN, dtype=np.int8)
for _i, _ch in enumerate(ALPHABET):
    _LUT[ord(_ch)] = _i
    if _ch.isalpha():
        _LUT[ord(_ch.lower())] = _i      # c > 'Z'  ->  c -= 32   (sequence.cpp:62-68)


def encode(seq: str) -> np.ndarray:
    raw = np.frombuffer(seq.encode("ascii", "replace"), dtype=np.uint8)
    raw = raw[raw != ord("-")]
    return _LUT[raw]


def encode_gapped(row: str) -> np.ndarray:
    """One row of a finished alignment as famsa_prof_put_rows and famsa_prof_refine take it (uint8): '-' -> GAP,
    every other letter as encode() maps it (CGappedSequence's constructor, sequence.cpp:214-272)."""
    raw = np.frombuffer(row.encode("ascii", "replace"), dtype=np.uint8)
    return np.where(raw == ord("-"), GAP, _LUT[raw]).astype(np.uint8)


def decode(codes: np.ndarray) -> str:
    return "".join(ALPHABET[int(c)] for c in codes)


def read_fasta(path: str) -> tuple[list[str], list[str]]:
    ids, seqs, cur = [], [], []
    with open(path) as fh:
        for line in fh:
            line = line.rstrip("\r\n")
            if line.startswith(">"):
                if cur or ids:
                    seqs.append("".join(cur))
                ids.append(line[1:])
                cur = []
            elif line:
                cur.append(line)
    if ids:
        seqs.append("".join(cur))
    return ids, seqs


def pack(code_list: list[np.ndarray]) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Concatenate per-sequence code arrays into (codes int8, offsets uint64, lens uint32)."""
    lens = np.array([len(c) for c in code_list], dtype=np.uint32)
    offsets = np.zeros(len(code_list), dtype=np.uint64)
    if len(code_list) > 1:
        offsets[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    codes = np.concatenate(code_list).astype(np.int8) if code_list else np.zeros(0, np.int8)
    if codes.size == 0:
        codes = np.zeros(1, np.int8)
    return np.ascontiguousarray(codes), offsets, lens


def synth_family(n: int, length: int, seed: int, sub: float = 0.30, dele: float = 0.03,
                 ins: float = 0.03, n_subroots: int = 0, sub_root: float = 0.25,
                 sub_member: float = 0.20, sort_desc: bool = True,
                 chunk: int = 65536) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """SURVEY.md section 8(d) generator: one root of `length` uniform residues over the 20 valid
    amino acids; every member = root with per-site substitution `sub`, deletion `dele`, insertion
    `ins`.  With n_subroots > 0 a two-level family (config C5) is produced.  Returns the packed
    (codes, offsets, lens); with sort_desc the set is in FAMSA's length-descending order
    (msa.cpp:245-256) so it is what the guide-tree stage actually sees."""
    rng = np.random.default_rng(seed)
    root = rng.integers(0, N_VALID, size=length, dtype=np.int8)

    def mutate(parents: np.ndarray, p_sub: float) -> list[np.ndarray]:
        m, L = parents.shape
        out = parents.copy()
        s = rng.random((m, L)) < p_sub
        out[s] = rng.integers(0, N_VALID, size=int(s.sum()), dtype=np.int8)
        keep = rng.random((m, L)) >= dele
        add = rng.random((m, L)) < ins
        add_codes = rng.integers(0, N_VALID, size=(m, L), dtype=np.int8)
        res = []
        for r in range(m):
            # interleave: site (if kept) followed by an inserted residue (if any)
            two = np.stack([out[r], add_codes[r]], axis=1).reshape(-1)
            mask = np.stack([keep[r], add[r]], axis=1).reshape(-1)
            res.append(two[mask])
        return res

    members: list[np.ndarray] = []
    if n_subroots > 0:
        subs = mutate(np.broadcast_to(root, (n_subroots, length)), sub_root)
        sub_len = min(len(s) for s in subs)
        subs_arr = np.stack([s[:sub_len] for s in subs])
        assign = rng.integers(0, n_subroots, size=n)
        for start in range(0, n, chunk):
            idx = assign[start:start + chunk]
            members.extend(mutate(subs_arr[idx], sub_member))
    else:
        for start in range(0, n, chunk):
            m = min(chunk, n - start)
            members.extend(mutate(np.broadcast_to(root, (m, length)), sub))
    if sort_desc:
        order = sorted(range(n), key=lambda i: (-len(members[i]), members[i].tobytes()))
        members = [members[i] for i in order]
    return pack(members)
