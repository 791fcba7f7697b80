"""Shared helpers of the famsa_prof_refine tests: random families, the device path (famsa_prof_align_tree -> host row
assembly -> famsa_prof_refine) and the reference's progressive alignment + RefineAlignment through the harness."""
from __future__ import annotations

import numpy as np

import dp_cases
from famsa_b200 import seqio
from oracle import pyoracle

GAP = 30


def letters(codes: np.ndarray) -> str:
    return "".join(seqio.ALPHABET[int(c)] for c in codes)


def family(n: int, length: int, seed: int) -> list[str]:
    codes, off, lens = seqio.synth_family(n, length, seed=seed)
    return [letters(codes[int(o):int(o) + int(l)]) for o, l in zip(off, lens)]


def to_codes(row: str) -> np.ndarray:
    return np.array([GAP if ch == "-" else seqio.ALPHABET.index(ch) for ch in row], dtype=np.uint8)


def to_letters(row: np.ndarray) -> str:
    return "".join("-" if c == GAP else seqio.ALPHABET[int(c)] for c in row)


def id_order(ids: list[str]) -> list[int]:
    """The order of RefineAlignment's rows: std::sort by CGappedSequence::id, byte-wise (msa_refinement.cpp:116)."""
    return sorted(range(len(ids)), key=lambda i: ids[i].encode())


def scoring(n: int):
    dp = pyoracle.RefDp(n)
    g, sm = dp.gaps(), dp.score_matrix()
    dp.close()
    return g, sm


def device_refine(eng, seqs, merges, gaps, sm, n_refinements=100, flags=0, ids=None):
    """Rows {seq_no: string}, width, total, stats and refined id of the device path."""
    n = len(seqs)
    ids = ids or [f"s{i}" for i in range(n)]
    eng.upload(*seqio.pack([seqio.encode(s) for s in seqs]))
    eng.prof_set_scoring(sm)
    root, res, _ = eng.align_tree(merges, gaps)
    rows = dp_cases.assemble_rows(seqs, merges, res)
    order = id_order(ids)
    arr = np.stack([to_codes(rows[i]) for i in order])
    out, width, total, stats, rid = eng.refine(root, arr, gaps, n_refinements, flags)
    return {i: to_letters(out[k]) for k, i in enumerate(order)}, width, total, stats, rid
