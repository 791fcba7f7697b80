"""Sequence sets that take famsa_dist_export (famsa_b200/csrc/dist_export.cu) past the sizes where its loops repeat, and
a plain restatement of its host chunk planner.

Pass 1 (k_dist_row_bytes) strides one block of kFmtThreads threads over a row's columns; pass 2 (k_dist_format) formats
kFmtTile columns per iteration, each with its own block scan, 16-byte phase of the moving destination and ragged-end
stores, out of a shared-memory stage of kFmtTile * kMaxValueChars + 32 bytes.  The LCS triangle it reads is uint16
below a longest sequence of ELEM_WIDTH_LEN residues and uint32 from there on (ctx.h: elem_bytes()).  The host cuts the
rows into chunks of at most chunk_bytes (a row wider than that is a chunk of its own; 0 = kDefaultChunk).  The cases:

  widths_tri       2 050 short sequences in triangle mode: row r has r columns, so every width 0 .. 2 049 is exported
  widths_sq_<n>    square mode at n = 256, 257, 1 024, 1 025, 2 049 columns (2 049: more text than kDefaultChunk)
  widest           two groups with no residue in common: each group-B row's first tile is kFmtTile cells of +inf text,
                   the widest a value prints (38 characters), starting at every 16-byte phase
  ids              ids of 0 .. 5 000 bytes, UTF-8 and a ','
  wide_elem        a 70 000-residue sequence (uint32 triangle) with flagged and over-long sequences around it;
                   wide_elem_65535 / wide_elem_65536: the two sides of the element-width threshold, each with an LCS
                   equal to its longest sequence
  empty            length-0 sequences first, in the middle and last
"""
from __future__ import annotations

import functools

import numpy as np

from conftest import QUIRK_SEQS, random_set
from famsa_b200 import seqio
import dist_export_oracle as O
import lcs_shapes

# dist_export.cu
K_FMT_THREADS = 256
K_FMT_PER_THREAD = 4
K_FMT_TILE = K_FMT_THREADS * K_FMT_PER_THREAD
K_MAX_VALUE_CHARS = 40
K_DEFAULT_CHUNK = 32 << 20
STAGE_BYTES = K_FMT_TILE * K_MAX_VALUE_CHARS + 32
# ctx.h: the LCS triangle is uint32 once the longest sequence has this many residues
ELEM_WIDTH_LEN = 65536

INF_TEXT = b"9223372036854775808.223372036854775808"      # +inf and NaN

TRI, TRI1, TRI_PID = (0, False, False), (1, False, False), (0, False, True)
SQ, SQ1, SQ_PID = (0, True, False), (1, True, False), (0, True, True)
ALL_MODES = (TRI, TRI1, TRI_PID, SQ, SQ1, SQ_PID)
SQ_WIDTHS = (256, 257, 1024, 1025, 2049)

WIDEST_A, WIDEST_B = 1100, 60
WIDE_LEN = 70000
ID_LENGTHS = (0,) + tuple(range(1, 18)) + (255, 256, 257, 1000, 5000)


# the modes each case is exported in
MODES = {"widths_tri": (TRI, TRI1, TRI_PID),
         **{f"widths_sq_{n}": (SQ,) if n > 2048 else (SQ, SQ_PID) for n in SQ_WIDTHS},
         "widest": (TRI, TRI1, TRI_PID), "ids": ALL_MODES, "wide_elem": ALL_MODES,
         f"wide_elem_{ELEM_WIDTH_LEN - 1}": (TRI, TRI1, SQ_PID), f"wide_elem_{ELEM_WIDTH_LEN}": (TRI, TRI1, SQ_PID),
         "empty": ALL_MODES}


def _case(name, code_list, ids, **claims) -> dict:
    return dict(name=name, code_list=code_list, ids=[i.encode() if isinstance(i, str) else bytes(i) for i in ids],
                modes=MODES[name], claims=claims)


def _short(rng, n: int) -> list[np.ndarray]:
    """n sequences of 5..60 residues over all 20 codes and B/Z/X/*."""
    return random_set(rng, n, 5, 60)


@functools.lru_cache(maxsize=None)
def widths_tri() -> dict:
    cl = _short(np.random.default_rng(4100), 2050)
    return _case("widths_tri", cl, [f"t{i}" for i in range(len(cl))])


@functools.lru_cache(maxsize=None)
def widths_sq(n: int) -> dict:
    cl = _short(np.random.default_rng(4200 + n), n)
    return _case(f"widths_sq_{n}", cl, [f"s{n}_{i}" for i in range(n)])


def _widest_ids(code_list) -> list[str]:
    """Group A's ids, then group B's of 1..16 characters, each chosen so that its row's first value starts at a given
    16-byte phase of a single-chunk triangle export: rows 0-15 and 32-47 of group B take phases 0..15 in kind 0, rows
    16-31 and 48-59 in kind 1.  The row bytes other than the id come from the restated text."""
    codes, offsets, lens = seqio.pack(code_list)
    lcs = O.lcs_square(codes, offsets, lens)
    body = {k: [len(x) + 1 for x in O.csv_from_lcs(lcs, lens, [b""] * len(lens), k).split(b"\n")[:-1]] for k in (0, 1)}
    ids = [f"a{i}" for i in range(WIDEST_A)]
    start = {k: sum(len(ids[r]) + body[k][r] for r in range(WIDEST_A)) for k in (0, 1)}
    for j in range(WIDEST_B):
        k = (j // 16) % 2
        n_id = (j % 16 - start[k] - 1) % 16 or 16
        ids.append((f"B{j}" + "_" * 16)[:n_id])
        for k in (0, 1):
            start[k] += n_id + body[k][WIDEST_A + j]
    return ids


@functools.lru_cache(maxsize=None)
def widest() -> dict:
    """WIDEST_A sequences over residue codes 0..9, then WIDEST_B over 10..19, no B/Z/X/*: every LCS across the groups is
    0, so in kinds 0 and 1 a group-B row's first WIDEST_A >= kFmtTile cells print as +inf, and in pid as 0.000000.  The
    ids start that +inf tile at every 16-byte phase in both kinds."""
    rng = np.random.default_rng(4300)
    a = random_set(rng, WIDEST_A, 5, 60, alphabet=10, with_specials=False)
    b = [(x + 10).astype(np.int8) for x in random_set(rng, WIDEST_B, 5, 60, alphabet=10, with_specials=False)]
    return _case("widest", a + b, _widest_ids(a + b), group_b=WIDEST_A)


@functools.lru_cache(maxsize=None)
def ids_case() -> dict:
    """One sequence per id length of ID_LENGTHS (printable ASCII), then UTF-8 ids, ids with ',' and ordinary ones."""
    rng = np.random.default_rng(4400)
    printable = np.array([c for c in range(0x20, 0x7f) if c != ord(",")], dtype=np.uint8)
    ids = [bytes(rng.choice(printable, size=k)) for k in ID_LENGTHS]
    ids += ["séquence-α|β".encode(), "蛋白质_7".encode(), bytes(range(0x80, 0x100)), "Ω".encode() * 300]
    ids += [b"a,b", b",", b"x,,y,", b"\xff,\xfe"]
    ids += [f"id{i}".encode() for i in range(40 - len(ids))]
    cl = random_set(rng, len(ids), 1, 300)
    return _case("ids", cl, ids)


def _flagged(rng, length: int, start: int) -> np.ndarray:
    """Random residues over 4 codes with an aligned 64-run of 'A' at `start`: lcs_shapes.quirky."""
    c = rng.integers(0, 4, size=length).astype(np.int8)
    c[start:start + 64] = lcs_shapes.A
    return c


@functools.lru_cache(maxsize=None)
def wide_elem() -> dict:
    """1 044 sequences around one of WIDE_LEN residues, so the triangle is uint32 and rows cross a tile:
      * flagged sequences (an aligned 64-run, as QUIRK_SEQS) before and after it;
      * an over-long pair (> 2048 residues) whose later member is flagged, as in test_dist_export_gpu's quirk_order;
        the WIDE_LEN sequence lies between them, so square mode reads its side row (it is over-long and comes before
        the last flagged over-long sequence) next to the 4-byte triangle."""
    rng = np.random.default_rng(4500)
    quirk = [seqio.encode(s) for s in QUIRK_SEQS[1::2]] + [_flagged(rng, 300, 128), _flagged(rng, 200, 64)]
    long_pair = random_set(rng, 2, 2100, 2400, alphabet=4)
    long_pair[1][128:192] = lcs_shapes.A + 1
    wide = rng.integers(0, 20, size=WIDE_LEN).astype(np.int8)
    cl = (random_set(rng, 500, 1, 300) + quirk[:2] + long_pair[:1] + random_set(rng, 530, 1, 300) + [wide]
          + random_set(rng, 3, 1, 300) + quirk[2:] + long_pair[1:] + random_set(rng, 4, 1, 300))
    at = {id(c): i for i, c in enumerate(cl)}
    return _case("wide_elem", cl, [f"w{i}/{len(c)}" for i, c in enumerate(cl)],
                 wide=at[id(wide)], long=sorted(at[id(c)] for c in long_pair),
                 flagged=sorted(at[id(c)] for c in quirk + long_pair[1:]))


@functools.lru_cache(maxsize=None)
def wide_elem_edge(max_len: int) -> dict:
    """A sequence of max_len residues (no B/Z/X/*), short ones, and a copy of it: their LCS is max_len itself, 65 535 in
    a uint16 triangle or 65 536 in a uint32 one."""
    rng = np.random.default_rng(4600 + max_len)
    big = rng.integers(0, 20, size=max_len).astype(np.int8)
    cl = [big] + random_set(rng, 10, 1, 300) + [big.copy()]
    return _case(f"wide_elem_{max_len}", cl, [f"e{i}" for i in range(len(cl))])


@functools.lru_cache(maxsize=None)
def empty() -> dict:
    rng = np.random.default_rng(4700)
    e = lambda: np.zeros(0, np.int8)
    cl = [e()] + random_set(rng, 5, 1, 50) + [e()] + random_set(rng, 3, 1, 50) + [e()]
    return _case("empty", cl, [f"z{i}" for i in range(len(cl))], empty=(0, 6, 10))


def case(name: str) -> dict:
    """The case called `name` (a key of MODES)."""
    if name.startswith("widths_sq_"):
        return widths_sq(int(name[len("widths_sq_"):]))
    if name.startswith("wide_elem_"):
        return wide_elem_edge(int(name[len("wide_elem_"):]))
    return {"widths_tri": widths_tri, "widest": widest, "ids": ids_case, "wide_elem": wide_elem, "empty": empty}[name]()


def cases() -> list[dict]:
    return [case(name) for name in MODES]


# ---------------------------------------------------------------- the text's layout
def split_rows(text: bytes, square: bool) -> tuple[int | None, list[int]]:
    """(header bytes or None, bytes of every row) of an export: each row and the header end with its only '\\n'."""
    lines = [len(x) + 1 for x in text.split(b"\n")[:-1]]
    assert sum(lines) == len(text)
    return (lines[0], lines[1:]) if square else (None, lines)


def chunk_plan(row_lengths, chunk_bytes: int, header: int | None = None) -> list[int]:
    """The sizes of famsa_dist_export's write calls: the header (square mode), then one per chunk.  A chunk takes rows
    while they fit in chunk_bytes (0 = K_DEFAULT_CHUNK); a row that does not fit starts the next chunk, and a row wider
    than chunk_bytes is a chunk of its own."""
    limit = chunk_bytes or K_DEFAULT_CHUNK
    out = [] if header is None else [header]
    acc = 0
    for b in row_lengths:
        if acc and acc + b > limit:
            out.append(acc)
            acc = 0
        acc += b
    if acc:
        out.append(acc)
    return out


def value_starts(row_lengths, ids, rows) -> list[int]:
    """Byte offset of the first value of each of `rows` from the start of the first row: in a single-chunk export, where
    k_dist_format's first tile of the row starts in the chunk buffer (its 16-byte phase is this offset mod 16)."""
    starts = np.concatenate([[0], np.cumsum(row_lengths)])
    return [int(starts[r]) + len(ids[r]) + 1 for r in rows]
