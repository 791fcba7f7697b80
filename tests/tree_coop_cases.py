"""Case generator for the cooperative guide-tree tests (tests/test_tree_coop_host.py, tests/test_tree_coop_gpu.py).

The guide-tree kernels of famsa_b200/csrc/tree.cu run on cooperative grids of 1024-thread blocks, capped at what stays
co-resident (about 135 k threads on an H100).  Two regimes are reached only by large inputs:

  * a thread that owns more than one sequence (k_prim<*>, k_upgma<*>): its first sequence lives in registers, the others
    are looped over through global memory (st[], visited[], the owner block b.id % gthreads / blockDim.x), and a k_nj
    warp that scans dozens of rows.  FAMSA_TREE_MAX_BLOCKS=<k> caps those grids at k blocks, so the sizes of SIZES(k)
    reach that loop with a few thousand sequences: exact fit, the first sequence of the second pass, a third pass;
  * float triangles of more than 2^32 elements (n > 92 682): big_upgma_pattern() plants LCS values past 2^32 in an
    otherwise constant triangle, with expectations derived by hand (big_upgma_expected) and confirmed by the restated
    computeTree on the same pattern moved into a small set (small_analogue).

prim_vectorised() is treeutil.prim_restated (MSTPrim's vertex loop with its lower-bound skip and key tie rule) with one
numpy pass per step, fast enough for ten thousand sequences.
"""
from __future__ import annotations

import numpy as np

from conftest import random_set
from famsa_b200 import seqio
from oracle import pyoracle as P
import upgma_cases as U

# tree.cu constants the cases are built on (test_tree_coop_host.py reads them from the source and compares)
COOP_THREADS = 1024     # threads per block of k_prim, k_upgma and k_nj
K_MST_CHUNK = 1024      # rows per block of k_mst_cols
NJ_ROWS_PER_BLOCK = 64  # k_nj: one block per 64 rows, before the co-residency cap

CAPS = [1, 2, 3]


def sizes(cap: int) -> list[int]:
    """n for a grid of `cap` blocks: exact fit, the first second-pass sequence, the second pass just short of, at and one
    past its end, and a third pass."""
    t = COOP_THREADS * cap
    return [t, t + 1, 2 * t - 1, 2 * t, 2 * t + 1, 3 * t + 5]


SETS = ["family", "dups", "abc3", "carry"]

# every (cap, n) gets the family set and one of the others in turn, so every set meets every cap
CASES = [(cap, n, s) for cap in CAPS for i, n in enumerate(sizes(cap)) for s in ("family", SETS[1 + (i + cap) % 3])]

NJ_CASES = [(1, 65), (1, 129), (1, 1025), (1, 2100), (2, 129), (2, 2100)]


def carry_positions(n: int, cap: int) -> list[int]:
    """Where the 8 dropped-carry sequences go: at indices >= 1024 * cap where the set has them (the loop path of k_prim),
    else at the end."""
    t = COOP_THREADS * cap
    pos = []
    for p in [t + o for o in (0, 1, 31, 32, 500, 1023, 1024, 2047)] + list(range(n - 1, -1, -1)):
        if p < n and p not in pos:
            pos.append(p)
        if len(pos) == 8:
            break
    return sorted(pos)


def sequence_set(name: str, n: int, cap: int, seed: int = 0):
    """(codes, offsets, lens, exact_ids) of a named set of n sequences; exact_ids: the sequences whose LCS values may
    depend on which side is the row (dropped-carry corner), whose rows and columns the restatement takes from the
    oracle."""
    rng = np.random.default_rng(1000 * n + 7 * cap + seed)
    exact = []
    if name == "family":
        return (*seqio.synth_family(n, 60, seed=int(rng.integers(1 << 30))), [])
    if name == "dups":                          # every sequence about eight times, copies spread over all blocks
        base = random_set(rng, max(n // 8, 1), 10, 40, alphabet=6, with_specials=False)
        cl = [base[i % len(base)].copy() for i in range(n)]
        cl = [cl[i] for i in rng.permutation(n)]
    elif name == "abc3":                        # three letters: whole rows of equal distances
        cl = random_set(rng, n, 15, 50, alphabet=3, with_specials=False)
    elif name == "carry":
        dc = U.dropped_carry_codes(rng)
        flagged, short = dc[50:], dc[:50]
        zero = np.zeros(1, np.int8)
        short += [np.concatenate([c, zero]) for c in random_set(rng, n - 58, 1, 8, alphabet=4, with_specials=False)]
        short = [short[i] for i in rng.permutation(len(short))]
        exact = carry_positions(n, cap)
        cl, it_f, it_s = [], iter(flagged), iter(short)
        for i in range(n):
            cl.append(next(it_f) if i in exact else next(it_s))
    else:
        raise KeyError(name)
    return (*seqio.pack(cl), exact)


# ------------------------------------------------------------------ Prim, vectorised
def pow075_table(max_indel: int) -> np.ndarray:
    """The host (double) pow(i, 0.75) table the device reads, through the oracle's Transform (LCS 1: pow075[indel] / 1)."""
    return np.array([P.transform(0, 1, i + 1, 1, True) for i in range(max_indel + 1)], dtype=np.float64)


NEVER_F64 = float(np.nextafter(np.finfo(np.float64).max, 0))


def transform_f64(kind: int, lcs, l1, l2, pow075) -> np.ndarray:
    """Transform<double, kind> element-wise (kinds 0 and 1), bit for bit the oracle's."""
    lcs = np.asarray(lcs, np.int64)
    indel = np.asarray(l1, np.int64) + np.asarray(l2, np.int64) - 2 * lcs
    num = pow075[indel] if kind == 0 else indel.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = num / lcs.astype(np.float64)
    return np.where(lcs == 0, NEVER_F64, d)


class LcsRows:
    """lcs[v][:] with v as the row, from a packed triangle of true (orientation-free) LCS values, with the rows and
    columns of exact_ids taken from the oracle."""

    def __init__(self, tri, codes, offsets, lens, exact_ids=()):
        self.tri = np.asarray(tri)
        self.n = n = len(lens)
        self.exact = np.array(sorted(exact_ids), dtype=np.int64)
        self.rows = {}
        if len(self.exact):
            r = P.lcs_rows(codes, offsets, lens, self.exact)
            self.rows = {int(v): r[k].astype(np.int64) for k, v in enumerate(self.exact)}
            self.cols = P.lcs_rows(codes, offsets, lens, np.arange(n), col_ids=self.exact).astype(np.int64)
        self.j = np.arange(n, dtype=np.int64)

    def __call__(self, v: int) -> np.ndarray:
        if v in self.rows:
            return self.rows[v]
        j = self.j
        hi, lo = np.maximum(j, v), np.minimum(j, v)
        idx = hi * (hi - 1) // 2 + lo
        idx[v] = 0
        out = self.tri[idx].astype(np.int64) if self.tri.size else np.zeros(self.n, np.int64)
        out[v] = 0
        if len(self.exact):
            out[self.exact] = self.cols[v]
        return out


def prim_vectorised(row_of, lens, kind, prune=True):
    """treeutil.prim_restated with one vector pass per step: (edge_from, edge_to, edge_dist, prim_order).  row_of(v)
    gives the LCS values of v (the row) against every sequence."""
    n = len(lens)
    L = np.asarray(lens, np.int64)
    pw = pow075_table(int(2 * L.max()) + 1) if kind == 0 else None
    dist = np.full(n, np.finfo(np.float64).max)
    key = np.zeros(n, dtype=np.uint64)
    visited = np.zeros(n, dtype=bool)
    order = np.full(n, n, dtype=np.int32)
    visited[0] = True
    order[0] = 0
    j = np.arange(n, dtype=np.uint64)
    full = np.uint64(0xFFFFFFFFFFFFFFFF)
    ef, et, ed = [], [], []
    v = 0
    for step in range(1, n):
        lv = int(L[v])
        tried = ~visited
        if prune:
            tried &= transform_f64(kind, np.minimum(L, lv), lv, L, pw) <= dist
        d = transform_f64(kind, row_of(v), lv, L, pw)
        vv = np.uint64(v)
        k = full ^ ((np.minimum(j, vv) << np.uint64(32)) + np.maximum(j, vv))
        upd = tried & (d <= dist) & ((d < dist) | (k < key))
        dist[upd] = d[upd]
        key[upd] = k[upd]
        cand = np.flatnonzero(~visited)
        c = cand[dist[cand] == dist[cand].min()]
        best = int(c[np.argmin(key[c])])
        p = int(full ^ key[best])
        ef.append(p >> 32); et.append(p & 0xFFFFFFFF); ed.append(dist[best])
        order[best] = step
        visited[best] = True
        v = best
    return np.array(ef, np.int32), np.array(et, np.int32), np.array(ed, np.float64), order


def distance_triangle_f64(kind, tri, lens) -> np.ndarray:
    """Transform<double, kind> of a packed LCS triangle (the Boruvka rounds' float64 triangle)."""
    n = len(lens)
    L = np.asarray(lens, np.int64)
    ii, jj = np.tril_indices(n, -1)                                  # row-major: the packed order
    pw = pow075_table(int(2 * L.max()) + 1) if kind == 0 else None
    return transform_f64(kind, np.asarray(tri), L[ii], L[jj], pw)


# ------------------------------------------------------------------ crafted UPGMA triangles in the loop path
def craft_coop(n: int, case: str, cap: int):
    """(LCS triangle uint16, lens) of n sequences of U.CRAFT_LEN residues on a background triangle:
    owner_tie     equal minima in rows j and j + 1024 * cap (the same thread's first and second row), partners at the
                  end: the first row wins, then the second
    stale_second  (0, 1) closest, (1, r) next with r = 1024 * cap + 3, the second row of thread 3: merging 0 and 1
                  relabels r's neighbour to 0 and keeps its old distance, so the next merge is r's
    last_row      the unique smallest distance in row n - 1, the last loop row of its thread"""
    t = COOP_THREADS * cap
    if case == "last_row":
        return U.craft(n, "last_row")
    lcs, lens = U.craft(n, "random")
    lcs[:] = U.BACKGROUND
    if case == "owner_tie":
        j = 3
        lcs[U.tri_index(j, n - 1)] = U.CLOSEST
        lcs[U.tri_index(j + t, n - 2)] = U.CLOSEST
    elif case == "stale_second":
        r = t + 3
        lcs[U.tri_index(0, 1)] = U.CLOSEST
        lcs[U.tri_index(1, r)] = U.SECOND
    else:
        raise KeyError(case)
    return lcs, lens


def craft_first_merges(n: int, case: str, cap: int):
    """The merges each crafted case is built to start with."""
    t = COOP_THREADS * cap
    if case == "owner_tie":
        return [(3, n - 1), (3 + t, n - 2)]
    if case == "stale_second":
        return [(0, 1), (t + 3, n)]
    return [(5, n - 1)]


CRAFT_CASES = [(cap, n, c) for cap in CAPS for n, c in ((2 * COOP_THREADS * cap + 1, "owner_tie"),
                                                        (3 * COOP_THREADS * cap + 5, "owner_tie"),
                                                        (COOP_THREADS * cap + 4, "stale_second"),
                                                        (3 * COOP_THREADS * cap + 5, "stale_second"),
                                                        (COOP_THREADS * cap + 1, "last_row"),
                                                        (3 * COOP_THREADS * cap + 5, "last_row"))]


# ------------------------------------------------------------------ a float triangle past 2^32 elements
BIG_N = 93000
TWO32 = 1 << 32
BIG_LEN, BIG_BG = 100, 50
# disjoint pairs (i, j, LCS), merged first, in this order; (37 075, 92 682) is the first cell of row 92 682 at or past
# 2^32, the others lie in rows wholly past it, and (10, 92 999) is far left in the last row
BIG_PAIRS = [(37075, 92682, 99), (50000, 92900, 98), (92750, 92990, 97), (10, 92999, 96)]
# the triple: (a, b) next, then the row a writes for the cluster ab (offsets past 2^32) decides the merge with c
BIG_TRIPLE = (92800, 92850, 92950)
BIG_TRIPLE_LCS = (95, 90)                       # LCS(a, b), LCS(a, c) = LCS(b, c)


def tri_index(i, j):
    return U.tri_index(i, j)


def big_cells():
    """(offset, LCS) of every planted cell of the big pattern."""
    a, b, c = BIG_TRIPLE
    x, y = BIG_TRIPLE_LCS
    cells = [(tri_index(i, j), v) for i, j, v in BIG_PAIRS]
    cells += [(tri_index(a, b), x), (tri_index(a, c), y), (tri_index(b, c), y)]
    return cells


def f32_dist(lcs: int) -> np.float32:
    """Transform<float, 0> of two BIG_LEN-residue sequences with this LCS."""
    return np.float32(P.transform(0, lcs, BIG_LEN, BIG_LEN, False))


def modified_avg(d1: np.float32, d2: np.float32) -> np.float32:
    """k_upgma's MAFFT-style average, each operation rounded to float as the kernel does."""
    f = np.float32
    return f(f(f(0.05) * f(d1 + d2)) + f(f(0.9) * min(d1, d2)))


def big_upgma_expected(n: int, pairs, triple, modified: bool):
    """The first len(pairs) + 2 merges of UPGMA on a constant background with the pattern planted (lens all BIG_LEN,
    background LCS BIG_BG).  The pairs are closer than the triple and than one another in their listed order, so they
    merge first, each as (lower, higher): both of its rows cache the pair's distance, and the lower row comes first.
    Then (a, b).  Row a's new cache is the average of d(a, c) and d(b, c), equal values; c's cache is the old d(a, c)
    pointing at a.  The normal average reproduces that distance exactly, so row a (a < c) is picked: (n + k, c).  The
    modified average may round it away: smaller or equal keeps (n + k, c), larger makes c's stale cache win: (c, n + k)."""
    out = [(i, j) for i, j, _ in pairs]
    a, b, c = triple
    out.append((a, b))
    k = n + len(pairs)
    dy = f32_dist(BIG_TRIPLE_LCS[1])
    new = modified_avg(dy, dy) if modified else np.float32(np.float32(dy + dy) * np.float32(0.5))
    out.append((k, c) if new <= dy else (c, k))
    return out


def small_analogue():
    """The big pattern moved into a small set with the same index order: (n, pairs, triple, LCS triangle, lens)."""
    ids = sorted({i for p in BIG_PAIRS for i in p[:2]} | set(BIG_TRIPLE) | {0, 1, 5})
    # keep a few background rows around every planted index, and rows 0.. as the big set has
    m = {}
    nxt = 0
    for i in range(max(ids) + 1):
        if i in ids or i < 3:
            m[i] = nxt
            nxt += 2                                                   # one background row between planted ones
    n = nxt + 2
    pairs = [(m[i], m[j], v) for i, j, v in BIG_PAIRS]
    triple = tuple(m[x] for x in BIG_TRIPLE)
    lcs = np.full(n * (n - 1) // 2, BIG_BG, dtype=np.uint16)
    for i, j, v in pairs:
        lcs[tri_index(i, j)] = v
    a, b, c = triple
    x, y = BIG_TRIPLE_LCS
    lcs[tri_index(a, b)] = x
    lcs[tri_index(a, c)] = y
    lcs[tri_index(b, c)] = y
    return n, pairs, triple, lcs, np.full(n, BIG_LEN, dtype=np.uint32)


def valid_tree(merges: np.ndarray, n: int) -> bool:
    """Every leaf and every internal node but the root is a child exactly once, and a node is used after it exists."""
    m = np.asarray(merges)
    if m.shape != (n - 1, 2):
        return False
    seen = np.zeros(2 * n - 1, dtype=bool)
    for k, (x, y) in enumerate(m.tolist()):
        for c in (x, y):
            if not (0 <= c < n + k) or seen[c]:
                return False
            seen[c] = True
    return bool(seen[:2 * n - 2].all())
