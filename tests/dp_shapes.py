"""Case generator for the profile-DP shape tests (tests/test_dp_shapes_host.py, tests/test_dp_shapes_gpu.py).

The DP kernels of famsa_b200/csrc/dp.cu have several fill kernels (one warp per merge, teams, the compact kernel,
thread-block clusters, producer / consumer pairs, the fused merge kernel), three ways to compute the column-pair scores T
(byte-digit IMMA with one or two counter digits, a scalar 32 x 64 path) and a T ring of 4- or 8-byte entries.  Realistic
families reach these by chance; the cases here reach each of them on purpose, at the boundaries the code is built around:

  * LAUNCH_SHAPES: development knobs (environment) that force each launch shape, with the class the `[dp]` debug line
    must report for it;
  * geometry_jobs(tw): stripe counts 1, TW-1, TW, TW+1, 2TW+1 for a team of TW warps, WR mod 32 in {0, 1, 31}, column
    widths around the steady-state gate, the 64-entry rings and the 512-thread row-0 scan of the prep kernel;
  * arithmetic_cases(): SeqSeq / SeqProf / ProfProf x 4- / 8-byte T ring, ProfProf x tmode 0 / 1 / 2, both sides of every
    decision, score digits at their extremes, and profiles whose counters sum past what the 4-byte ring allows;
  * traceback_cases(): wide x narrow merges whose paths leave the traceback's 64-step window and its speculative window;
  * tie_cases(): the ProfProf orientation rule at nz1 * W2 == nz2 * W1 and one off on either side;
  * fused_limit_cases(): merges on both sides of the fused kernel's limit for a direction matrix in shared memory.

Large member counts cost nothing: profile tables are linear in their members (counters and scores of a union of aligned
blocks of equal width are the sums of the blocks' tables, column 0 included), so a few small blocks, scaled and summed,
give a consistent profile of any member count (linear_profile).  label() computes from the tables alone what the prep
kernel decides: variant, orientation, counter digits (tmode), the T-ring width and the largest |T| of the merge.
"""
from __future__ import annotations

import numpy as np

from famsa_b200 import profiles

# dp.cu constants the cases are built on (test_dp_shapes_host.py reads them from the source and compares)
K_CHUNK = 8             # columns per chunk
K_RING = 64             # column-record window (columns mod 64)
K_TRING = 64            # T ring (wavefront steps mod 64)
K_TRACE_WIN = 96        # traceback window, wavefront steps
K_SPEC_SLACK = 16       # columns of slack of the speculative traceback window
K_DP_WARPS = 4          # merges per block of the one-warp kernel
K_DP_TEAM_WARPS = 8     # warps of the largest team / of a throughput-cluster block
K_DP_CLUSTER = 8        # blocks of a throughput cluster
K_FUSED_WARPS = 8       # warps of k_merge_fused
K_COL_FIELDS = 8
K_S2_STRIDE = 34
DIGIT1_MAX = 127        # members of a row profile whose counters are one byte digit
DIGIT2_MAX = 32767      # ... two byte digits
K_PREP_THREADS = 512
STRIPE = 32
SYNC_WIN = 64           # steps the traceback loads synchronously: st_hi - 63 .. st_hi

# sizeof(WarpShared): boundary cells, column records, staged scores, parked cells, T ring (all int64)
WARP_SHARED_BYTES = 8 * (2 * K_CHUNK * 4 + K_COL_FIELDS * K_RING + 2 * K_CHUNK * K_S2_STRIDE + K_CHUNK * 3 + K_TRING * 32)
FUSED_DIRS_LIMIT = K_FUSED_WARPS * WARP_SHARED_BYTES     # skewed direction bytes k_merge_fused keeps in shared memory

GAPS = np.array([-14850, -1250, -660, -660], dtype=np.int64)
RUN_GAPS = np.array([-3000, -20, -40, -5], dtype=np.int64)       # cheap extension: long gap runs
BIG = 1 << 20           # a development-knob width no merge reaches

# (name, env, target class, warps per merge TW, team line (warps, compact) for class 1, cluster size)
LAUNCH_SHAPES = [
    dict(name="one_warp", env={"FAMSA_DP_LATENCY_MODE": "0", "FAMSA_DP_TEAM_MIN": str(BIG), "FAMSA_DP_CLUSTER_MIN": str(BIG)},
         cls=0, tw=1),
    *[dict(name=f"team{n}", env={"FAMSA_DP_LATENCY_MODE": "0", "FAMSA_DP_TEAM_MIN": "0", "FAMSA_DP_CLUSTER_MIN": str(BIG),
                                 "FAMSA_DP_COMPACT": "0", "FAMSA_DP_TEAM_WARPS": str(n)}, cls=1, tw=n, team=(n, 0))
      for n in (2, 4, 8)],
    *[dict(name=f"compact{n}", env={"FAMSA_DP_LATENCY_MODE": "0", "FAMSA_DP_TEAM_MIN": "0", "FAMSA_DP_CLUSTER_MIN": str(BIG),
                                    "FAMSA_DP_COMPACT": "2", "FAMSA_DP_TEAM_WARPS": str(n)}, cls=1, tw=n, team=(n, 1))
      for n in (2, 4, 6)],
    dict(name="tp_cluster", env={"FAMSA_DP_LATENCY_MODE": "0", "FAMSA_DP_TEAM_MIN": "0", "FAMSA_DP_CLUSTER_MIN": "0"},
         cls=2, tw=K_DP_TEAM_WARPS * K_DP_CLUSTER),
    *[dict(name=f"latency_cl{cl}", env={"FAMSA_DP_LATENCY_MODE": "1", "FAMSA_DP_DUO": "0", "FAMSA_DP_MAX_CLUSTER": str(cl)},
           cls=10 + cl, tw=4 * cl, cl=cl) for cl in (1, 2, 4, 8, 16)],
    *[dict(name=f"duo_cl{cl}", env={"FAMSA_DP_LATENCY_MODE": "1", "FAMSA_DP_DUO": "1", "FAMSA_DP_MAX_CLUSTER": str(cl)},
           cls=100 + cl, tw=4 * cl, cl=cl) for cl in (2, 4, 8, 16)],
]
SHAPES = {s["name"]: s for s in LAUNCH_SHAPES}
# the shapes the arithmetic matrix runs through (plus the default shape and the fused kernel)
ARITH_SHAPES = ["one_warp", "compact2", "compact4", "compact6", "team2", "team4", "team8", "tp_cluster", "latency_cl2", "duo_cl2"]

GATE_WC = list(range(1, 10)) + [39, 40, 41]
RING_WC = [63, 64, 65, 127, 128, 129]
PREP_WC = [511, 512, 513]
GEOMETRY_WC = GATE_WC + RING_WC + PREP_WC
WR_RESIDUES = (0, 1, 31)


# ------------------------------------------------------------------ profiles
def score_matrix(seed: int = 1) -> np.ndarray:
    return profiles.synth_score_matrix(np.random.default_rng(seed))


def block_rows(n: int, cons: np.ndarray, rng, sub: float = 0.3, gap_runs: int = 1) -> np.ndarray:
    """n aligned rows around a consensus: substitutions and short internal gap runs; every row keeps a residue."""
    w = len(cons)
    rows = np.where(rng.random((n, w)) < sub, rng.integers(0, 20, size=(n, w)), cons[None, :]).astype(np.int8)
    for r in range(n):
        for _ in range(gap_runs if w >= 6 else 0):
            a = int(rng.integers(1, w - 1)); rows[r, a:a + int(rng.integers(1, 4))] = profiles.GAP
        if (rows[r] < 0).all():
            rows[r, 0] = cons[0]
    empty = (rows < 0).all(axis=0)                                    # no all-gap column (CProfile has none)
    rows[0, empty] = cons[empty]
    return rows


def add_tables(parts):
    """Sum of m x tables over (m, (scores, counters, card)) -- the tables of the union of the blocks' members."""
    s = sum(np.int64(m) * t[0] for m, t in parts)
    c = sum(np.int64(m) * t[1].astype(np.int64) for m, t in parts)
    k = sum(m * t[2] for m, t in parts)
    return s.astype(np.int64), c.astype(np.int32), int(k)


def linear_blocks(card: int, width: int, rng):
    """Three blocks (3, 2 and 1 rows around one consensus) and multiplicities (mx, my, mz) with 3 mx + 2 my + mz = card.
    From 600 members on my lies in 128..255, so that the cells only the second block fills hold one-digit counters with
    the top bit set while the shared cells reach two digits."""
    assert card >= 6
    cons = rng.integers(0, 20, size=width)
    blocks = [block_rows(3, cons, rng), block_rows(2, cons, rng, sub=0.5), block_rows(1, cons, rng)]
    my = 128 + card % 97 if card >= 600 else max(1, card // 8)
    mz = (card - 2 * my) % 3 or 3
    mx = (card - 2 * my - mz) // 3
    assert mx >= 1 and 3 * mx + 2 * my + mz == card
    return blocks, (mx, my, mz)


def linear_profile(card: int, width: int, rng, sm, gaps):
    blocks, mult = linear_blocks(card, width, rng)
    return add_tables([(m, profiles.tables_from_rows(b, sm, gaps)) for m, b in zip(mult, blocks)])


def expand_rows(blocks, mult) -> np.ndarray:
    """The explicit member rows of a linear profile (what tables_from_rows would see)."""
    return np.concatenate([np.repeat(b, m, axis=0) for b, m in zip(blocks, mult)])


def diverse_profile(card: int, width: int, rng, sm, gaps, sub: float = 0.9):
    """Many distinct residues per column: more non-zero counters per column than any linear profile has."""
    cons = rng.integers(0, 20, size=width)
    return profiles.tables_from_rows(block_rows(card, cons, rng, sub=sub), sm, gaps)


def seq_profile(width: int, rng, sm, gaps, residues=None):
    r = rng.integers(0, 24, size=width).astype(np.int8) if residues is None else np.asarray(residues, dtype=np.int8)
    return profiles.tables_from_rows(r[None, :], sm, gaps)


def distinct_profile(card: int, distinct: list[int], rng, sm, gaps):
    """A gap-free profile whose column c holds exactly distinct[c] different residues (so nz = sum(distinct))."""
    w = len(distinct)
    rows = np.zeros((card, w), dtype=np.int8)
    for c, d in enumerate(distinct):
        res = rng.permutation(24)[:d]
        rows[:, c] = res[np.minimum(np.arange(card), d - 1)]
    return profiles.tables_from_rows(rows, sm, gaps)


# ------------------------------------------------------------------ labels (what k_dp_prep decides)
def nz(counters) -> int:
    return int(np.count_nonzero(counters))


def label(job) -> dict:
    """Variant, orientation, row / column widths and members, tmode, the T-ring width (before and after the column-sum
    check) and the largest |T| over all cells, exactly (int64) from the tables."""
    s1, c1, k1, s2, c2, k2 = job
    w1, w2 = s1.shape[0] - 1, s2.shape[0] - 1
    if k1 == 1 and k2 == 1:
        var, sw = 0, 0
    elif k1 == 1:
        var, sw = 1, 0
    elif k2 == 1:
        var, sw = 1, 1
    else:
        var = 2
        sw = 0 if nz(c1) * w2 < nz(c2) * w1 else 1
    (sr, cr, nr), (sc, cc, nc) = ((s2, c2, k2), (s1, c1, k1)) if sw else ((s1, c1, k1), (s2, c2, k2))
    wr, wc = sr.shape[0] - 1, sc.shape[0] - 1
    col = sc[1:, :30].astype(np.int64)
    smax = int(np.abs(col).max())
    wide = bool(((col < -(1 << 31)) | (col >= (1 << 31))).any())
    if var == 2:
        csum = int(cr[1:, :30].astype(np.int64).sum(axis=1).max())
        tmode = 2 if wide else (0 if nr <= DIGIT1_MAX else (1 if nr <= DIGIT2_MAX else 2))
        t32_old = smax < (1 << 31) // (7 * nr)
        t32 = t32_old and csum <= 7 * nr
        T = cr[1:, :30].astype(np.int64) @ col.T
    else:
        csum, tmode = 1, 2
        t32_old = t32 = smax < (1 << 31)
        resid = [next((k for k in range(24) if cr[i, k]), 22) for i in range(1, wr + 1)]
        T = col[:, resid].T
    return dict(var=var, sw=sw, wr=wr, wc=wc, nr=nr, nc=nc, tmode=tmode, t32=t32, t32_old=t32_old, smax=smax,
                csum=csum, tmax=int(np.abs(T).max()), wide=wide)


# ------------------------------------------------------------------ geometry
def stripe_counts(tw: int) -> list[int]:
    return sorted({max(1, tw - 1), 1, tw, tw + 1, 2 * tw + 1})


def geometry_jobs(tw: int, seed: int = 0, max_min_width: int | None = None):
    """Jobs covering stripe counts x WR mod 32 x WC for a team of tw warps; SeqSeq, SeqProf and ProfProf in turn.
    Every (stripes, residue) pair gets three column widths from different parts of GEOMETRY_WC and every column width
    appears at least twice.  max_min_width keeps min(W1, W2) at or below a bound (the class-1 shapes: the host hands
    merges wider than 256 to the throughput cluster when there are few of them)."""
    rng = np.random.default_rng(1000 + 7 * tw + seed)
    sm = score_matrix(2)
    combos = [(s, r) for s in stripe_counts(tw) for r in WR_RESIDUES]
    n_wc = len(GEOMETRY_WC)
    jobs, meta = [], []
    for q, (s, r) in enumerate(combos):
        wr = STRIPE * s if r == 0 else STRIPE * (s - 1) + r
        for t in range(3):
            wc = GEOMETRY_WC[(3 * q + 7 * t) % n_wc]
            if max_min_width is not None and min(wr, wc) > max_min_width:
                wc -= 384                                             # 511..513 -> 127..129: still a ring boundary
            var = (q + t) % 3
            if var == 0:
                a, b = seq_profile(wr, rng, sm, GAPS), seq_profile(wc, rng, sm, GAPS)
            elif var == 1:
                a, b = seq_profile(wr, rng, sm, GAPS), diverse_profile(int(rng.integers(2, 7)), wc, rng, sm, GAPS)
            else:
                # the row profile: few distinct residues (two similar members); the column profile: many
                a = diverse_profile(2, wr, rng, sm, GAPS, sub=0.1)
                b = diverse_profile(int(rng.integers(5, 12)), wc, rng, sm, GAPS)
            jobs.append((*a, *b))
            meta.append(dict(stripes=s, wr=wr, wc=wc, var=var))
    # a ProfProf merge that the host, which sees only min(W1, W2) before the orientation is known, also gives tw stripes
    if tw > 1:
        wr, wc = STRIPE * tw + 1, STRIPE * tw - 1
        jobs.append((*diverse_profile(2, wr, rng, sm, GAPS, sub=0.1), *diverse_profile(7, wc, rng, sm, GAPS)))
        meta.append(dict(stripes=tw + 1, wr=wr, wc=wc, var=2))
    return jobs, meta


def host_stripes(job) -> int:
    """Stripes of a merge as the host estimates them before the prep kernel has decided the orientation."""
    w1, k1, w2, k2 = job[0].shape[0] - 1, job[2], job[3].shape[0] - 1, job[5]
    rows = w1 if k1 == 1 else (w2 if k2 == 1 else min(w1, w2))
    return (rows + STRIPE - 1) // STRIPE


def expected_classes(jobs, shape, cl_cap: int, duo_cap: int) -> dict:
    """{class: merges} the host assigns to a batch under `shape` (dp_run_device's cls())."""
    out = {}
    for j in jobs:
        if shape["cls"] < 10:
            c = shape["cls"]
        else:
            st = host_stripes(j)
            if st < 2:
                c = 0
            else:
                want, cl = (st + 3) // 4, 1
                while cl < want and cl < cl_cap:
                    cl *= 2
                duo = shape["env"].get("FAMSA_DP_DUO") != "0"
                c = 100 + min(cl, duo_cap) if duo and cl >= 2 and j[2] > 1 and j[5] > 1 else 10 + cl
        out[c] = out.get(c, 0) + 1
    return out


# ------------------------------------------------------------------ arithmetic
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
EXTREME_DIGITS = [I32_MIN, I32_MAX, -1, 0x80, 0xFF, -0x80, -0x81, 0x7F80, -0x7F01, 0x40FF80FF - (1 << 31)]
SMALL_DIGITS = [-1, 0x80, 0xFF, -0x80, -0x81, -0x100, 0x17F, -0xFF]


def _set_col_scores(prof, values, rng):
    """Column scores (rows 0..29 of columns 1..W) drawn from `values`, each value placed at least once."""
    s = prof[0].copy()
    w = s.shape[0] - 1
    v = np.asarray(values, dtype=np.int64)
    s[1:, :30] = v[rng.integers(0, len(v), size=(w, 30))]
    for q, x in enumerate(v):
        s[1 + q % w, (3 * q) % 24] = x
    return (s, prof[1], prof[2])


def _bounded_col(prof, smax, rng, hit_rows=None):
    """Column scores uniform in [-smax, smax]; +-smax itself at every row symbol in hit_rows (residue codes)."""
    s = prof[0].copy()
    w = s.shape[0] - 1
    s[1:, :30] = rng.integers(-smax, smax + 1, size=(w, 30))
    for q, k in enumerate(hit_rows or []):
        s[1:, k] = smax if q % 2 == 0 else -smax
    return (s, prof[1], prof[2])


def stacked_row(card: int, width: int, symbols: list[int]):
    """An inconsistent row profile that passes every check of the prep kernel: in every column, each of `symbols` is
    held by all `card` members (no gap counters), so a column's counters sum to len(symbols) * card."""
    s = np.zeros((width + 1, 32), dtype=np.int64)
    c = np.zeros((width + 1, 32), dtype=np.int32)
    c[1:, symbols] = card
    s[1:, :24] = -1000 * card
    s[0, profiles.GO], s[0, profiles.GE], s[0, profiles.TE], s[0, profiles.TO] = (card * g for g in GAPS[[0, 1, 3, 2]])
    return (s, c, card)


def t32_threshold(nr: int) -> int:
    """The largest column |score| the 4-byte ring admits for a ProfProf row profile of nr members."""
    return (1 << 31) // (7 * nr) - 1


def arithmetic_cases(seed: int = 5):
    """[(name, job, claims)]: claims are label() fields the case must have."""
    rng = np.random.default_rng(seed)
    sm = score_matrix(3)
    out = []

    def add(name, a, b, **claims):
        out.append((name, (*a, *b), claims))

    # SeqSeq / SeqProf: T is a column score; 4 bytes while |score| < 2^31
    for var in (0, 1):
        for name, vals, t32 in (("edge32", [I32_MAX, -I32_MAX, 5, -7], True), ("edge64", [I32_MIN, 3, I32_MAX], False),
                                ("wide", [5 << 32, -(3 << 33) + 1, 77], False)):
            row = seq_profile(134, rng, sm, GAPS, residues=rng.integers(0, 24, size=134))
            col = seq_profile(161, rng, sm, GAPS) if var == 0 else diverse_profile(5, 161, rng, sm, GAPS)
            col = _set_col_scores(col, vals, rng)
            add(f"var{var}_{name}", row, col, var=var, sw=0, t32=t32)
            if var == 1:                                              # the sequence second: swapped
                add(f"var1_{name}_swapped", col, row, var=1, sw=1, t32=t32)

    # ProfProf: tmode by the row profile's members, ring width by max|score| (threshold and threshold + 1)
    for nr, tmode in ((127, 0), (128, 1), (255, 1), (256, 1), (32767, 1), (32768, 2), (40000, 2)):
        for over in (0, 1):
            row = linear_profile(nr, 134, rng, sm, GAPS)
            col = diverse_profile(24, 165, rng, sm, GAPS)
            thr = t32_threshold(nr) + over
            col = _bounded_col(col, thr, rng, hit_rows=list(range(20)))
            add(f"pp_n{nr}_{'t64' if over else 't32'}", row, col, var=2, sw=0, tmode=tmode, t32=not over, nr=nr)
    # ProfProf with scores beyond int32: tmode 2 through the scores
    for nr in (7, 300):
        row = linear_profile(nr, 130, rng, sm, GAPS)
        col = _set_col_scores(diverse_profile(24, 154, rng, sm, GAPS), [(1 << 33) + 5, -(1 << 32) - 0x80, I32_MIN - 1, 17], rng)
        add(f"pp_n{nr}_wide", row, col, var=2, sw=0, tmode=2, t32=False, wide=True)
    # score digits at their extremes (8-byte ring: |INT32_MIN| = 2^31) and small scores with 0x80 / 0xFF low bytes (4 bytes)
    for nr, tmode in ((9, 0), (127, 0), (200, 1), (5000, 1)):
        row = linear_profile(nr, 132, rng, sm, GAPS)
        col = _set_col_scores(diverse_profile(24, 159, rng, sm, GAPS), EXTREME_DIGITS, rng)
        add(f"pp_n{nr}_extreme_digits", row, col, var=2, sw=0, tmode=tmode, t32=False)
        row = linear_profile(nr, 132, rng, sm, GAPS)
        col = _set_col_scores(diverse_profile(24, 159, rng, sm, GAPS), SMALL_DIGITS, rng)
        add(f"pp_n{nr}_small_digits", row, col, var=2, sw=0, tmode=tmode, t32=True)
    # counters and scores in rows 30 (GAP) and 31 (GUARD): part of neither T nor any check, so they must change nothing
    for nr, tmode in ((9, 0), (300, 1)):
        row = linear_profile(nr, 132, rng, sm, GAPS)
        c = row[1].copy()
        c[1:, 30], c[1:, 31] = 0x1FF, 0x2A5
        col = diverse_profile(24, 159, rng, sm, GAPS)
        sc = col[0].copy()
        sc[1:, 30:32] = rng.integers(-30000, 30000, size=(159, 2))
        add(f"pp_n{nr}_guard_rows", (row[0], c, nr), (sc, col[1], col[2]), var=2, sw=0, tmode=tmode, t32=True)
    # |T| at the 4-byte bound: seven symbols held by every member, scores +-threshold (sum = 7 card: still 4 bytes)
    for nr in (3, 100):
        thr = t32_threshold(nr)
        row = stacked_row(nr, 136, [0, 1, 2, 3, 4, 5, 6])
        for sign in (1, -1):
            col = diverse_profile(24, 163, rng, sm, GAPS)
            s = col[0].copy()
            s[1:, :30] = rng.integers(-thr, thr + 1, size=(163, 30))
            s[1::2, :7] = sign * thr                                 # every other column: T = sign * 7 * card * threshold
            add(f"pp_bound_n{nr}_{'pos' if sign > 0 else 'neg'}", row, (s, col[1], col[2]), var=2, sw=0, tmode=0, t32=True,
                tmax=7 * nr * thr)
        # one more member's worth of counters in a column: 8 bytes
        row8 = stacked_row(nr, 136, [0, 1, 2, 3, 4, 5, 6])
        c8 = row8[1].copy()
        c8[40, 7] = 1
        col = diverse_profile(24, 163, rng, sm, GAPS)
        s = col[0].copy()
        s[1:, :30] = rng.integers(-thr, thr + 1, size=(163, 30))
        add(f"pp_bound_n{nr}_sum_over", (row8[0], c8, nr), (s, col[1], col[2]), var=2, sw=0, tmode=0, t32=False, t32_old=True)
    return out


def overflow_witness(seed: int = 11):
    """A row profile whose columns hold ten symbols with every member on each (a sum of 10 x card, which the prep kernel
    lets through) against column scores just under the 4-byte threshold: |T| ~ 10/7 x 2^31.  A ring chosen from
    max|score| alone truncates T to 32 bits.  The row profile has 10 non-zero counters per column, so the column profile
    gets more (24 diverse members) to keep it on the row side."""
    rng = np.random.default_rng(seed)
    sm = score_matrix(4)
    nr = 6
    row = stacked_row(nr, 60, list(range(10)))
    col = diverse_profile(24, 90, rng, sm, GAPS)
    thr = t32_threshold(nr)
    s = col[0].copy()
    s[1:, :30] = rng.integers(thr // 2, thr + 1, size=(90, 30))
    return (*row, s, col[1], col[2])


def mixed_batch(seed: int = 5):
    """The arithmetic cases in one batch: 4- and 8-byte merges side by side (the compact kernel leaves the 8-byte ones
    to the k_dp_fill launch behind it)."""
    return [job for _, job, _ in arithmetic_cases(seed)]


# ------------------------------------------------------------------ traceback
def walk(path, wr: int, wc: int):
    """Replays a path backwards from (wr, wc) the way k_dp_trace does.  Returns (the longest run of moves inside one visit
    of a stripe, [exit column - diagonal prediction] for every stripe left through its first row)."""
    i, j = wr, wc
    longest, run, devs = 0, 0, []
    entry = None                                                      # (stripe, row inside it, column) where the visit began
    for d in np.asarray(path)[::-1]:
        if i == 0:                                                    # row 0: the rest is H moves, outside every stripe
            break
        if entry is None:
            entry, run = ((i - 1) // STRIPE, (i - 1) % STRIPE, j), 0
        i -= int(d != 1)
        j -= int(d != 2)
        run += 1
        if i == 0 or (i - 1) // STRIPE != entry[0]:
            longest = max(longest, run)
            if i >= 1:                                                # into the stripe above: p = j0 - (l0 + 1) predicted
                devs.append(j - (entry[2] - (entry[1] + 1)))
            entry = None
    return max(longest, run), devs


def traceback_cases(seed: int = 13):
    """Wide x narrow merges with cheap gap extension: long H runs in a 2-stripe matrix, long V runs in a 40-column one."""
    rng = np.random.default_rng(seed)
    sm = score_matrix(5)
    out = []
    for wr, wc, kind in ((33, 3000, "seqprof"), (500, 40, "seqprof"), (33, 3000, "profprof"), (500, 40, "profprof"),
                         (70, 1200, "seqseq")):
        if kind == "seqseq":
            a, b = seq_profile(wr, rng, sm, RUN_GAPS), seq_profile(wc, rng, sm, RUN_GAPS)
        elif kind == "seqprof":
            a, b = seq_profile(wr, rng, sm, RUN_GAPS), diverse_profile(3, wc, rng, sm, RUN_GAPS, sub=0.3)
        else:
            a, b = diverse_profile(2, wr, rng, sm, RUN_GAPS, sub=0.05), diverse_profile(9, wc, rng, sm, RUN_GAPS)
        out.append((f"{kind}_{wr}x{wc}", (*a, *b)))
    return out


# ------------------------------------------------------------------ orientation tie
def tie_cases(seed: int = 17):
    """ProfProf pairs of widths 40 and 41 with nz1 * 41 - nz2 * 40 in {-1, 0, +1}: the rule swaps unless nz1 * W2 < nz2 * W1."""
    rng = np.random.default_rng(seed)
    sm = score_matrix(6)
    out = []
    for delta, (n1, n2) in ((-1, (119, 122)), (0, (120, 123)), (1, (121, 124))):
        d1, d2 = [3] * 40, [3] * 41
        d1[0] += n1 - 120
        d2[0] += n2 - 123
        a = distinct_profile(4, d1, rng, sm, GAPS)
        b = distinct_profile(5, d2, rng, sm, GAPS)
        out.append((delta, (*a, *b)))
    return out


# ------------------------------------------------------------------ fused kernel
def fused_dirs_bytes(wr: int, wc: int) -> int:
    return ((wr + STRIPE - 1) // STRIPE) * (wc + 32) * 32


def fused_limit_cases(seed: int = 19):
    """SeqProf merges (the sequence is the row side) just inside and just outside the fused kernel's limit for holding the
    skewed direction matrix in shared memory: 16 stripes (512 rows, the fused kernel's row limit) and 2 stripes."""
    rng = np.random.default_rng(seed)
    sm = score_matrix(7)
    out = []
    for wr in (512, 64):
        st = (wr + STRIPE - 1) // STRIPE
        wc_max = FUSED_DIRS_LIMIT // (st * 32) - 32
        for wc in (wc_max, wc_max + 1):
            a = seq_profile(wr, rng, sm, GAPS)
            b = diverse_profile(4, wc, rng, sm, GAPS)
            out.append((wr, wc, fused_dirs_bytes(wr, wc) <= FUSED_DIRS_LIMIT, (*a, *b)))
    return out
