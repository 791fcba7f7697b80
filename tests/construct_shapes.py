"""Cases for the ConstructProfile shape tests (tests/test_construct_shapes_host.py, tests/test_construct_shapes_gpu.py).

Every merged profile is built by construct_tile (famsa_b200/csrc/prof_dev.cuh), in k_prof_construct (one 64-column tile
per block) and in k_merge_fused (one block walks all tiles of a merge).  It computes every merged column on its own from
prefix counts over the path and the children's counters at src / src + 1 (prof.cu's header, DESIGN §4b), where the
reference walks the path once.  A case here is one merge -- two children, gap costs -- and the classes of that
derivation it claims to reach:

  * natural cases: children built from (gapped) rows, the DP picks the path;
  * forced cases: the children keep the counters of their rows, but the column profile's residue scores are crafted so
    that the DP's optimum is a path chosen in advance.  CProfile::Align reads the stored score table (profile_par.cpp
    takes profile2->scores), so the reference runs its own Align on the same tables (RefDp.set_scores).

path_classes() names what a path reaches; ALL_CLASSES is the list the cases together must cover.  construct_np() restates
construct_tile's independent-column formulas in numpy, as written in the kernel.
Path codes: 0 = D, 1 = H (a gap column in the row child), 2 = V (a gap column in the column child)."""
from __future__ import annotations

import os
import zlib

import numpy as np

from famsa_b200 import profiles, seqio
from oracle import pyoracle

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "construct_shapes.npz")

TILE = 64                      # kConTile (prof_dev.cuh)
FUSED_MAX_HOST_ROWS = 512      # kFusedMaxHostRows (tree_plan.h)
FUSED_MAX_WIDTH = 8192         # kFusedMaxWidth
GO, GE, TE, TO, GAP_LANE, N_AA = 25, 26, 27, 28, 30, 24
BIG = 10 ** 8                  # crafted residue score: dwarfs every gap cost of the forced cases
LETTERS = seqio.ALPHABET       # "ARNDCQEGHILKMFPSTWYVBZX*"

SIDES = ("R", "C")
ALL_CLASSES = sorted(
    [f"{s}_start_{w}_len{n}" for s in SIDES for w in ("src0", "srcw", "interior") for n in ("1", "2+")]
    + [f"{s}_interior_run_gt64" for s in SIDES]
    + [f"{s}_transfer_col1" for s in SIDES] + [f"{s}_transfer_interior" for s in SIDES]
    + ["transfer_after_other_gap", "transfer_go", "transfer_to", "adjacent_HV", "adjacent_VH"]
    + [f"split_{k}_{t}" for k in ("start", "cont") for t in ("go_s", "ge_s", "to_s", "te_s", "to_n")]
    + ["all_gap_child_column"]
    + [f"event_mod{m}" for m in (62, 63, 0, 1)] + ["tile_start_prev_in_previous_tile", "tile_first_continues_run"]
    + [f"W1_mod{m}" for m in (63, 0, 1)] + ["W_sum_minus_1", "W_max"]
    + ["swapped", "not_swapped"]
    + ["cards_1x1", "cards_1xN", "cards_NxM", "rows_at_fused_limit", "card_65536", "width_over_fused", "all_24_letters"])


# ------------------------------------------------------------------ scoring
_sm = None


def score_matrix() -> np.ndarray:
    """The reference's substitution matrix (its gap rescaling does not touch it): live, else the fixture's copy."""
    global _sm
    if _sm is None:
        if pyoracle.have_ref():
            dp = pyoracle.RefDp(0)
            _sm = dp.score_matrix()
            dp.close()
        else:
            _sm = np.load(FIXTURE)["score_matrix"]
    return _sm


def codes(row: str) -> np.ndarray:
    """A gapped row as tables_from_rows takes it: residue codes, -1 for '-'."""
    return np.array([-1 if ch == "-" else LETTERS.index(ch) for ch in row], dtype=np.int8)


def child_tables(child, gaps, sm=None):
    """(scores, counters, card) of a child: ("leaf", letters) or ("rows", [gapped rows]), crafted scores if given."""
    kind, body = child[0], child[1]
    rows = [body] if kind == "leaf" else body
    s, c, k = profiles.tables_from_rows(np.stack([codes(r) for r in rows]), score_matrix() if sm is None else sm, gaps)
    if len(child) > 2 and child[2] is not None:
        s = child[2]
    if len(child) > 3 and child[3] is not None:
        c = child[3]
    return s, c, k


def nonzero(counters) -> int:
    return int(np.count_nonzero(counters))


def orientation(t1, t2) -> bool:
    """CProfile::Align's choice (profile.cpp:254-304): is the DP's row profile the second child?"""
    if t1[2] == 1 and t2[2] == 1:
        return False
    if t1[2] == 1:
        return False
    if t2[2] == 1:
        return True
    w1, w2 = t1[0].shape[0] - 1, t2[0].shape[0] - 1
    return not (nonzero(t1[1]) * w2 < nonzero(t2[1]) * w1)


# ------------------------------------------------------------------ classes
def run_length(path, k0: int) -> int:
    """Length of the run that starts at path index k0."""
    d, n = path[k0], 1
    while k0 + n < len(path) and path[k0 + n] == d:
        n += 1
    return n


def path_classes(path, rows_tab, cols_tab) -> set:
    """The derivation's classes a path reaches; rows_tab / cols_tab: (scores, counters, card) of the DP's row / column
    child (after the orientation swap)."""
    path = np.asarray(path, dtype=np.uint8)
    cr, cc = rows_tab[1], cols_tab[1]
    wr, wc = cr.shape[0] - 1, cc.shape[0] - 1
    out = set()
    nh = np.cumsum(path == 1)
    nv = np.cumsum(path == 2)
    W = len(path)
    for k in range(1, W + 1):
        d, prev = int(path[k - 1]), int(path[k - 2]) if k >= 2 else 0
        i, j = k - int(nh[k - 1]), k - int(nv[k - 1])
        if d != prev and k % TILE in (62, 63, 0, 1):
            out.add(f"event_mod{k % TILE}")
        if d != 0:
            side = "R" if d == 1 else "C"
            src, w, cnt = (i, wr, cr) if d == 1 else (j, wc, cc)
            kind = "cont" if prev == d else "start"
            if kind == "start":
                where = "src0" if src == 0 else "srcw" if src >= w else "interior"
                n = run_length(path, k - 1)
                out.add(f"{side}_start_{where}_len{'1' if n == 1 else '2+'}")
                if where == "interior" and n > TILE:
                    out.add(f"{side}_interior_run_gt64")
                if prev != 0 and prev != d:
                    out.add("adjacent_HV" if prev == 1 else "adjacent_VH")
                if k % TILE == 0:
                    out.add("tile_start_prev_in_previous_tile")
            elif k % TILE == 0:
                out.add("tile_first_continues_run")
            if 0 < src < w:
                for lane, name in ((GO, "go_s"), (GE, "ge_s"), (TO, "to_s"), (TE, "te_s")):
                    if cnt[src, lane]:
                        out.add(f"split_{kind}_{name}")
                if cnt[src + 1, TO]:
                    out.add(f"split_{kind}_to_n")
        for side, gap_dir, col, cnt in (("R", 1, i, cr), ("C", 2, j, cc)):
            if d != gap_dir and prev == gap_dir:           # this step consumes a column of the child the run was in
                out.add(f"{side}_transfer_col1" if col == 1 else f"{side}_transfer_interior")
                if d != 0:
                    out.add("transfer_after_other_gap")
                if col > 1 and cnt[col, GO]:
                    out.add("transfer_go")
                if cnt[col, TO]:
                    out.add("transfer_to")
    if (W + 1) % TILE in (63, 0, 1):
        out.add(f"W1_mod{(W + 1) % TILE}")
    if W == wr + wc - 1:
        out.add("W_sum_minus_1")
    if W == max(wr, wc):
        out.add("W_max")
    for c in (cr, cc):
        if (c[1:, :N_AA].sum(axis=1) == 0).any():
            out.add("all_gap_child_column")
    return out


def case_classes(case, t1, t2, res) -> set:
    """Path classes plus what the children and the outcome say: orientation, cards, widths, letters."""
    sw = bool(res["swapped"])
    rt, ct = (t2, t1) if sw else (t1, t2)
    out = path_classes(res["path"], rt, ct)
    out.add("swapped" if sw else "not_swapped")
    k1, k2 = t1[2], t2[2]
    w1, w2 = t1[0].shape[0] - 1, t2[0].shape[0] - 1
    out.add("cards_1x1" if k1 == k2 == 1 else "cards_1xN" if min(k1, k2) == 1 else "cards_NxM")
    if fused_eligible(t1, t2) and host_rows(t1, t2) == FUSED_MAX_HOST_ROWS:
        out.add("rows_at_fused_limit")
    if max(k1, k2) >= 65536:
        out.add("card_65536")
    if max(w1, w2) > FUSED_MAX_WIDTH:
        out.add("width_over_fused")
    for ch in (case["a"], case["b"]):
        if ch[0] == "leaf" and set(ch[1]) >= set(LETTERS):
            out.add("all_24_letters")
    return out


def host_rows(t1, t2) -> int:
    """dp_plan.h host_rows: the DP's row count as the launch planner sees it."""
    w1, w2 = t1[0].shape[0] - 1, t2[0].shape[0] - 1
    return w1 if t1[2] == 1 else w2 if t2[2] == 1 else min(w1, w2)


def fused_eligible(t1, t2) -> bool:
    w1, w2 = t1[0].shape[0] - 1, t2[0].shape[0] - 1
    return host_rows(t1, t2) <= FUSED_MAX_HOST_ROWS and max(w1, w2) <= FUSED_MAX_WIDTH


# ------------------------------------------------------------------ construct_tile, restated
def construct_np(rows_tab, cols_tab, path, gaps):
    """construct_tile's formulas (prof_dev.cuh) for every merged column at once: prefix H / V counts give the child
    columns i, j; a consumed column takes the transfer when the previous step was a gap in its child (no open part at
    column 1); a gap column is gap_split of the child's counters at src and src + 1.  Returns (scores, counters)."""
    go, ge, to, te = (int(x) for x in gaps)
    sr, cr, kr = rows_tab
    sc, cc, kc = cols_tab
    wr, wc = cr.shape[0] - 1, cc.shape[0] - 1
    path = np.asarray(path, dtype=np.int64)
    W = len(path)
    os_ = np.zeros((W + 1, 32), dtype=np.int64)
    oc = np.zeros((W + 1, 32), dtype=np.int64)
    os_[0, [GO, GE, TO, TE]] = np.array([go, ge, to, te], dtype=np.int64) * (kr + kc)
    if W == 0:
        return os_, oc.astype(np.int32)
    k = np.arange(1, W + 1)
    d = path
    prev = np.concatenate([[0], path[:-1]])                      # "previous" of column 1 is D
    i = k - np.cumsum(d == 1)
    j = k - np.cumsum(d == 2)
    for gap_dir, col, s_t, c_t in ((1, i, sr, cr), (2, j, sc, cc)):
        m = d != gap_dir                                         # this child supplies a column
        ks, cs = k[m], col[m]
        c = c_t[cs].astype(np.int64)
        s = s_t[cs].astype(np.int64)
        after = prev[m] == gap_dir
        tt = np.where(after, c[:, TO], 0)
        tg = np.where(after & (cs != 1), c[:, GO], 0)
        c[:, GE] += tg; c[:, GO] -= tg; c[:, TE] += tt; c[:, TO] -= tt
        s[:, :N_AA] += (tg * (ge - go) + tt * (te - to))[:, None]
        os_[ks] += s
        oc[ks] += c
    m = d != 0
    ks, dm, pm = k[m], d[m], prev[m]
    isH = dm == 1
    src = np.where(isH, i[m], j[m])
    w = np.where(isH, wr, wc)
    card = np.where(isH, kr, kc).astype(np.int64)
    col = np.where(isH[:, None], cr[np.minimum(src, wr)], cc[np.minimum(src, wc)]).astype(np.int64)
    nxt_r = cr[np.minimum(src + 1, wr)]
    nxt_c = cc[np.minimum(src + 1, wc)]
    to_n = np.where(src < w, np.where(isH, nxt_r[:, TO], nxt_c[:, TO]), 0).astype(np.int64)
    go_s, ge_s, to_s, te_s = col[:, GO], col[:, GE], col[:, TO], col[:, TE]
    starts = pm != dm
    z = np.zeros_like(card)
    # starting: src == 0 / src >= w / interior
    s_to = np.where(src == 0, card, np.where(src >= w, card - (to_s + te_s), to_n))
    s_te = np.where(src == 0, z, to_s + te_s)
    s_e = np.where((src == 0) | (src >= w), z, go_s + ge_s)
    s_o = np.where((src == 0) | (src >= w), z, card - s_e - s_to - s_te)
    # continuing: src == 0 or src == w / interior
    ends = (src == 0) | (src == w)
    c_te = np.where(ends, card, to_n + to_s + te_s)
    c_e = np.where(ends, z, card - c_te)
    o = np.where(starts, s_o, z)
    e = np.where(starts, s_e, c_e)
    t_o = np.where(starts, s_to, z)
    t_e = np.where(starts, s_te, c_te)
    oc[ks, GO] += o; oc[ks, GE] += e; oc[ks, TO] += t_o; oc[ks, TE] += t_e; oc[ks, GAP_LANE] += card
    os_[ks, :N_AA] += (o * go + e * ge + t_o * to + t_e * te)[:, None]
    return os_, oc.astype(np.int32)


# ------------------------------------------------------------------ random children and paths (derivation test)
def random_child(rng, width: int, card: int, gap_p: float):
    """A gapped block of `card` rows (every row keeps a residue; all-gap columns allowed) and its tables."""
    rows = rng.integers(0, 24, size=(card, width)).astype(np.int8)
    rows[rng.random((card, width)) < gap_p] = -1
    for r in range(card):
        if (rows[r] < 0).all():
            rows[r, rng.integers(0, width)] = rng.integers(0, 24)
    return rows


def random_path(rng, wr: int, wc: int) -> np.ndarray:
    """A random monotone path from (0, 0) to (wr, wc): runs of random lengths in random directions."""
    out = []
    i = j = 0
    while i < wr or j < wc:
        choices = [dd for dd, ok in ((0, i < wr and j < wc), (1, j < wc), (2, i < wr)) if ok]
        dd = int(rng.choice(choices))
        n = int(rng.choice([1, 1, 2, 3, 5, 70])) if dd else int(rng.integers(1, 4))
        for _ in range(n):
            if (dd == 0 and i < wr and j < wc) or (dd == 1 and j < wc) or (dd == 2 and i < wr):
                out.append(dd)
                i += dd != 1
                j += dd != 2
    return np.array(out, dtype=np.uint8)


# ------------------------------------------------------------------ the cases
def _rand_letters(rng, n: int, alphabet: str = LETTERS[:20]) -> str:
    return "".join(alphabet[x] for x in rng.integers(0, len(alphabet), size=n))


def _block(rng, n_rows: int, base: str, gap_p: float = 0.0, sub: float = 0.15) -> list[str]:
    """Rows around a consensus with substitutions and random gaps (each row keeps a residue)."""
    out = []
    for _ in range(n_rows):
        r = [ch if rng.random() > sub else LETTERS[rng.integers(0, 20)] for ch in base]
        r = ["-" if rng.random() < gap_p else ch for ch in r]
        if all(ch == "-" for ch in r):
            r[0] = base[0]
        out.append("".join(r))
    return out


def _crafted(rows_child, good_cols, row_letter_w: str = "W", gaps=None):
    """Column-side child `rows_child` with residue scores that reward only 'A' rows on its good columns: a D step of an
    'A' column of the row child on a good column scores +BIG per residue, every other pairing -BIG."""
    s, c, _ = profiles.tables_from_rows(np.stack([codes(r) for r in rows_child[1]]), score_matrix(), gaps)
    s = s.copy()
    good = np.zeros(s.shape[0], dtype=bool)
    good[np.asarray(good_cols, dtype=np.int64)] = True
    s[1:, :N_AA] = -BIG
    s[1:, LETTERS.index("A")] = np.where(good[1:], BIG, -BIG)
    return ("rows", rows_child[1], s)


def _cols_with_gap_kinds(rng, width: int, j0: int, all_gap_col: int) -> list[str]:
    """Seven rows of `width` columns whose counters at column j0 hold GO, GE, TO and TE, and at j0 + 1 TO and GO
    (1-based columns); column all_gap_col is a gap in every row."""
    base = _rand_letters(rng, width)
    rows = [list(base) for _ in range(7)]
    a, b = j0 - 1, j0                      # 0-based indices of columns j0, j0 + 1
    rows[1][a - 1] = rows[1][a] = "-"      # GO at j0 - 1, GE at j0
    rows[2][a] = "-"                       # GO at j0
    for x in range(0, a + 1):
        rows[3][x] = "-"                   # leading terminal run 1..j0: TE at j0
    for x in range(a, width):
        rows[4][x] = "-"                   # trailing terminal run from j0: TO at j0
    for x in range(b, width):
        rows[5][x] = "-"                   # trailing terminal run from j0 + 1: TO at j0 + 1
    rows[6][b] = "-"                       # GO at j0 + 1
    for r in rows:
        r[all_gap_col - 1] = "-"
    return ["".join(r) for r in rows]


def cases() -> list[dict]:
    """dict(name, a, b, gaps, claims) -- a / b: ("leaf", letters) or ("rows", gapped rows[, crafted scores])."""
    out = []
    g_def = (-14000, -1200, -3000, -500)
    rng = np.random.default_rng(2024)

    # ---- natural: two leaves, an insertion at a chosen merged column (identical prefix: all D)
    no_w = LETTERS[:17] + LETTERS[18:20]
    for p, n_ins in ((61, 1), (62, 3), (63, 2), (64, 1), (127, 5)):
        base = _rand_letters(rng, 150, no_w)
        ins = "W" * n_ins                                        # no W around it: the run cannot slide
        out.append(dict(name=f"leaves_insert_at{p + 1}_len{n_ins}", a=("leaf", base), b=("leaf", base[:p] + ins + base[p:]),
                        gaps=g_def, claims={f"event_mod{(p + 1) % TILE}", "cards_1x1"}))
    # all 24 letters in both leaves; the second drops one residue
    base = "".join(rng.permutation(list(LETTERS * 3)))
    out.append(dict(name="leaves_all_letters", a=("leaf", base), b=("leaf", base[:40] + base[41:]), gaps=g_def,
                    claims={"all_24_letters", "cards_1x1", "C_start_interior_len1"}))
    # infix: leading and trailing runs in the shorter child, both orientations
    core = _rand_letters(rng, 90)
    for lead, trail in ((1, 1), (4, 3)):
        full = _rand_letters(rng, lead) + core + _rand_letters(rng, trail)
        ln = "1" if lead == 1 else "2+"
        out.append(dict(name=f"infix_{lead}_{trail}", a=("leaf", full), b=("leaf", core), gaps=g_def,
                        claims={f"C_start_src0_len{ln}", f"C_start_srcw_len{ln}", "C_transfer_col1"}))
    prof = _block(rng, 5, core, gap_p=0.05)
    out.append(dict(name="infix_profile_first", a=("rows", prof), b=("leaf", _rand_letters(rng, 3) + core + _rand_letters(rng, 2)),
                    gaps=g_def, claims={"swapped", "cards_1xN"}))
    out.append(dict(name="infix_leaf_first", a=("leaf", _rand_letters(rng, 3) + core + _rand_letters(rng, 2)), b=("rows", prof),
                    gaps=g_def, claims={"not_swapped", "cards_1xN"}))
    # identical children: W = w, the tiles counted from 2w + 1 are half empty
    for w in (62, 63, 64):
        blk = _block(rng, 3, _rand_letters(rng, w), gap_p=0.04)
        out.append(dict(name=f"identical_w{w}", a=("rows", blk), b=("rows", list(blk)), gaps=g_def,
                        claims={"W_max", f"W1_mod{(w + 1) % TILE}", "cards_NxM"}))
    # disjoint blocks that score negatively and cheap gaps: an H run right next to a V run
    pre, suf = _rand_letters(rng, 30), _rand_letters(rng, 30)
    out.append(dict(name="disjoint_blocks", a=("leaf", pre + "WWWWWW" + suf), b=("leaf", pre + "DDDDD" + suf),
                    gaps=(-200, -100, -200, -100), claims={"R_start_interior_len2+", "C_start_interior_len2+"}))
    # a deletion longer than a tile
    base = _rand_letters(rng, 300)
    out.append(dict(name="deletion_70", a=("leaf", base), b=("leaf", base[:100] + base[170:]), gaps=g_def,
                    claims={"C_interior_run_gt64"}))
    # N x M at the fused kernel's row limit
    b512 = _rand_letters(rng, FUSED_MAX_HOST_ROWS)
    out.append(dict(name="profiles_at_fused_row_limit", a=("rows", _block(rng, 4, b512, gap_p=0.03)),
                    b=("rows", _block(rng, 6, b512[:200] + b512[203:] + "KKK", gap_p=0.03)), gaps=g_def,
                    claims={"rows_at_fused_limit", "cards_NxM"}))
    # 65 536 rows against a leaf with an insertion
    b40 = _rand_letters(rng, 40)
    big = _block(rng, 64, b40, gap_p=0.05) * 1024
    out.append(dict(name="rows_65536", a=("rows", big), b=("leaf", b40[:20] + "PP" + b40[20:]), gaps=g_def,
                    claims={"card_65536"}))
    # wider than the fused kernel takes
    base = _rand_letters(rng, 8300)
    out.append(dict(name="wide_8300", a=("leaf", base), b=("leaf", base[:4000] + base[4075:]), gaps=g_def,
                    claims={"width_over_fused"}))

    # ---- forced: the row child is a leaf of 'A' (matched) and 'W' (unmatched) columns, the column child's scores
    # reward 'A' on its good columns only (SeqProf: the leaf is the DP's row profile)
    def forced(name, r_letters, c_rows, good, gaps, claims, swap=False):
        c = _crafted(("rows", c_rows), good, gaps=gaps)
        a, b = ("leaf", r_letters), c
        out.append(dict(name=name, a=b if swap else a, b=a if swap else b, gaps=gaps, claims=claims))

    # alternating length-1 runs: nothing matches, an open costs little, an extension much
    cheap_open = (-100, -100000, -100, -100000)
    forced("forced_alternating", "W" * 40, _block(rng, 3, _rand_letters(rng, 40)), [], cheap_open,
           {"adjacent_HV", "adjacent_VH", "R_start_interior_len1", "C_start_interior_len1", "transfer_after_other_gap"})
    # nothing matches and runs are dear: all H, then all V.  The DP cannot avoid every D (in the first row and column a
    # gap state only extends its own run), so one D leads and W = w1 + w2 - 1 is the widest path; here W + 1 = 64
    few_runs = (-100000, -1, -100000, -1)
    forced("forced_all_gaps", "W" * 30, _block(rng, 2, _rand_letters(rng, 34)), [], few_runs,
           {"W_sum_minus_1", "W1_mod0"})
    # runs that cover whole tiles, starting / ending at tile edges: D x p, H x 66, D x rest
    for p in (61, 62, 63):
        wc = p + 66 + 40
        good = list(range(1, p + 1)) + list(range(p + 67, wc + 1))
        forced(f"forced_tile_run_after{p}", "A" * (p + 40), _block(rng, 2, _rand_letters(rng, wc)), good, g_def,
               {"R_interior_run_gt64", "tile_first_continues_run", f"event_mod{(p + 1) % TILE}"})
    # runs at both ends of the row child (H) and of the column child (V), lengths 1 and >= 2
    for lead, trail in ((1, 1), (3, 2)):
        wc = lead + 50 + trail
        forced(f"forced_row_child_ends_{lead}_{trail}", "A" * 50, _block(rng, 2, _rand_letters(rng, wc)),
               range(lead + 1, lead + 51), g_def, {"R_start_src0_len" + ("1" if lead == 1 else "2+"), "R_transfer_col1"})
        forced(f"forced_col_child_ends_{lead}_{trail}", "W" * lead + "A" * 50 + "W" * trail,
               _block(rng, 2, _rand_letters(rng, 50)), range(1, 51), g_def,
               {"C_start_src0_len" + ("1" if lead == 1 else "2+"), "C_start_srcw_len" + ("1" if trail == 1 else "2+"),
                "C_transfer_col1"})
    # a V run (gap in the column child) at a column whose counters hold every gap kind, and the transfer after it
    for n in (1, 3):
        j0 = 20
        rows = _cols_with_gap_kinds(rng, 45, j0, all_gap_col=35)
        forced(f"forced_gap_kinds_v{n}", "A" * j0 + "W" * n + "A" * 25, rows, range(1, 46), g_def,
               {"all_gap_child_column", "split_start_go_s", "split_start_te_s", "transfer_go", "transfer_to"}
               | ({"split_cont_to_n", "split_cont_ge_s"} if n > 1 else set()))
    # H next to V inside the alignment: 'W' rows of the row child against bad columns of the column child
    forced("forced_h_next_to_v", "A" * 10 + "WWW" + "A" * 10, _block(rng, 2, _rand_letters(rng, 22)),
           list(range(1, 11)) + list(range(13, 23)), g_def, {"transfer_after_other_gap"})
    forced("forced_swapped_run_at_tile_start", "A" * 63 + "A" * 20, _block(rng, 2, _rand_letters(rng, 63 + 5 + 20)),
           list(range(1, 64)) + list(range(69, 89)), g_def, {"tile_start_prev_in_previous_tile", "swapped"}, swap=True)
    return out


def go_at_column1_cases() -> list[dict]:
    """Tables no rows give: the column child's column 1 counts a gap open (a gap in column 1 of a row is terminal, so
    GO[1] is 0 in every profile built from rows or merged from such), and a leading V run is followed by a D.  Only here
    is the rule "no open transfer when the run sat before the first column" observable; famsa_prof_put accepts such
    tables, and the C restatement of the reference's walk (dp_construct) is the oracle."""
    rng = np.random.default_rng(11)
    out = []
    gaps = (-14000, -1200, -3000, -500)
    for lead in (1, 3):
        rows = _block(rng, 3, _rand_letters(rng, 50))
        rows[1] = "-" + rows[1][1:]
        s = _crafted(("rows", rows), range(1, 51), gaps=gaps)[2]
        c = profiles.tables_from_rows(np.stack([codes(r) for r in rows]), score_matrix(), gaps)[1].copy()
        c[1, GO], c[1, TO] = c[1, TO], 0
        out.append(dict(name=f"go_at_column1_lead{lead}", a=("leaf", "W" * lead + "A" * 50), b=("rows", rows, s, c),
                        gaps=gaps, claims={"C_transfer_col1"}))
        # the same in the row child: two profiles (ProfProf), the relabeled one the DP's rows, a leading H run
        r_rows = ["A" * 50, "-" + "A" * 49]
        rc = profiles.tables_from_rows(np.stack([codes(r) for r in r_rows]), score_matrix(), gaps)[1].copy()
        rc[1, GO], rc[1, TO] = rc[1, TO], 0
        c_rows = ["W" * lead + "A" * 50, "Y" * lead + "C" * 50]
        out.append(dict(name=f"go_at_column1_rows_lead{lead}", a=("rows", r_rows, None, rc),
                        b=_crafted(("rows", c_rows), range(lead + 1, lead + 51), gaps=gaps), gaps=gaps,
                        claims={"R_transfer_col1", "not_swapped"}))
    return out


# ------------------------------------------------------------------ running a case
def tables_of(case):
    return child_tables(case["a"], case["gaps"]), child_tables(case["b"], case["gaps"])


def oracle_merge(case, t1=None, t2=None):
    """The C restatement: Align (dp_align) then the sequential ConstructProfile walk (dp_construct).  Returns
    (result dict, merged scores, merged counters)."""
    if t1 is None:
        t1, t2 = tables_of(case)
    res = pyoracle.dp_align(t1[0], t1[1], t1[2], t2[0], t2[1], t2[2], case["gaps"])
    rt, ct = (t2, t1) if res["swapped"] else (t1, t2)
    s, c, _, _ = pyoracle.dp_construct(rt, ct, res["path"], case["gaps"])
    return res, s, c


def crafted(case) -> bool:
    """Does a child of the case carry crafted scores (which the reference takes through RefDp.set_scores)?"""
    return any(len(ch) > 2 and ch[2] is not None for ch in (case["a"], case["b"]))


def reference_merge(case):
    """The reference's own Align + ConstructProfile on the same children (scores crafted where the case crafts them).
    Returns dict(total, scores, counters, card, kids = the children's tables as the reference holds them)."""
    dp = pyoracle.RefDp(0)
    dp.set_gaps(np.asarray(case["gaps"], dtype=np.int64))
    hs = []
    for k, ch in enumerate((case["a"], case["b"])):
        nos = [k] if ch[0] == "leaf" else list(range(2 + 200000 * k, 2 + 200000 * k + len(ch[1])))
        # a profile built from rows as text leaves out their last column (DESIGN §4e): one more, a gap in every row
        h = dp.leaf(ch[1], nos[0]) if ch[0] == "leaf" else dp.profile([r + "-" for r in ch[1]], nos)
        if len(ch) > 2 and ch[2] is not None:
            dp.set_scores(h, ch[2])
        hs.append(h)
    kids = [dp.tables(h) for h in hs]
    m, total = dp.align(hs[0], hs[1])
    s, c, card = dp.tables(m)
    dp.free(m)
    dp.close()
    return dict(total=total, scores=s, counters=c, card=card, kids=kids)


def tree_cases() -> list[dict]:
    """Small guide trees for align_tree: a chain of near-identical sequences (a queued child's bound w1 + w2 is about
    twice its real width, and the parent resolves the widths on the device) and a caterpillar of short leaves (later
    levels are single small merges: one fused launch, whose idle warps build the next level's leaves)."""
    rng = np.random.default_rng(77)
    base = _rand_letters(rng, 120)
    chain = [base] * 10 + [base[:60] + "W" + base[60:], base[:30] + base[31:]]
    n = len(chain)
    chain_tree = [(0, 1)] + [(n + k, k + 2) for k in range(n - 2)]
    fam = [_rand_letters(rng, int(rng.integers(30, 90))) for _ in range(6)]
    cat = [f[:int(rng.integers(0, 5))] + base[:80] + f[:int(rng.integers(0, 5))] for f in fam * 3]
    m = len(cat)
    cat_tree = [(0, 1)] + [(m + k, k + 2) for k in range(m - 2)]
    return [dict(name="chain_identical", seqs=chain, merges=chain_tree),
            dict(name="caterpillar", seqs=cat, merges=cat_tree)]


def crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def first_difference(got, want, path):
    """(column, lane, class of the column) of the first differing cell, for a failure message."""
    bad = np.argwhere(got != want)
    if not len(bad):
        return None
    k, lane = (int(x) for x in bad[0])
    if k == 0:
        return k, lane, "column 0"
    d, prev = int(path[k - 1]), int(path[k - 2]) if k >= 2 else 0
    kind = "D" if d == 0 else ("H" if d == 1 else "V") + (" continuing its run" if prev == d else " starting a run")
    if prev and prev != d:
        kind += f" after {'H' if prev == 1 else 'V'}"
    return k, lane, f"{kind}, tile column {k % TILE}"
