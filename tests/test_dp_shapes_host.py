"""CPU tests of tests/dp_shapes.py: the generator is built on dp.cu's constants, every case carries the label it claims
(computed exactly from its tables), the arithmetic matrix reaches every cell on the side it claims, the traceback cases
produce the window events they are for, and the linear construction of large profiles equals the tables of the explicit
rows -- and, where the reference is built, the reference's own tables and alignment."""
import os
import re

import numpy as np
import pytest

import dp_shapes as D
from famsa_b200 import profiles
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "famsa_b200", "csrc", "dp.cu")).read()


def constexpr(name: str) -> int:
    m = re.search(rf"constexpr\s+(?:int|uint32_t|size_t)\s+{name}\s*=\s*(\d+)\s*;", SRC)
    assert m, name
    return int(m.group(1))


def test_constants_match_dp_cu():
    for name, value in (("kChunk", D.K_CHUNK), ("kRing", D.K_RING), ("kTRing", D.K_TRING), ("kTraceWin", D.K_TRACE_WIN),
                        ("kSpecSlack", D.K_SPEC_SLACK), ("kDpWarps", D.K_DP_WARPS), ("kDpTeamWarps", D.K_DP_TEAM_WARPS),
                        ("kDpCluster", D.K_DP_CLUSTER), ("kFusedWarps", D.K_FUSED_WARPS), ("kColFields", D.K_COL_FIELDS),
                        ("kS2Stride", D.K_S2_STRIDE), ("kPrepThreads", D.K_PREP_THREADS)):
        assert constexpr(name) == value, name
    # the digit limits of the tmode decision and the steady-state gate
    assert re.search(r"nR <= %d \? 0 : \(nR <= %d \? 1 : 2\)" % (D.DIGIT1_MAX, D.DIGIT2_MAX), SRC)
    assert len(re.findall(r"m >= 5 && s_begin \+ kChunk - 1 < WC", SRC)) == 2
    # the synchronous traceback window and the fused kernel's shared-memory limit for the direction matrix
    assert "wsb = st_hi >= %d ? st_hi - %d : 0;" % (D.SYNC_WIN - 1, D.SYNC_WIN - 1) in SRC
    assert "bytes <= kFusedWarps * sizeof(WarpShared)" in SRC
    # WarpShared: the fields the generator's size is made of, in order
    body = re.search(r"struct __align__\(16\) WarpShared \{(.*?)\n\};", SRC, re.S).group(1)
    fields = re.findall(r"^\s+(?:Cell|long long) (\w+)((?:\[\w+\])+);", body, re.M)
    assert fields == [("brow", "[2][kChunk]"), ("col", "[kColFields][kRing]"), ("s2", "[2][kChunk][kS2Stride]"),
                      ("park", "[kChunk][3]"), ("t", "[kTRing][32]")]
    assert D.WARP_SHARED_BYTES % 16 == 0


def test_stripe_counts_and_geometry():
    for s in D.LAUNCH_SHAPES:
        tw = s["tw"]
        cap = 256 if s["cls"] == 1 else None
        jobs, meta = D.geometry_jobs(tw, max_min_width=cap)
        assert {m["stripes"] for m in meta} == set(D.stripe_counts(tw)) == {1, max(1, tw - 1), tw, tw + 1, 2 * tw + 1}
        assert {m["wr"] % 32 for m in meta} == set(D.WR_RESIDUES)
        for m in meta:
            assert (m["wr"] + 31) // 32 == m["stripes"]
        wcs = [m["wc"] for m in meta]
        want = set(D.GEOMETRY_WC) if cap is None else {w for w in D.GEOMETRY_WC if w <= 256}
        assert set(wcs) >= want
        if cap is not None:
            assert all(min(j[0].shape[0], j[3].shape[0]) - 1 <= cap for j in jobs)
        labels = [D.label(j) for j in jobs]
        assert {L["var"] for L in labels} == {0, 1, 2}
        for L, m, j in zip(labels, meta, jobs):
            assert (L["wr"], L["wc"], L["var"]) == (m["wr"], m["wc"], m["var"]), m
    one = D.SHAPES["one_warp"]
    assert len(D.geometry_jobs(one["tw"])[0]) % D.K_DP_WARPS != 0                    # a partial last block


def test_latency_shapes_reach_their_cluster_size():
    """Under every latency shape some merges get exactly the shape's cluster size (the host's own rule, mirrored)."""
    for name, s in D.SHAPES.items():
        if s["cls"] < 10:
            continue
        jobs, _ = D.geometry_jobs(s["tw"])
        got = D.expected_classes(jobs, s, cl_cap=s["cl"], duo_cap=s["cl"])
        assert got.get(s["cls"], 0) >= 1, (name, got)


def test_arithmetic_matrix_is_covered():
    """Every cell of VAR x ring width, and of ProfProf tmode x ring width, is reached on the side each case claims; the
    4-byte cases at the bound carry |T| = 7 x card x threshold, within a handful of 2^31."""
    cells = set()
    for name, job, claims in D.arithmetic_cases():
        L = D.label(job)
        for k, v in claims.items():
            assert L[k] == v, (name, k, L[k], v)
        if L["t32"]:
            assert L["tmax"] < 2 ** 31, name                          # the ring's width is sound
        cells.add((L["var"], L["t32"], L["tmode"] if L["var"] == 2 else None, L["wide"] if L["var"] == 2 else None))
        if name.startswith("pp_bound") and L["t32"]:
            assert 2 ** 31 - L["tmax"] <= 7 * L["nr"] * 2, name
    for var in (0, 1):
        assert (var, True, None, None) in cells and (var, False, None, None) in cells
    for tmode in (0, 1, 2):
        assert (2, True, tmode, False) in cells and (2, False, tmode, False) in cells
    assert (2, False, 2, True) in cells                               # tmode 2 through scores beyond int32
    names = [n for n, _, _ in D.arithmetic_cases()]
    for nr in (127, 128, 255, 256, 32767, 32768, 40000):
        assert f"pp_n{nr}_t32" in names and f"pp_n{nr}_t64" in names


def test_digit_cells():
    """tmode-1 row profiles hold counters >= 256 (a high digit) next to counters in 128..255 (an unsigned low digit);
    the extreme-digit column scores contain INT32_MIN, INT32_MAX, -1 and low bytes 0x80 / 0xFF."""
    for name, job, claims in D.arithmetic_cases():
        L = D.label(job)
        if L["var"] != 2 or L["wide"] or L["nr"] < 600:
            continue
        c = (job[4] if L["sw"] else job[1])[1:, :30]
        assert (c >= 256).any() and ((c >= 128) & (c <= 255)).any(), name
    ext = [job for name, job, _ in D.arithmetic_cases() if name.endswith("extreme_digits")]
    for job in ext:
        v = job[3][1:, :30]
        for x in (D.I32_MIN, D.I32_MAX, -1):
            assert (v == x).any()
        assert ((v & 0xFF) == 0x80).any() and ((v & 0xFF) == 0xFF).any()
    small = [job for name, job, _ in D.arithmetic_cases() if name.endswith("small_digits")]
    for job in small:
        v = job[3][1:, :30]
        assert ((v & 0xFF) == 0x80).any() and ((v & 0xFF) == 0xFF).any() and (v == -1).any()


def test_overflow_witness_labels():
    """The witness passes every check of the prep kernel, sits on the row side, and its |T| leaves int32 while its
    column scores are under the old 4-byte threshold: a ring chosen from max|score| alone is wrong for it."""
    job = D.overflow_witness()
    L = D.label(job)
    assert L["var"] == 2 and L["sw"] == 0                             # the stacked profile is the row side
    assert D.nz(job[1]) * (job[3].shape[0] - 1) < D.nz(job[4]) * (job[0].shape[0] - 1)
    c = job[1]
    assert (c >= 0).all() and (c[:, :30] <= job[2]).all()
    assert L["csum"] == 10 * L["nr"] > 7 * L["nr"]
    assert L["t32_old"] and not L["t32"] and L["tmax"] > 2 ** 31
    r = pyoracle.dp_align(*job, D.GAPS)
    assert r["variant"] == 2 and not r["swapped"]


def test_traceback_events():
    """On the oracle's path: a run of more than 64 moves inside one stripe (past the synchronous window), and stripe exits
    more than kSpecSlack columns left and right of the diagonal the speculative window predicts."""
    longest, devs = 0, []
    for name, job in D.traceback_cases():
        r = pyoracle.dp_align(*job, D.RUN_GAPS)
        L = D.label(job)
        assert r["swapped"] == bool(L["sw"])
        lo, dv = D.walk(r["path"], L["wr"], L["wc"])
        longest, devs = max(longest, lo), devs + dv
    assert longest > D.SYNC_WIN
    assert max(devs) > D.K_SPEC_SLACK and min(devs) < -D.K_SPEC_SLACK


def test_walk_on_known_paths():
    # all-D through 64 rows: two stripe visits of 32 moves, the exit exactly on the prediction
    lo, dv = D.walk(np.zeros(64, dtype=np.uint8), 64, 64)
    assert lo == 32 and dv == [0]
    # 100 H moves on row 33, then 33 V moves: the first visit is 100 + 1 moves long
    path = np.array([2] * 33 + [1] * 100, dtype=np.uint8)
    lo, dv = D.walk(path, 33, 100)
    assert lo == 101 and dv == [-99]


def test_orientation_tie():
    for delta, job in D.tie_cases():
        w1, w2 = job[0].shape[0] - 1, job[3].shape[0] - 1
        assert D.nz(job[1]) * w2 - D.nz(job[4]) * w1 == delta
        want_sw = 0 if delta < 0 else 1
        assert D.label(job)["sw"] == want_sw
        assert pyoracle.dp_align(*job, D.GAPS)["swapped"] == bool(want_sw)


def test_fused_limit_cases():
    cases = D.fused_limit_cases()
    assert [fits for *_, fits, _ in cases] == [True, False, True, False]
    for wr, wc, fits, job in cases:
        L = D.label(job)
        assert (L["wr"], L["wc"], L["var"], L["sw"]) == (wr, wc, 1, 0)
        b = D.fused_dirs_bytes(wr, wc)
        assert (b <= D.FUSED_DIRS_LIMIT) == fits and (fits or b - D.FUSED_DIRS_LIMIT <= (wr + 31) // 32 * 32)


@pytest.mark.parametrize("card", [127, 128, 255, 256, 32767, 32768, 40000])
def test_linear_profile_equals_explicit_rows(card):
    rng = np.random.default_rng(card)
    sm = D.score_matrix(8)
    blocks, mult = D.linear_blocks(card, 37, rng)
    lin = D.add_tables([(m, profiles.tables_from_rows(b, sm, D.GAPS)) for m, b in zip(mult, blocks)])
    exp = profiles.tables_from_rows(D.expand_rows(blocks, mult), sm, D.GAPS)
    assert lin[2] == exp[2] == card
    assert np.array_equal(lin[1], exp[1]) and np.array_equal(lin[0], exp[0])


def _gapped(rows) -> list[str]:
    """Gapped strings for the reference's string constructor, whose width is the string length - 1 (see
    test_profiles_host.py): one more column that continues every row's trailing gap or residue."""
    from famsa_b200 import seqio
    last = np.where(rows[:, -1:] < 0, -1, 0)
    last[0, 0] = 0
    return ["".join("-" if x < 0 else seqio.ALPHABET[x] for x in r) for r in np.concatenate([rows, last], axis=1)]


@pytest.mark.skipif(not pyoracle.have_ref(), reason="oracle/_ref/libfamsa_ref.so not built")
@pytest.mark.parametrize("card,wide", [(128, False), (300, False), (32768, False), (40000, False), (200, True)])
def test_oracle_equals_reference_on_large_profiles(card, wide):
    """The reference's CProfile from the explicit gapped rows has the linear construction's tables, and its Align gives
    the oracle's total and path -- far above the member counts of the realistic families (wide: gap costs x 300000,
    column scores beyond int32)."""
    rng = np.random.default_rng(card + wide)
    dp = pyoracle.RefDp(8)
    try:
        if wide:
            dp.set_gaps(dp.gaps() * 300_000)
        g, sm = dp.gaps(), dp.score_matrix()
        blocks, mult = D.linear_blocks(card, 45, rng)
        rows = D.expand_rows(blocks, mult)
        other = D.block_rows(20, rng.integers(0, 20, size=52), rng, sub=0.9)
        big = D.add_tables([(m, profiles.tables_from_rows(b, sm, g)) for m, b in zip(mult, blocks)])
        small = profiles.tables_from_rows(other, sm, g)
        pa = dp.profile(_gapped(rows), list(range(card)))
        pb = dp.profile(_gapped(other), list(range(card, card + 20)))
        for p, t in ((pa, big), (pb, small)):
            s, c, k = dp.tables(p)
            assert k == t[2] and np.array_equal(c, t[1]) and np.array_equal(s, t[0])
        if wide:
            assert np.abs(small[0][1:, :30]).max() > 2 ** 31 or np.abs(big[0][1:, :30]).max() > 2 ** 31
        want = pyoracle.dp_align(*big, *small, g)
        m, total = dp.align(pa, pb)
        got_rows = dp.rows(m)
        dp.free(m)
        assert total == want["total"]
        path = pyoracle.path_from_rows(got_rows, set(range(card)), set(range(card, card + 20)), want["swapped"])
        assert np.array_equal(path[:len(want["path"])], want["path"])     # (the rows carry the constructor's extra column)
    finally:
        dp.close()
