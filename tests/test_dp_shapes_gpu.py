"""GPU tests of every profile-DP fill path at its stripe, chunk and T-arithmetic boundaries (cases: tests/dp_shapes.py).

Every merge is compared with the oracle (pyoracle.dp_align): total, last, path, orientation, variant and the whole
direction matrix.  Each launch shape is forced with the development knobs and the `[dp]` debug line must report the
class (and, for teams, the team width and whether the compact kernel ran) the shape stands for."""
import re

import numpy as np
import pytest

import dp_shapes as D
from oracle import pyoracle

pytestmark = pytest.mark.gpu

LINE = re.compile(r"\[dp\] batch of (\d+): class (\d+) x (\d+) .*?cl_cap (\d+), latency_mode (\d)(?:, team (\d+), compact (\d))?")
_want = {}


def oracle(job, gaps, key=None):
    if key is None or key not in _want:
        w = pyoracle.dp_align(*job, gaps)
        if key is None:
            return w
        _want[key] = w
    return _want[key]


def assert_same(got, want, what):
    assert got["variant"] == want["variant"] and got["swapped"] == want["swapped"], what
    assert got["total"] == want["total"], f"{what}: total {got['total']} != {want['total']}"
    assert np.array_equal(got["last"], want["last"]), what
    assert np.array_equal(got["path"], want["path"]), f"{what}: path differs"
    if "dirs" in got:
        assert np.array_equal(got["dirs"], want["dirs"]), f"{what}: direction matrix differs"


def run_shape(engine, monkeypatch, capfd, shape, jobs, gaps):
    """The batch under the shape's knobs; returns (results, [(class, merges, cl_cap, team, compact) per class line])."""
    for k in ("FAMSA_DP_LATENCY_MODE", "FAMSA_DP_TEAM_MIN", "FAMSA_DP_TEAM_WARPS", "FAMSA_DP_CLUSTER_MIN",
              "FAMSA_DP_MAX_CLUSTER", "FAMSA_DP_DUO", "FAMSA_DP_COMPACT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (shape["env"] if shape else {}).items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("FAMSA_DP_DEBUG", "1")
    capfd.readouterr()
    got = engine.dp_align_batch(jobs, gaps, want_dirs=True)
    err = capfd.readouterr().err
    lines = [(int(m[2]), int(m[3]), int(m[4]), m[6] and int(m[6]), m[7] and int(m[7])) for m in LINE.finditer(err)]
    assert lines, "no [dp] class line"
    return got, lines


def check_classes(shape, lines, jobs):
    """Every class line is the one the shape stands for; skips (with the reason) what the device does not allow."""
    cl_cap = lines[0][2]
    if "cl" in shape and shape["cl"] > cl_cap:
        pytest.skip(f"the device allows clusters of up to {cl_cap} blocks of the 4-warp fill kernel, not {shape['cl']}")
    got = {c: n for c, n, *_ in lines}
    if shape["cls"] >= 100:
        duo = [c for c in got if c >= 100]
        if shape["cl"] == 16 and duo and max(duo) < 116:
            pytest.skip(f"the device allows producer / consumer clusters of up to {max(duo) - 100} blocks, not 16")
    assert got == D.expected_classes(jobs, shape, cl_cap, shape.get("cl", cl_cap)), (shape["name"], got)
    assert shape["cls"] in got
    if shape["cls"] == 1:
        assert {(t, c) for c_, n, cap, t, c in lines} == {shape["team"]}, lines


@pytest.fixture(scope="module")
def engine():
    import famsa_b200
    e = famsa_b200.Engine(0)
    yield e
    e.close()


@pytest.mark.parametrize("name", [s["name"] for s in D.LAUNCH_SHAPES])
def test_geometry(engine, monkeypatch, capfd, name):
    """Stripe counts 1, TW-1, TW, TW+1, 2TW+1, WR mod 32 in {0, 1, 31}, WC around the steady-state gate, the rings and
    the prep scan, SeqSeq / SeqProf / ProfProf -- under the launch shape, against the oracle."""
    shape = D.SHAPES[name]
    jobs, meta = D.geometry_jobs(shape["tw"], max_min_width=256 if shape["cls"] == 1 else None)
    got, lines = run_shape(engine, monkeypatch, capfd, shape, jobs, D.GAPS)
    for k, (r, j, m) in enumerate(zip(got, jobs, meta)):
        assert_same(r, oracle(j, D.GAPS, ("geo", shape["tw"], shape["cls"] == 1, k)), f"{name} job {k} {m}")
    check_classes(shape, lines, jobs)


@pytest.mark.parametrize("name", [None] + D.ARITH_SHAPES)
def test_arithmetic_matrix(engine, monkeypatch, capfd, name):
    """VAR x 4/8-byte T ring, ProfProf x tmode 0/1/2 on both sides of every decision, extreme score digits and |T| at the
    4-byte bound -- one mixed batch, so the compact kernel leaves its 8-byte merges to the launch behind it."""
    cases = D.arithmetic_cases()
    jobs = [j for _, j, _ in cases]
    shape = D.SHAPES[name] if name else None
    got, lines = run_shape(engine, monkeypatch, capfd, shape, jobs, D.GAPS)
    for r, (cname, j, _) in zip(got, cases):
        assert_same(r, oracle(j, D.GAPS, ("arith", cname)), f"{name}: {cname}")
    if shape:
        check_classes(shape, lines, jobs)


@pytest.mark.parametrize("name", [None, "one_warp", "compact4", "latency_cl2", "duo_cl2"])
def test_overflow_witness(engine, monkeypatch, capfd, name):
    """A row profile whose column counters sum to 10 x its members (every check of the prep kernel passes) against column
    scores under the old 4-byte threshold: |T| reaches ~1.3 x 2^31 and must not be truncated to 32 bits."""
    job = D.overflow_witness()
    shape = D.SHAPES[name] if name else None
    got, _ = run_shape(engine, monkeypatch, capfd, shape, [job], D.GAPS)
    assert_same(got[0], oracle(job, D.GAPS, ("witness",)), f"overflow witness under {name}")


def test_traceback_windows(engine, monkeypatch, capfd):
    """Paths with runs past the 64-step synchronous window and stripe exits outside the speculative window's slack."""
    cases = D.traceback_cases()
    for shape in (None, D.SHAPES["one_warp"], D.SHAPES["latency_cl2"]):
        got, _ = run_shape(engine, monkeypatch, capfd, shape, [j for _, j in cases], D.RUN_GAPS)
        for r, (cname, j) in zip(got, cases):
            assert_same(r, oracle(j, D.RUN_GAPS, ("trace", cname)), cname)


def test_orientation_tie(engine, monkeypatch, capfd):
    cases = D.tie_cases()
    got, _ = run_shape(engine, monkeypatch, capfd, None, [j for _, j in cases], D.GAPS)
    for r, (delta, j) in zip(got, cases):
        assert r["swapped"] == (delta >= 0)
        assert_same(r, oracle(j, D.GAPS), f"tie {delta}")


def _resident(engine, jobs, gaps):
    """famsa_prof_put + famsa_prof_merge_batch; returns (results, merged tables)."""
    profs = []
    for j in jobs:
        profs += [j[:3], j[3:]]
    ids = engine.prof_put(profs)
    pairs = [(ids[2 * k], ids[2 * k + 1]) for k in range(len(jobs))]
    widths = [(j[0].shape[0] - 1, j[3].shape[0] - 1) for j in jobs]
    mids, res = engine.prof_merge_batch(pairs, gaps, widths)
    tables = [engine.prof_get(m) for m in mids]
    engine.prof_drop(mids)
    return res, tables


def _check_resident(res, tables, jobs, gaps, what):
    for k, (r, t, j) in enumerate(zip(res, tables, jobs)):
        want = oracle(j, gaps)
        assert_same(r, want, f"{what} merge {k}")
        rp, cp = (j[3:], j[:3]) if want["swapped"] else (j[:3], j[3:])
        s, c, _, _ = pyoracle.dp_construct(rp, cp, want["path"], gaps)
        assert t[2] == j[2] + j[5]
        assert np.array_equal(t[1], c) and np.array_equal(t[0], s), f"{what} merge {k}: merged tables differ"


@pytest.mark.parametrize("fused", ["0", "1"])
def test_resident_fused_limit(engine, monkeypatch, fused):
    """Merges just inside and just outside the fused kernel's limit for keeping the direction matrix in shared memory,
    through the resident path with and without the fused kernel; merged tables against dp_construct."""
    monkeypatch.setenv("FAMSA_PROF_FUSED", fused)
    cases = D.fused_limit_cases()
    jobs = [j for *_, j in cases]
    for k in range(len(jobs)):                                        # one merge per launch: each decides alone
        res, tables = _resident(engine, [jobs[k]], D.GAPS)
        _check_resident(res, tables, [jobs[k]], D.GAPS, f"fused={fused} {cases[k][:3]}")


@pytest.mark.parametrize("fused", ["0", "1"])
def test_resident_arithmetic(engine, monkeypatch, fused):
    """The arithmetic matrix and the overflow witness through famsa_prof_put + famsa_prof_merge_batch (fused kernel or
    the batched kernels): paths, totals and merged tables."""
    monkeypatch.setenv("FAMSA_PROF_FUSED", fused)
    cases = D.arithmetic_cases()
    jobs = [j for _, j, _ in cases if j[0].shape[0] <= 513] + [D.overflow_witness()]
    res, tables = _resident(engine, jobs, D.GAPS)
    _check_resident(res, tables, jobs, D.GAPS, f"fused={fused}")
