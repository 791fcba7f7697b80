"""CPU tests of the DP launch planner (famsa_b200/csrc/dp_plan.h), compiled alone with g++ into tests/cpp/dp_plan_check.cpp.

The knobs go through the environment as in the library.  For every launch shape of tests/dp_shapes.py and the batches
test_dp_shapes_gpu.py runs, the planner must give the classes, team widths and `[dp]` lines the GPU test asserts -- here
also for the cluster caps a given H100 may not allow.  Throughput mode must deal the team merges in snake rows, and
the sub-batch cut must respect FAMSA_DP_MAX_CELLS."""
import functools
import os
import re
import subprocess

import numpy as np
import pytest

import dp_shapes as D
from cpp_build import build_cpp
from test_dp_shapes_gpu import LINE

SMS = 132
CAPS = [(8, 8), (16, 8), (16, 16)]                                   # (4-warp cluster cap, producer / consumer cluster cap)
KNOBS = ("FAMSA_DP_MAX_CELLS", "FAMSA_DP_TEAM_MIN", "FAMSA_DP_TEAM_WARPS", "FAMSA_DP_CLUSTER_MIN", "FAMSA_DP_MAX_CLUSTER",
         "FAMSA_DP_LATENCY_MODE", "FAMSA_DP_DUO", "FAMSA_DP_COMPACT", "FAMSA_DP_DEBUG")
# the whole line as dp.cu prints it
FULL_LINE = re.compile(r"\[dp\] batch of \d+: class \d+ x \d+ \(first \d+ x \d+, \d+ stripes\), demand \d+, cl_cap \d+, "
                       r"latency_mode [01](, team \d+, compact [01])?")


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    return build_cpp("dp_plan_check", tmp_path_factory.mktemp("dp_plan"))


def dims(jobs):
    return [(j[0].shape[0] - 1, j[2], j[3].shape[0] - 1, j[5]) for j in jobs]


def plan(exe, batch, env, caps=(16, 16)):
    """The planner on [(w1, card1, w2, card2)] under `env`: one dict per sub-batch."""
    e = {k: v for k, v in os.environ.items() if k not in KNOBS}
    e.update(env)
    # the kernel shapes as tests/dp_shapes.py has them (test_dp_shapes_host.py checks them against dp.cu)
    args = [exe, str(SMS), str(caps[0]), str(caps[1]), str(D.K_DP_TEAM_WARPS), str(D.K_DP_CLUSTER)]
    out = subprocess.run(args, input="".join("%d %d %d %d\n" % m for m in batch), env=e, capture_output=True, text=True,
                         check=True).stdout
    subs = []
    for line in out.splitlines():
        w = line.split()
        if w[0] == "sub":
            subs.append(dict(j0=int(w[1]), j1=int(w[2]), order=None, launches=[], lines=[]))
        elif w[0] == "order":
            subs[-1]["order"] = [int(x) for x in w[1:]]
        elif w[0] == "launch":
            subs[-1]["launches"].append(tuple(int(x) for x in w[1:]))   # cls kernel nw cluster wide_only q0 q1 slot
        else:
            subs[-1]["lines"].append(line)
    return subs


@functools.lru_cache(maxsize=None)
def geometry(tw, cap):
    return D.geometry_jobs(tw, max_min_width=cap)[0]


@functools.lru_cache(maxsize=None)
def mixed():
    return D.mixed_batch()


CASES = [(s["name"], "geometry") for s in D.LAUNCH_SHAPES] + [(name, "mixed") for name in D.ARITH_SHAPES]


@pytest.mark.parametrize("caps", CAPS, ids=lambda c: "cl%d_duo%d" % c)
@pytest.mark.parametrize("name,batch", CASES)
def test_launch_classes(planner, name, batch, caps):
    """The classes test_dp_shapes_gpu.py's check_classes asserts (dp_shapes.expected_classes), from the real planner."""
    shape = D.SHAPES[name]
    jobs = geometry(shape["tw"], 256 if shape["cls"] == 1 else None) if batch == "geometry" else mixed()
    (sub,) = plan(planner, dims(jobs), dict(shape["env"], FAMSA_DP_DEBUG="1"), caps)
    assert all(FULL_LINE.fullmatch(t) for t in sub["lines"]), sub["lines"]
    matches = [LINE.fullmatch(t) for t in sub["lines"]]
    assert all(matches), sub["lines"]
    lines = [(int(m[1]), int(m[2]), int(m[3]), int(m[4]), m[6] and int(m[6]), m[7] and int(m[7])) for m in matches]
    assert len(lines) == len({L[0] for L in sub["launches"]})         # one line per class
    assert {m for m, *_ in lines} == {len(jobs)} and sum(n for _, _, n, *_ in lines) == len(jobs)
    cl_cap = lines[0][3]
    assert cl_cap == min(caps[0], shape.get("cl", caps[0]))
    got = {c: n for _, c, n, *_ in lines}
    assert got == D.expected_classes(jobs, shape, cl_cap, caps[1]), (name, got)
    if shape.get("cl", 0) <= cl_cap and (shape["cls"] < 100 or shape["cl"] <= caps[1]):
        assert shape["cls"] in got                                     # the shape reaches its class where the caps allow it
    if shape["cls"] == 1:
        assert {(t, c) for *_, t, c in lines} == {shape["team"]}, lines


@pytest.mark.parametrize("compact", ["0", "1"])
def test_snake_order(planner, compact):
    """Throughput mode: classes in descending order, each sorted by size; team merges dealt in rows of one per SM,
    every other row reversed, so that a row never holds a merge larger than one of the row before."""
    rng = np.random.default_rng(3)
    batch = [(int(a), 3, int(b), 5) for a, b in rng.integers(100, 700, size=(700, 2))] + \
            [(int(a), 1, int(b), 1) for a, b in rng.integers(10, 90, size=(50, 2))]
    (sub,) = plan(planner, batch, {"FAMSA_DP_LATENCY_MODE": "0", "FAMSA_DP_COMPACT": compact})
    order, size = sub["order"], [w1 * w2 for w1, _, w2, _ in batch]
    assert sorted(order) == list(range(len(batch)))
    classes = [L for L in sub["launches"] if not L[4]]
    assert [L[0] for L in classes] == [1, 0]
    assert [(L[1], L[2]) for L in sub["launches"]] == ([(1, 4), (0, 4)] if compact == "1" else [(0, 2)]) + [(0, 1)]
    for cls, _, _, _, _, q0, q1, _ in classes:
        rows = [[size[j] for j in order[r:min(q1, r + SMS)]] for r in range(q0, q1, SMS)] if cls == 1 else [[size[j] for j in order[q0:q1]]]
        assert cls != 1 or len(rows) > 2
        for i, row in enumerate(rows):
            assert row == sorted(row, reverse=i % 2 == 0)
            assert i == 0 or max(row) <= min(rows[i - 1])


def test_sub_batch_cut(planner):
    """FAMSA_DP_MAX_CELLS=60000 (test_dp_gpu.py's value): consecutive sub-batches, none above the limit unless it is a
    single merge, each cut where the next merge would cross it."""
    rng = np.random.default_rng(5)
    batch = [(int(a), 1, int(b), int(c)) for a, b, c in zip(rng.integers(1, 400, 300), rng.integers(1, 400, 300), rng.integers(1, 9, 300))]
    limit = 60000
    subs = plan(planner, batch, {"FAMSA_DP_MAX_CELLS": str(limit)})
    cells = [(w1 + 1) * (w2 + 1) for w1, _, w2, _ in batch]
    assert [s["j0"] for s in subs] == [0] + [s["j1"] for s in subs[:-1]] and subs[-1]["j1"] == len(batch)
    assert any(s["j1"] - s["j0"] == 1 and cells[s["j0"]] > limit for s in subs)
    for s in subs:
        total = sum(cells[s["j0"]:s["j1"]])
        assert total <= limit or s["j1"] - s["j0"] == 1
        assert s["j1"] == len(batch) or total + cells[s["j1"]] > limit
        assert sorted(s["order"]) == list(range(s["j0"], s["j1"]))
