"""Times famsa_lcs_slink (-gt slink) on the 10 000 x 400 aa bench family (C2) and on 40 000 x 60 aa, both in FAMSA's
length-descending order, and the reference's SingleLinkage<indel075_div_lcs>::run on the same set (oracle/_ref, where
built) on all granted CPU threads.

One JSON line per set: the call's device time (LCS tile kernels, and all kernels) and wall time (best of --reps, after a
warm-up call), for the Boruvka rounds and for the sequential loop (FAMSA_PRIM_SEQUENTIAL), whether the two trees agree,
the reference's wall time and whether its tree is the same.  The card's name and power limit come from nvidia-smi.

    python tools/slink_time.py [--reps 3] [--no-ref]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import famsa_b200  # noqa: E402
from famsa_b200 import seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402
import slink_oracle as S  # noqa: E402

SETS = (("C2", 10000, 400, 1), ("40k", 40000, 60, 45))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def timed(eng, reps):
    eng.slink(0)                                             # warm-up: allocations of this shape
    walls, dev = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        tree = eng.slink(0)
        walls.append(time.perf_counter() - t0)
        dev.append(eng.last_timing())
    best = int(np.argmin(walls))
    total, main_ms, pairs = dev[best]
    return tree, dict(wall_s=round(walls[best], 4), device_ms=round(total, 2), lcs_kernel_ms=round(main_ms, 2), pairs=pairs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    name, power = gpu_info()
    threads = len(os.sched_getaffinity(0))
    for label, n, length, seed in SETS:
        codes, offsets, lens = seqio.synth_family(n, length, seed=seed)
        eng = famsa_b200.Engine(0)
        try:
            eng.upload(codes, offsets, lens)
            tree, boruvka = timed(eng, a.reps)
            os.environ["FAMSA_PRIM_SEQUENTIAL"] = "1"
            try:
                tree_seq, sequential = timed(eng, a.reps)
            finally:
                del os.environ["FAMSA_PRIM_SEQUENTIAL"]
        finally:
            eng.close()
        rec = dict(set=label, n=n, len=length, gpu=name, power_limit=power, boruvka=boruvka, sequential=sequential,
                   engines_agree=bool(np.array_equal(tree, tree_seq)))
        if pyoracle.have("ref_slink") and not a.no_ref:
            letters = [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(offsets, lens)]
            t0 = time.perf_counter()
            want = S.ref_slink_tree(letters, 0, n_threads=threads)
            rec.update(ref_threads=threads, ref_wall_s=round(time.perf_counter() - t0, 3), same_as_ref=bool(np.array_equal(tree, want)))
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
