"""Times famsa_lcs_nj (-gt nj) on 2 000 and 10 000 (C2) x 400 aa bench families in FAMSA's length-descending order, and
the reference's NeighborJoining<indel075_div_lcs>::run on the same set (oracle/_ref, where built; one thread, as its
distance matrix and computeTree run) up to --ref-max sequences.

One JSON line per set: the call's device time (all kernels; the LCS tile kernels alone; the rest = distances, sums and
the agglomeration) and wall time, best of --reps after a warm-up call, the reference's wall time and whether its tree is
the same.  The card's name and power limit come from nvidia-smi in the same run.

    python tools/nj_time.py [--reps 3] [--ref-max 2000]
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
import nj_oracle as N  # noqa: E402

SETS = (("2k", 2000, 400, 1), ("C2", 10000, 400, 1))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def timed(eng, reps):
    eng.nj(0)                                                # warm-up: allocations of this shape
    walls, dev = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        tree = eng.nj(0)
        walls.append(time.perf_counter() - t0)
        dev.append(eng.last_timing())
    best = int(np.argmin(walls))
    total, main_ms, pairs = dev[best]
    return tree, dict(wall_s=round(walls[best], 4), device_ms=round(total, 2), lcs_kernel_ms=round(main_ms, 2),
                      tree_ms=round(total - main_ms, 2), pairs=pairs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-max", type=int, default=2000)
    a = ap.parse_args()
    name, power = gpu_info()
    for label, n, length, seed in SETS:
        codes, offsets, lens = seqio.synth_family(n, length, seed=seed)
        eng = famsa_b200.Engine(0)
        try:
            eng.upload(codes, offsets, lens)
            tree, dev = timed(eng, a.reps)
        finally:
            eng.close()
        rec = dict(set=label, n=n, len=length, gpu=name, power_limit=power, device=dev)
        if pyoracle.have("ref_nj") and n <= a.ref_max:
            letters = [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(offsets, lens)]
            want, sec = N.ref_tree(letters, 0)
            rec.update(ref_threads=1, ref_wall_s=round(sec, 3), same_as_ref=bool(np.array_equal(tree, want)))
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
