"""Times famsa_dist_export on the 10 000 x 400 aa bench family in input order, in all four -dist_export modes, and
the reference's DistanceCalculator writing the same file (oracle/_ref, where built) on all granted CPU threads.

One JSON line per mode: bytes, LCS tile-kernel ms and the rest of the call's kernels (Transform + text, plus the
few exact rows), wall time with a discarding sink and with a file in a temporary directory, the reference's wall
time, and whether the two files' SHA-256 agree.  The card's name and power limit come from nvidia-smi --query-gpu.

    python tools/dist_export_time.py [--n 10000] [--len 400] [--reps 3]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import famsa_b200  # noqa: E402
from famsa_b200 import seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402
import dist_export_oracle as O  # noqa: E402

LETTERS = "ARNDCQEGHILKMFPSTWYVBZX*"
MODES = (("dist", False, False), ("pid", False, True), ("dist_sq", True, False), ("pid_sq", True, True))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


class Discard:
    def write(self, b):
        return len(b)


def sha_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as fh:
        for blk in iter(lambda: fh.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--len", type=int, default=400)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    name, power = gpu_info()
    codes, offsets, lens = seqio.synth_family(a.n, a.len, seed=1, sort_desc=False)
    ids = [f"seq{i}" for i in range(a.n)]
    threads = len(os.sched_getaffinity(0))
    eng = famsa_b200.Engine(0)
    eng.upload(codes, offsets, lens)
    eng.dist_export(ids[:], pid=True, out=Discard())            # warm-up: allocations, pinned buffers
    have_ref = pyoracle.have("ref_dist")
    letters = ["".join(LETTERS[c] for c in codes[offsets[i]:offsets[i] + lens[i]]) for i in range(a.n)] if have_ref else None
    with tempfile.TemporaryDirectory() as tmp:
        for mode, square, pid in MODES:
            rec = dict(mode=mode, n=a.n, len=a.len, gpu=name, power_limit=power)
            walls = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                nbytes = eng.dist_export(ids, 0, square, pid, out=Discard())
                walls.append(time.perf_counter() - t0)
            total, main_ms, cells = eng.last_timing()
            rec.update(bytes=nbytes, cells=cells, lcs_kernel_ms=round(main_ms, 3), other_kernel_ms=round(total - main_ms, 3),
                       wall_discard_s=round(min(walls), 4))
            path = os.path.join(tmp, mode + ".csv")
            t0 = time.perf_counter()
            with open(path, "wb", buffering=0) as fh:
                eng.dist_export(ids, 0, square, pid, out=fh)
            rec["wall_file_s"] = round(time.perf_counter() - t0, 4)
            rec["sha256"] = sha_file(path)
            if have_ref:
                rpath = os.path.join(tmp, mode + ".ref.csv")
                t0 = time.perf_counter()
                O.ref_dist_export(letters, ids, 0, square, pid, path=rpath, n_threads=threads)
                rec["ref_wall_s"] = round(time.perf_counter() - t0, 4)
                rec["ref_threads"] = threads
                rec["sha256_equal"] = sha_file(rpath) == rec["sha256"]
                os.unlink(rpath)
            os.unlink(path)
            print(json.dumps(rec), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
