"""Times famsa_prof_tree_rows -- the final alignment's rows built on the device from famsa_prof_align_tree's paths -- next
to what it replaces and what it follows:

  * hemopexin (4 188 sequences) under its default single-linkage tree and its medoid-sl tree (tests/golden);
  * synth_family(2000, 400) and synth_family(10000, 400) under a default-style single-linkage tree (famsa_lcs_slink);
  * a pure chain of 10 000 leaves (synth_family(10000, 60), each merge adds the next sequence).

One JSON line per set: tree_rows' device time (torch.profiler: the call's kernels, memsets and copies, and k_tree_rows
alone) and wall time, with and without the download of the rows (best of --reps after a warm-up call); the
famsa_prof_align_tree call on the same tree (wall and device ms); the Python dp_cases.assemble_rows on the same paths
(where n <= --host-max, it copies every member row at every merge); and, where oracle/_ref is built and n <= --ref-max,
the reference's time.alignment (ref_align_tree_mt, all granted CPU threads).  The card's name and power limit come from
nvidia-smi.  Every set also checks the device rows against assemble_rows where that ran.

    python tools/tree_rows_time.py [--reps 5] [--host-max 4200] [--ref-max 4200]
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
import dp_cases  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def device_ms(fn):
    """Device time of what fn() queues, from torch.profiler (CUPTI sees the library's own stream): every kernel, memset
    and copy, and k_tree_rows alone."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    total = kern = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if not t or e.key.startswith("cudaDevice"):
            continue
        total += t
        if "k_tree_rows" in e.key:
            kern += t
    return total / 1e3, kern / 1e3


def sets():
    yield from (("hemopexin_sl", "hemopexin_sl"), ("hemopexin_medoid_sl", "hemopexin_medoid_sl"))
    yield ("synth_2000x400_slink", (2000, 400, 1))
    yield ("synth_10000x400_slink", (10000, 400, 1))
    yield ("chain_10000x60", "chain")


def load(eng, spec):
    if isinstance(spec, str) and spec != "chain":
        z = np.load(os.path.join(GOLDEN, spec + ".npz"))
        t = np.load(os.path.join(GOLDEN, "adeno_upgma_merges.npz"))
        seqs = [str(s) for s in z["seqs"]]
        eng.upload(*seqio.pack([seqio.encode(s) for s in seqs]))
        return seqs, np.asarray(z["merges"], dtype=np.int32), z["gaps"], t["score_matrix"]
    t = np.load(os.path.join(GOLDEN, "adeno_upgma_merges.npz"))
    if spec == "chain":
        codes, off, lens = seqio.synth_family(10000, 60, seed=2)
    else:
        n, length, seed = spec
        codes, off, lens = seqio.synth_family(n, length, seed=seed)
    seqs = [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(off, lens)]
    eng.upload(codes, off, lens)
    n = len(seqs)
    if spec == "chain":
        merges = np.array([(0, 1)] + [(n + k - 2, k) for k in range(2, n)], dtype=np.int32)
    else:
        merges = eng.slink(0)
    return seqs, merges, t["gaps"], t["score_matrix"]


def best(fn, reps):
    fn()
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        walls.append(time.perf_counter() - t0)
    return min(walls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max", type=int, default=4200)
    ap.add_argument("--ref-max", type=int, default=4200)
    a = ap.parse_args()
    name, power = gpu_info()
    threads = len(os.sched_getaffinity(0))
    for label, spec in sets():
        eng = famsa_b200.Engine(0)
        try:
            seqs, merges, gaps, sm = load(eng, spec)
            n = len(seqs)
            eng.prof_set_scoring(sm)
            t0 = time.perf_counter()
            root, res, st = eng.align_tree(merges, gaps)
            tree_wall = time.perf_counter() - t0
            rec = dict(set=label, n=n, gpu=name, power_limit=power, width=len(res[-1]["path"]),
                       levels=None, align_tree=dict(wall_ms=round(tree_wall * 1e3, 2), device_ms=round(st["device_ms"], 2)))
            from famsa_b200.schedule import ready_levels
            rec["levels"] = len(ready_levels(n, [tuple(m) for m in merges.tolist()]))
            rows = eng.tree_rows()
            dev, kern = device_ms(lambda: eng.tree_rows(download=False))
            rec["tree_rows"] = dict(device_ms=round(dev, 3), kernel_ms=round(kern, 3),
                                    wall_ms_on_device=round(best(lambda: eng.tree_rows(download=False), a.reps) * 1e3, 3),
                                    wall_ms_with_download=round(best(lambda: eng.tree_rows(), a.reps) * 1e3, 3))
            if n <= a.host_max:
                t0 = time.perf_counter()
                host = dp_cases.assemble_rows(seqs, [tuple(m) for m in merges.tolist()], res)
                rec["assemble_rows_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                rec["rows_equal_assemble_rows"] = bool(all(
                    seqio.decode(r[r != 30]) == seqs[i] and "".join("-" if c == 30 else seqio.ALPHABET[c] for c in r) == host[i]
                    for i, r in enumerate(rows)))
            else:
                rec["assemble_rows_ms"] = "not measured"
            eng.prof_drop([root])
        finally:
            eng.close()
        if pyoracle.have("ref", "ref_align_tree_mt") and n <= a.ref_max:
            dp = pyoracle.RefDp(n)
            sec, *_ = dp.align_tree_mt(seqs, merges, threads)
            dp.close()
            rec.update(ref_threads=threads, ref_alignment_ms=round(sec * 1e3, 1))
        else:
            rec["ref_alignment_ms"] = "not measured"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
