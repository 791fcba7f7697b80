"""Times FAMSA's profile-profile mode (famsa in1 in2 out) on the device against the reference.

Two synthetic families (seqio.synth_family, default 8 000 x 400 aa each) are aligned on the device, each with
famsa_prof_align_tree along its single-linkage tree.  Timed, best of --reps after a warm-up:
  device          famsa_prof_put_rows of both alignments (FAMSA_PUT_ROWS_FROM_TEXT) + one famsa_prof_merge_batch, the
                  path copy to the host included, from rows already encoded as codes;
  device_rows     the same plus profiles.rows_after_merge, i.e. from codes to the merged text rows;
  reference       the reference's CProfile build of both alignments + CProfile(p1, p2, ..., no_threads = 1), what
                  CFAMSA::alignProfiles runs (oracle/_ref), from the rows as strings: the CGappedSequence objects are
                  built from text inside the timing, as loadFasta would have built them before.  The harness session,
                  the upper-casing and the read-back of rows are outside it.
One JSON line with the three times, whether the merged rows, order and total are identical, and the card's name and
power limit from nvidia-smi.

    python tools/profile_align_time.py [--n 8000] [--len 400] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import famsa_b200  # noqa: E402
from famsa_b200 import profiles, seqio  # noqa: E402
from oracle import pyoracle  # noqa: E402
import dp_cases  # noqa: E402
import profile_mode_cases as pmc  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    return tuple(x.strip() for x in out.split(","))


def device_alignment(eng, n, length, seed):
    """A family aligned on the device along its single-linkage tree: text rows in FAMSA's order."""
    codes, off, lens = seqio.synth_family(n, length, seed=seed)
    seqs = [seqio.decode(codes[int(o):int(o) + int(ln)]) for o, ln in zip(off, lens)]
    g, sm = pmc.reference_gaps(n)
    eng.upload(codes, off, lens)
    eng.prof_set_scoring(sm)
    merges = eng.slink(0)
    root, res, _ = eng.align_tree(merges, g)
    eng.prof_drop([root])
    rows = dp_cases.assemble_rows(seqs, [tuple(int(x) for x in m) for m in merges], res)
    return [rows[i] for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8000)
    ap.add_argument("--len", type=int, default=400)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not pyoracle.have_ref():
        raise SystemExit("oracle/_ref (the compiled reference) is not built")
    name, power = gpu_info()
    eng = famsa_b200.Engine(0)
    rows1 = device_alignment(eng, a.n, a.len, 1)
    rows2 = device_alignment(eng, a.n, a.len, 2)
    g, sm = pmc.reference_gaps(len(rows1) + len(rows2))
    eng.prof_set_scoring(sm)
    enc = [pmc.encode(r) for r in (rows1, rows2)]
    widths = [(enc[0].shape[1] - 1, enc[1].shape[1] - 1)]

    def device_mode():
        ids = [eng.prof_put_rows(e, g, from_text=True) for e in enc]
        (merged,), (res,) = eng.prof_merge_batch([tuple(ids)], g, widths)
        return merged, res

    merged, res = device_mode()                                     # warm-up
    eng.prof_drop([merged])
    dev, dev_rows = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        merged, res = device_mode()
        t1 = time.perf_counter()
        order, rows = profiles.rows_after_merge(rows1, rows2, res["path"], res["swapped"], from_text=True)
        t2 = time.perf_counter()
        dev.append(t1 - t0)
        dev_rows.append(t2 - t0)
        eng.prof_drop([merged])
    eng.close()

    n1, n2 = len(rows1), len(rows2)
    up1, up2 = [r.upper() for r in rows1], [r.upper() for r in rows2]
    dp = pyoracle.RefDp(n1 + n2)
    ref_s = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        p1 = dp.profile(up1, list(range(n1)))
        p2 = dp.profile(up2, list(range(n1, n1 + n2)))
        m, total = dp.align(p1, p2, 1)
        ref_s.append(time.perf_counter() - t0)
        ref_rows = dp.rows(m)
        dp.free(m)
    dp.close()
    print(json.dumps(dict(n1=n1, n2=n2, w1=enc[0].shape[1], w2=enc[1].shape[1], width=len(rows[0]), gpu=name,
                          power_limit=power, device_s=round(min(dev), 4), device_rows_s=round(min(dev_rows), 4),
                          ref_s=round(min(ref_s), 3), ref_threads=1,
                          same_rows=[pmc.normalise(r) for r in rows] == list(ref_rows.values()),
                          same_order=order == list(ref_rows.keys()), same_total=res["total"] == total)), flush=True)


if __name__ == "__main__":
    main()
