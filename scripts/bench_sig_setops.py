"""`sig merge` / `sig intersect` / `sig subtract` on one GPU: batch.combine over the compare benchmark's sketch set,
synth.synth_sketches(10_000) (10^4 rows of about 5 000 hashes, 100 families; about 5 x 10^7 hashes), flat and with
abundances (1..99, seeded).

Parity first: for every op, batch.combine on the whole set must equal a numpy restatement (np.unique, run lengths,
np.add.at for the sums), and on the first 1 000 rows the reference's loop written with this package's MinHash (a chain
of MinHash.merge into copy_and_clear() of the first sketch; Python sets for intersect and subtract).  Only then are
times taken:

    device_ms        CUDA events around the combine step (sort, run pass, scan, scatter and the length readback;
                     smb_set_profiling), median of the repeats after a warm-up
    combine_ms       batch.combine from the resident set, copy-out to numpy included, median
    loop_1000_s      the reference-semantics loop on the first 1 000 rows (MinHash objects built beforehand)
    combine_1000_ms  batch.combine on the same 1 000 rows, median
    command_1000_s   `python -m sourmash_b200.sigsetops merge|intersect|subtract row0.sig rest.sig`: the same 1 000 flat
                     sketches from two .sig files (row 0; rows 1-999), end to end (interpreter start, parse, upload,
                     combine, write)

Writes one JSON line to stdout and, with --out, to that file.

    python scripts/bench_sig_setops.py [--n 10000] [--repeats 7] [--out profiles/h100/bench_sig_setops.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_sig_kmers import gpu_info  # noqa: E402

OPS = ("union", "all", "first_only")
COMMAND = {"union": "merge", "all": "intersect", "first_only": "subtract"}


def rows_of(h, off, a, n):
    rows = [h[int(off[i]):int(off[i + 1])] for i in range(n)]
    return rows, (None if a is None else [a[int(off[i]):int(off[i + 1])] for i in range(n)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000)
    ap.add_argument("--check-rows", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import sig_setops_cases as C
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import lib
    from sourmash_b200.signature import SourmashSignature, save_signatures_to_json
    from sourmash_b200.synth import synth_sketches
    if B.device_count() <= 0:
        raise SystemExit("no CUDA device: %s" % B.device_probe_error())
    result = {"gpu (name, power limit, max SM clock, SM clock at start)": gpu_info(), "n": args.n,
              "check_rows": args.check_rows}
    h, off = synth_sketches(args.n)
    ab = np.random.default_rng(1).integers(1, 100, size=len(h)).astype(np.uint64)
    result["hashes"] = int(len(h))
    m = args.check_rows
    with tempfile.TemporaryDirectory() as tmp:
        head_rows, _ = rows_of(h, off, None, m)
        sigs = [SourmashSignature(C.minhash_of(r, scaled=1000), name="s%d" % i) for i, r in enumerate(head_rows)]
        sig_files = [os.path.join(tmp, "row0.sig"), os.path.join(tmp, "rest.sig")]
        for path, part in zip(sig_files, (sigs[:1], sigs[1:])):
            with open(path, "wb") as fh:
                save_signatures_to_json(part, fh)
        for flavour, abund in (("flat", None), ("abund", ab)):
            full = B.SketchSet.from_host(h, off, abund)
            rows, abs_ = rows_of(h, off, abund, m)
            head = B.SketchSet.from_host(*C.csr(rows, abs_))
            mhs = [C.minhash_of(r, None if abs_ is None else abs_[i], scaled=1000) for i, r in enumerate(rows)]
            for op in OPS:
                tag = "%s/%s" % (flavour, op)
                got = B.combine(full, op)
                want = C.numpy_combine(op, [h[int(off[i]):int(off[i + 1])] for i in range(args.n)],
                                       None if abund is None else
                                       [abund[int(off[i]):int(off[i + 1])] for i in range(args.n)])
                C.assert_same(got, want, tag + " numpy")
                t0 = time.perf_counter()
                if op == "union":
                    mh = mhs[0].copy_and_clear()
                    for x in mhs:
                        mh.merge(x)
                    got_mh = mh.hashes
                    ref_h = np.array(sorted(got_mh), np.uint64)
                    ref = (ref_h, np.array([got_mh[int(x)] for x in ref_h], np.uint64) if abund is not None else None)
                else:
                    mins = set(mhs[0].hashes)
                    for x in mhs[1:]:
                        if op == "all":
                            mins.intersection_update(x.hashes)
                        else:
                            mins -= set(x.hashes)
                    ref = (np.array(sorted(mins), np.uint64), None)
                loop_s = time.perf_counter() - t0
                C.assert_same(B.combine(head, op), ref, tag + " reference loop")
                entry = {"out_len": int(len(got[0])), "loop_1000_s": round(loop_s, 4)}
                B.combine(full, op)                                  # warm-up
                lib.smb_set_profiling(True)
                dev, wall = [], []
                for _ in range(args.repeats):
                    t0 = time.perf_counter()
                    B.combine(full, op)
                    wall.append((time.perf_counter() - t0) * 1e3)
                    dev.append(lib.smb_last_kernel_ms(1))
                lib.smb_set_profiling(False)
                small = []
                for _ in range(args.repeats):
                    t0 = time.perf_counter()
                    B.combine(head, op)
                    small.append((time.perf_counter() - t0) * 1e3)
                entry.update(device_ms=round(statistics.median(dev), 3), combine_ms=round(statistics.median(wall), 3),
                             combine_ms_spread=[round(min(wall), 3), round(max(wall), 3)],
                             combine_1000_ms=round(statistics.median(small), 3))
                if flavour == "flat":
                    out = os.path.join(tmp, "out_%s.sig" % op)
                    cmd = [sys.executable, "-m", "sourmash_b200.sigsetops", COMMAND[op]] + sig_files
                    t0 = time.perf_counter()
                    r = subprocess.run(cmd + ["-o", out], capture_output=True, text=True, cwd=ROOT)
                    entry["command_1000_s"] = round(time.perf_counter() - t0, 3)
                    if r.returncode != 0:
                        raise SystemExit("command failed: %s\n%s" % (" ".join(cmd), r.stderr[-2000:]))
                result[tag] = entry
                print(tag, json.dumps(entry), file=sys.stderr, flush=True)
    result["gpu (name, power limit, max SM clock, SM clock at end)"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
