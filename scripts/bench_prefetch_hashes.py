"""Prefetch's matched / unmatched query hashes on one GPU (`b200prefetch --save-matching-hashes --save-unmatched-hashes`)
against the reference's per-match loop they replace (commands.py:1602-1622: `ident_mh += query_mh & match_mh` and
`noident_mh.remove_many(match_mh)`, each a merge against the whole query).

Workload: configs[4] at full size -- a 10^7-hash query (synth.search_query), 300 000 rows of ~5 000 hashes of which 1 %
hold 20-80 % of their hashes from the query (synth.database_plan / database_block, the seeds bench.py uses), resident in
HBM; the rows passing 50 kbp at scaled=1000 are the matches.

    device_ms        CUDA events around launch_query_cover (directory, bitmap, the cover kernel; smb_set_profiling),
                     median of --repeats after a warm-up; elements_probed = the summed length of the passing rows
    call_ms          batch.query_covered from the resident set, query upload and mask copy-out included, median
    extra_ms         what the two outputs add to b200prefetch after its CSV: Command_B200Prefetch._save_hashes (the
                     mask, both sketches built from arrays, both .sig files written), median
    cpu_loop         the reference's loop restated with this package's MinHash on --loop-rows passing rows, timed and
                     EXTRAPOLATED linearly to every passing row (labelled as such)

Parity first: the mask must equal np.isin over the passing rows.  Writes one JSON line to stdout and, with --out, to that
file; the card's name and power limit are read in the same run.

    python scripts/bench_prefetch_hashes.py [--repeats 5] [--out profiles/h100/bench_prefetch_hashes.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:                                   # noqa: BLE001
        return "nvidia-smi failed: %r" % (exc,)


def median_ms(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), [min(ts), max(ts)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--rows", type=int, default=300_000)
    ap.add_argument("--loop-rows", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bench
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import lib
    from sourmash_b200.minhash import MinHash
    from sourmash_b200.plugin import Command_B200Prefetch, _Loaded
    from sourmash_b200.signature import SourmashSignature
    from sourmash_b200.synth import database_plan, search_query
    if B.device_count() <= 0:
        raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
    entry = {"gpu": gpu_info(), "workload": "configs[4]: 1e7-hash query, %d rows, threshold 50 kbp, scaled 1000" % args.rows}
    query = search_query(10_000_000)
    sizes, frac = database_plan(args.rows, 4001, planted_frac=0.01)
    t0 = time.perf_counter()
    db, d_h, h_off = bench.build_database(torch, B, sizes, frac, query, 4002, 0, args.rows)
    entry["db_hashes"] = int(h_off[-1])
    entry["db_build_s"] = round(time.perf_counter() - t0, 1)
    counts = B.one_vs_many(query, db)
    rows = np.nonzero(counts.astype(np.int64) * 1000 >= 50_000)[0]
    probed = int(sizes[rows].sum())
    entry.update(query_hashes=len(query), passing_rows=len(rows), elements_probed=probed)
    # parity
    got = B.query_covered(query, db, rows)
    held = torch.cat([d_h[int(h_off[r]):int(h_off[r + 1])] for r in rows]).cpu().numpy().view(np.uint64)
    want = np.isin(query, held)
    assert np.array_equal(got, want), "query_covered differs from np.isin"
    entry["covered"] = int(got.sum())
    # device time
    lib.smb_set_profiling(True)
    dev = []
    for _ in range(args.repeats):
        B.query_covered(query, db, rows)
        dev.append(float(lib.smb_last_kernel_ms(1)))
    lib.smb_set_profiling(False)
    entry.update(device_ms=round(statistics.median(dev), 3), device_ms_spread=[round(min(dev), 3), round(max(dev), 3)],
                 probes_per_s=round(probed / (statistics.median(dev) / 1e3), 0))
    ms, spread = median_ms(lambda: B.query_covered(query, db, rows), args.repeats)
    entry.update(call_ms=round(ms, 3), call_ms_spread=[round(x, 3) for x in spread])
    # what the two outputs add to b200prefetch
    qmh = MinHash(0, 31, scaled=1000)
    qmh.add_many(query)
    qsig = SourmashSignature(qmh, name="q")
    src = _Loaded(None, None, qsig, qmh)
    with tempfile.TemporaryDirectory() as d:
        ns = types.SimpleNamespace(quiet=True, save_matching_hashes=os.path.join(d, "k.sig"),
                                   save_unmatched_hashes=os.path.join(d, "u.sig"))
        ms, spread = median_ms(lambda: Command_B200Prefetch._save_hashes(ns, qmh, db, rows.tolist(), src), args.repeats)
    entry.update(extra_ms=round(ms, 1), extra_ms_spread=[round(x, 1) for x in spread])
    # the reference's loop, restated, on a few rows, extrapolated
    ident, noident = qmh.copy_and_clear(), qmh.copy_and_clear()
    noident.merge(qmh)
    m = min(args.loop_rows, len(rows))
    mats = []
    for r in rows[:m]:
        mh = MinHash(0, 31, scaled=1000)
        mh.add_many(d_h[int(h_off[r]):int(h_off[r + 1])].cpu().numpy().view(np.uint64))
        mats.append(mh)
    t0 = time.perf_counter()
    for mh in mats:
        ident.merge(qmh & mh)
        noident.remove_many(mh)
    loop_s = time.perf_counter() - t0
    entry["cpu_loop"] = {"rows_timed": m, "rows_s": round(loop_s, 3),
                         "EXTRAPOLATED_all_rows_s": round(loop_s * len(rows) / max(m, 1), 1),
                         "note": "linear extrapolation of the timed rows to every passing row, not a measurement"}
    entry["speedup_vs_extrapolated_loop"] = round(loop_s * len(rows) / max(m, 1) / (entry["extra_ms"] / 1e3), 1)
    line = json.dumps(entry)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
