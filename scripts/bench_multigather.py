"""Multigather on one GPU: Q metagenome queries (configs[4]: synth.gather_workload under Q seeds) against one resident
50 000-row database, by batch.multigather (the rounds of all queries together) and by a loop of batch.gather (one
query after the other), for Q = 1, 8, 32, 128.  Both arms are timed with CUDA events around the whole call on the
resident database (query upload, prefetch, rounds, readback); every time is printed only after the picks (rows and
intersection sizes, per query) of the two arms were found equal.  Both arms start with the same first pass per query
(|query ∩ row| for every row), which stays query by query; ``first_counters_ms`` times that pass alone (a loop of
batch.one_vs_many), so that the rounds' share of each arm can be read off.  Prints one JSON line.

    python scripts/bench_multigather.py [--queries 1,8,32,128] [--repeats 5] [--db-rows 50000]
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

BLOCK = 6250
THRESHOLD = 50                                   # hashes, as bench.py's gather workload


def gpu_info():
    "name, power limit and max SM clock of GPU 0 (read-only query)"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", default="1,8,32,128")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--db-rows", type=int, default=50_000)
    args = ap.parse_args()
    qs_list = [int(x) for x in args.queries.split(",")]
    import torch

    from sourmash_b200 import batch as B
    from sourmash_b200.synth import database_block, multigather_workload
    if not torch.cuda.is_available() or B.device_count() <= 0:
        raise SystemExit("bench_multigather needs a CUDA device")
    t0 = time.time()
    queries, sizes, frac, overrides = multigather_workload(args.db_rows, max(qs_list))
    dev = torch.device("cuda")
    n_db = args.db_rows
    h_off = np.zeros(n_db + 1, dtype=np.uint64)
    h_off[1:] = np.cumsum(sizes)
    d_h = torch.empty(int(h_off[-1]), dtype=torch.int64, device=dev)
    for b in range(0, n_db, BLOCK):
        e = min(b + BLOCK, n_db)
        d_h[int(h_off[b]):int(h_off[e])] = database_block(sizes, frac, np.zeros(1, np.uint64), b, e, 5002,
                                                          overrides=overrides, torch=torch, device=dev)
    d_off = torch.from_numpy(h_off.view(np.int64)).to(dev)
    db = B.SketchSet.from_device(d_h.data_ptr(), d_off.data_ptr(), h_off, keepalive=(d_h, d_off))
    torch.cuda.synchronize()
    setup_s = time.time() - t0

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()                                                         # warm-up: module load, range-major copy, pools
        ms = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            e0.record()
            out = fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return out, ms

    results = []
    for nq in qs_list:
        qs = queries[:nq]
        stats = {}
        batched, ms_b = timed(lambda: B.multigather(qs, db, thresholds=THRESHOLD, stats=stats))
        loop, ms_l = timed(lambda: [B.gather(q, db, threshold=THRESHOLD) for q in qs])
        _, ms_p = timed(lambda: [B.one_vs_many(q, db) for q in qs])  # the first counters alone, query by query
        for i in range(nq):                                          # parity before any number is printed
            assert batched[i][0].tolist() == loop[i][0].tolist(), ("rows differ", nq, i)
            assert batched[i][1].tolist() == loop[i][1].tolist(), ("sizes differ", nq, i)
        rounds = [len(r[0]) for r in batched]
        results.append({"queries": nq, "batched_ms": float(np.median(ms_b)), "loop_ms": float(np.median(ms_l)),
                        "first_counters_ms": float(np.median(ms_p)), "batched_ms_all": ms_b, "loop_ms_all": ms_l,
                        "speedup": float(np.median(ms_l) / np.median(ms_b)),
                        "rounds_total": int(sum(rounds)), "rounds_max": int(max(rounds)),
                        "round_launches": stats["round_launches"], "picks_checked_equal": True})
    print(json.dumps({"metric": "multigather wall time vs a loop of gather (configs[4] queries)", "unit": "ms",
                      "gpu": gpu_info(), "db_rows": n_db, "db_hashes": int(h_off[-1]),
                      "query_hashes": [int(len(q)) for q in queries[:max(qs_list)]][:8],
                      "threshold_hashes": THRESHOLD, "repeats": args.repeats, "setup_s": setup_s,
                      "timing": "CUDA events around the whole call, median of the repeats after one warm-up call",
                      "results": results}))


if __name__ == "__main__":
    main()
