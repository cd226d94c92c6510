"""many_vs_many on one GPU: Q metagenome queries (configs[4]: synth.multigather_workload, as scripts/bench_multigather.py)
against one resident 50 000-row database, by batch.many_vs_many (groups of queries share one range-major pass) and by a
loop of batch.one_vs_many (one pass per query), for Q = 1, 8, 32, 128.  Both arms are timed with CUDA events around
the whole call (query upload, pass, Q x n counter readback), median of the repeats after one warm-up call.  The full
Q x n count matrices of the two arms are compared before any number is printed.

Algorithmic bytes of the batched arm: the database (8 bytes per hash) once per group, plus the queries' key stream;
over the time, and over the 3.35 TB/s HBM3 data-sheet peak of the H100 SXM.  ``readback_ms`` times the device-to-host
copy of the Q x n uint32 counters alone.  Prints one JSON line.

    python scripts/bench_many_vs_many.py [--queries 1,8,32,128] [--repeats 5] [--db-rows 50000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_multigather import BLOCK, gpu_info  # noqa: E402

HBM_PEAK = 3.35e12                        # bytes/s, H100 SXM data sheet
KEYS_PER_RANGE = 1024                     # csrc/compare_kernels.cu RM_GROUP_KEYS_PER_RANGE
GROUP_BYTES = 1 << 30                     # csrc/capi.cu many_vs_many_group_bytes


def n_groups(q_lens, n_rows, P):
    "groups of the batched pass (the cut of many_vs_many_plan in csrc/capi.cu)"
    if len(q_lens) < 2:
        return len(q_lens)
    groups, i = 0, 0
    while i < len(q_lens):
        keys, j = q_lens[i], i + 1
        while j < len(q_lens) and (j + 1 - i) * n_rows * 4 + (keys + q_lens[j]) * 12 <= GROUP_BYTES \
                and keys + q_lens[j] <= KEYS_PER_RANGE * P:
            keys += q_lens[j]
            j += 1
        groups, i = groups + 1, j
    return groups


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
        raise SystemExit("bench_many_vs_many needs a CUDA device")
    gpu = gpu_info()
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
    db_hashes = int(h_off[-1])
    P = 132 * 10 if db_hashes >= (32 << 20) else 132 * 2       # csrc/compare_kernels.cu range_major_parts

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        out = fn()                                                   # warm-up: module load, range-major copy, pools
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
        batched, ms_b = timed(lambda: B.many_vs_many(qs, db))
        loop, ms_l = timed(lambda: np.stack([B.one_vs_many(q, db) for q in qs]))
        assert batched.shape == loop.shape == (nq, n_db) and np.array_equal(batched, loop), ("counts differ", nq)
        d_c = torch.zeros((nq, n_db), dtype=torch.int32, device=dev)
        host = torch.empty((nq, n_db), dtype=torch.int32).numpy()
        _, ms_r = timed(lambda: host.__setitem__(slice(None), d_c.cpu().numpy()))
        q_lens = [len(q) for q in qs]
        groups = n_groups(q_lens, n_db, P)
        alg_bytes = 8 * db_hashes * groups + 12 * sum(q_lens)
        med = float(np.median(ms_b))
        results.append({"queries": nq, "batched_ms": med, "loop_ms": float(np.median(ms_l)),
                        "batched_ms_all": ms_b, "loop_ms_all": ms_l, "speedup": float(np.median(ms_l) / med),
                        "groups": groups, "algorithmic_bytes": alg_bytes,
                        "batched_bytes_per_s": alg_bytes / (med * 1e-3),
                        "share_of_hbm_peak": alg_bytes / (med * 1e-3) / HBM_PEAK,
                        "readback_ms": float(np.median(ms_r)), "counts_checked_equal": True})
    print(json.dumps({"metric": "many_vs_many wall time vs a loop of one_vs_many (configs[4] queries)", "unit": "ms",
                      "gpu": gpu, "db_rows": n_db, "db_hashes": db_hashes, "ranges": P,
                      "query_hashes": [int(len(q)) for q in queries[:max(qs_list)]][:8],
                      "repeats": args.repeats, "setup_s": setup_s, "hbm_peak_bytes_per_s": HBM_PEAK,
                      "timing": "CUDA events around the whole call, median of the repeats after one warm-up call; "
                                "readback_ms: the Q x n counter copy to the host alone",
                      "results": results}))


if __name__ == "__main__":
    main()
