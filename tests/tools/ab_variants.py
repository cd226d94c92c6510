#!/usr/bin/env python
"""A/B of the switchable paths in ONE process (one torch import, one workload build per workload):
every variant is first checked for equality with the default path's result on the same resident
inputs, then timed with CUDA events.  The library reads its switches with getenv() at call time, so
os.environ changes between runs take effect.

    python tests/tools/ab_variants.py [compare] [sketch] [search] [gather] > ab.json

Not a bench line (bench.py is): a development tool for GPU sessions."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from sourmash_b200 import batch as B  # noqa: E402
from sourmash_b200.synth import MAX_HASH_1000, rows_of, synth_sketches  # noqa: E402

SWITCHES = ("SMB_JOIN_LAYOUT", "SMB_COMPARE_ALGO", "SMB_SKETCH_FUSED", "SMB_SEARCH_LAYOUT", "SMB_STRIPE_TAGS", "SMB_STRIPE_CTAS", "SMB_STRIPE_SWIZZLE")


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def set_env(env):
    for k in SWITCHES:
        os.environ.pop(k, None)
    for k, v in env.items():
        os.environ[k] = str(v)


def timed(fn, steps=5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def ab_compare(out):
    h, off = bench.compare_workload()
    n = len(off) - 1
    sset = B.SketchSet.from_host(h, off)
    d_ref = torch.empty((n, n), dtype=torch.float64, device="cuda")
    d_out = torch.empty((n, n), dtype=torch.float64, device="cuda")
    B.set_profiling(True)
    set_env({})
    B.compare_jaccard_device(sset, d_ref.data_ptr())
    torch.cuda.synchronize()
    variants = [("stripe (default: u16 tags, upper + mirror, two CTAs per SM, swizzled counter columns)", {}),
                ("stripe, counters in column order", {"SMB_STRIPE_SWIZZLE": "0"}),
                ("stripe, one CTA per SM (five-row blocks)", {"SMB_STRIPE_CTAS": "1"}),
                ("stripe, u32 tags", {"SMB_STRIPE_TAGS": "u32"}),
                ("stripe_full (both directions)", {"SMB_JOIN_LAYOUT": "stripe_full"}),
                ("plain (global reductions)", {"SMB_JOIN_LAYOUT": "plain"}),
                ("tile kernel", {"SMB_COMPARE_ALGO": "tile"})]
    res = {}
    for name, env in variants:
        set_env(env)
        try:
            d_out.fill_(-1.0)
            B.compare_jaccard_device(sset, d_out.data_ptr())
            torch.cuda.synchronize()
            same = bool(torch.equal(d_out, d_ref))
            ms = timed(lambda: B.compare_jaccard_device(sset, d_out.data_ptr()))
            res[name] = {"ms": ms, "identical_to_first": same, "pipeline_ms": B.last_kernel_ms(0)}
        except Exception as exc:                                   # noqa: BLE001
            res[name] = {"error": repr(exc)[:300]}
        log("compare", name, res[name])
    # end to end through the host API (pinned in / pinned out)
    ph, po = B.pinned_empty(len(h), np.uint64), B.pinned_empty(len(off), np.uint64)
    ph.array[:] = h
    po.array[:] = off
    pout = B.pinned_empty((n, n), np.float64)
    ref_host = d_ref.cpu().numpy()
    for name, env in [("stripe (default)", {}), ("plain (global reductions)", {"SMB_JOIN_LAYOUT": "plain"})]:
        set_env(env)
        try:
            def e2e():
                s2 = B.SketchSet.from_host(ph.array, po.array)
                B.compare_jaccard(s2, out=pout.array)
            e2e()
            same = bool(np.array_equal(pout.array, ref_host))
            res["e2e " + name] = {"ms": timed(e2e, steps=3, warmup=1), "identical_to_first": same}
        except Exception as exc:                                   # noqa: BLE001
            res["e2e " + name] = {"error": repr(exc)[:300]}
        log("compare e2e", name, res["e2e " + name])
    set_env({})
    out["compare"] = res


def ab_sketch(out):
    seqs, offs = bench.sketch_workload()
    d_bases = torch.empty(len(seqs) + 64, dtype=torch.uint8, device="cuda")
    d_bases[: len(seqs)].copy_(torch.from_numpy(seqs))
    lens = np.diff(offs.astype(np.int64)).astype(np.uint64)
    B.set_profiling(True)
    res, ref = {}, None
    for name, env in [("one pass (default)", {}), ("three launches", {"SMB_SKETCH_FUSED": 0})]:
        set_env(env)
        try:
            sset, nk = B.sketch_streams_device(d_bases.data_ptr(), offs[:-1], lens, bench.KSIZES, scaled=bench.SCALED)
            hh, oo = sset.to_host()
            if ref is None:
                ref = (hh, oo)
            same = bool(np.array_equal(hh, ref[0]) and np.array_equal(oo, ref[1]))
            ms = timed(lambda: B.sketch_streams_device(d_bases.data_ptr(), offs[:-1], lens, bench.KSIZES, scaled=bench.SCALED))
            res[name] = {"ms": ms, "hash_ms": B.last_kernel_ms(1), "identical": same, "kmers": int(nk)}
        except Exception as exc:                                   # noqa: BLE001
            res[name] = {"error": repr(exc)[:300]}
        log("sketch", name, res[name])
    set_env({})
    out["sketch"] = res


def tiled_db(h, off, reps):
    "the bench's tiled database, built on the device (no 12 GB host array)"
    dh = torch.from_numpy(h.view(np.int64)).cuda().repeat(reps)
    sizes = np.tile(np.diff(off.astype(np.int64)), reps)
    h_off = np.zeros(len(sizes) + 1, dtype=np.uint64)
    h_off[1:] = np.cumsum(sizes)
    d_off = torch.from_numpy(h_off.view(np.int64)).cuda()
    return B.SketchSet.from_device(dh.data_ptr(), d_off.data_ptr(), h_off, keepalive=(dh, d_off))


def ab_search(out):
    import oracle as orc
    h, off = synth_sketches(bench.N_SKETCHES)
    rows = rows_of(h, off)
    rng = np.random.Generator(np.random.PCG64(4000))
    reps = bench.N_DB_SEARCH // bench.N_SKETCHES
    planted = rng.choice(bench.N_SKETCHES, size=100, replace=False)
    query = np.unique(np.concatenate([rng.integers(1, MAX_HASH_1000, size=bench.N_QUERY_SEARCH, dtype=np.uint64)] +
                                     [rows[j][: len(rows[j]) // 2] for j in planted]))
    t = time.time()
    want = np.tile(orc.one_vs_many(query, h, off, nthreads=bench.host_cores()), reps)   # the DB is the set tiled
    log("search: oracle counts for the %d base rows in %.1fs" % (len(off) - 1, time.time() - t))
    db = tiled_db(h, off, reps)
    pq = B.pinned_empty(len(query), np.uint64)
    pq.array[:] = query
    res = {}
    alg = 8.0 * (db.total_hashes + len(query))
    for name, env, index in [("range-major stream (default)", {}, False), ("global directory + bitmap", {"SMB_SEARCH_LAYOUT": "global"}, False),
                             ("inverted index", {}, True)]:
        set_env(env)
        try:
            info = {}
            if index:
                torch.cuda.synchronize()
                t = time.perf_counter()
                info["distinct_hashes"] = int(db.build_index())
                torch.cuda.synchronize()
                info["index_build_ms"] = (time.perf_counter() - t) * 1e3
            got = B.one_vs_many(pq.array, db)
            same = bool(np.array_equal(got, want))
            ms = timed(lambda: B.one_vs_many(pq.array, db), steps=5, warmup=2)
            res[name] = dict(info, ms=ms, counts_equal_oracle_all_subjects=same, algorithmic_GBps=alg / ms / 1e6)
            if index:
                db.drop_index()
        except Exception as exc:                                   # noqa: BLE001
            res[name] = {"error": repr(exc)[:300]}
        log("search", name, res[name])
    set_env({})
    out["search"] = res


def ab_gather(out):
    h, off = synth_sketches(bench.N_SKETCHES)
    rows = rows_of(h, off)
    rng = np.random.Generator(np.random.PCG64(4000))
    reps = bench.N_DB_GATHER // bench.N_SKETCHES
    planted = rng.choice(bench.N_SKETCHES, size=200, replace=False)
    query = np.unique(np.concatenate([rows[j][rng.random(len(rows[j])) < 0.6] for j in planted] +
                                     [rng.integers(1, MAX_HASH_1000, size=20_000, dtype=np.uint64)]))
    db = tiled_db(h, off, reps)
    res, ref = {}, None
    for name, env, index in [("default", {}, False), ("global directory", {"SMB_SEARCH_LAYOUT": "global"}, False),
                             ("inverted index", {}, True)]:
        set_env(env)
        try:
            info = {}
            if index:
                torch.cuda.synchronize()
                t = time.perf_counter()
                info["distinct_hashes"] = int(db.build_index())
                torch.cuda.synchronize()
                info["index_build_ms"] = (time.perf_counter() - t) * 1e3
            ids, sizes = B.gather(query, db, threshold=50)
            if ref is None:
                ref = (ids, sizes)
            same = bool(np.array_equal(ids, ref[0]) and np.array_equal(sizes, ref[1]))
            ms = timed(lambda: B.gather(query, db, threshold=50), steps=3, warmup=1)
            res[name] = dict(info, ms=ms, rounds=int(len(ids)), identical_to_plain=same)
            if index:
                db.drop_index()
        except Exception as exc:                                   # noqa: BLE001
            res[name] = {"error": repr(exc)[:300]}
        log("gather", name, res[name])
    set_env({})
    out["gather"] = res


def main():
    which = sys.argv[1:] or ["compare", "sketch", "search", "gather"]
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    out = {}
    for w in which:
        t = time.time()
        try:
            {"compare": ab_compare, "sketch": ab_sketch, "search": ab_search, "gather": ab_gather}[w](out)
        except Exception:                                          # noqa: BLE001 -- the other workloads still run
            import traceback
            out[w] = {"error": traceback.format_exc()[-1500:]}
            log(out[w]["error"])
        log("[ab] %s done in %.1fs" % (w, time.time() - t))
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
