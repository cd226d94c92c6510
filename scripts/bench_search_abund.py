"""Abundance search on one GPU: batch.search_angular and Index.search_abund against the per-subject loop they replace
(one `query.similarity(subject, downsample=True)` per subject).  Workloads (tests/search_abund_cases.bench_workload):

    1  genome database: 50 000 subjects of ~5 000 hashes, abundances 1..99, a 10^4-hash query (split-table layout)
    2  the same database, a 10^6-hash query (global directory + occupancy bitmap)
    3  sample vs samples: 1 000 subjects of ~2 x 10^5 hashes, a 2 x 10^5-hash query (long rows, large query)

Parity first: every score of every workload must equal the numpy restatement (u64 terms with wrapping, math.acos per
row) bit for bit, and the per-subject MinHash.similarity(downsample=True) loop on the first --check-rows rows.  Only
then are times taken:

    device_ms        CUDA events around the device step of search_angular (the memsets, the directory build for a large
                     query, the kernel; smb_set_profiling), median of --repeats after a warm-up
    hbm_bytes        16 B per subject element (hash + abundance) plus the query's keys and abundances (and the directory
                     and bitmap of the global layout); hbm_share = hbm_bytes / 3.35 TB/s (H100 SXM data sheet) / device_ms,
                     min_ms_from_bytes = hbm_bytes / 3.35 TB/s (what limits the kernel beyond that is not measured here)
    call_ms          batch.search_angular from the resident set, upload of the query and copy-out included, median
    search_abund_ms  LinearIndex.search_abund(query, threshold=0.08) over signature objects, groups already resident,
                     median; search_abund_first_ms is the first call on a new index, which gathers the subjects'
                     sketches from the objects and uploads them (what a one-shot search pays)
    loop_rows_s      the per-subject loop on the first --check-rows rows; loop_extrapolated_s scales it to every row
    b200search       workload 1's database as one .sig file and as a .zip: load_file_as_index + select, then
                     search_abund, against the same load and the per-subject loop it replaces, and
                     `python -m sourmash_b200.plugin b200search` end to end

Writes one JSON line to stdout and, with --out, to that file.

    python scripts/bench_search_abund.py [--repeats 5] [--out profiles/h100/bench_search_abund.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sig_kmers import gpu_info  # noqa: E402

HBM_PEAK = 3.35e12
SCALED = 1000


def signatures_of(sset, prefix):
    "the rows of a resident set as SourmashSignature objects (scaled 1000, k = 31), built in one library call"
    from sourmash_b200._ffi import rustcall
    from sourmash_b200._lowlevel import ffi, lib
    from sourmash_b200.signature import SourmashSignature
    ks = np.array([31], dtype=np.uint32)
    size = ffi.new("uintptr_t *")
    arr = rustcall(lib.smb_signatures_from_sketchset, sset._ptr, ffi.cast("uint32_t *", ks.ctypes.data), 1, 1, SCALED,
                   0, 42, size)
    sigs = [SourmashSignature._from_objptr(arr[i]) for i in range(size[0])]
    lib.signatures_array_free(arr, size[0])
    for i, s in enumerate(sigs):
        s._name = "%s%d" % (prefix, i)
    return sigs


def same_bits(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    if len(bad):
        raise SystemExit("parity failed (%s): rows %s got %s want %s" % (what, bad[:5].tolist(), got[bad[:5]].tolist(),
                                                                        want[bad[:5]].tolist()))


def median_ms(fn, repeats):
    fn()
    wall = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        wall.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(wall), [min(wall), max(wall)]


def run_workload(which, data, args, B, C, lib, all_sigs=None):
    from sourmash_b200.index import LinearIndex
    q, qa, h, off, ab = data
    n = len(off) - 1
    sset = B.SketchSet.from_host(h, off, ab)
    entry = {"subjects": n, "elements": int(len(h)), "query": int(len(q))}
    t0 = time.perf_counter()
    got = B.search_angular(q, qa, sset, C.U64_MAX)
    entry["first_call_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    same_bits(got, C.numpy_angular(q, qa, h, off, ab, C.U64_MAX), "workload %d numpy" % which)
    m = min(args.check_rows, n)
    head = sset.take_rows(np.arange(m))
    sigs = signatures_of(head, "s")
    query = signatures_of(B.SketchSet.from_rows([q], [qa]), "q")[0]
    t0 = time.perf_counter()
    loop = [query.similarity(s, downsample=True) for s in sigs]
    loop_s = time.perf_counter() - t0
    same_bits(got[:m], loop, "workload %d per-subject loop" % which)
    entry.update(loop_rows=m, loop_rows_s=round(loop_s, 3), loop_extrapolated_s=round(loop_s * n / m, 2))
    # device time and bytes
    lib.smb_set_profiling(True)
    dev = []
    B.search_angular(q, qa, sset, C.U64_MAX)
    for _ in range(args.repeats):
        B.search_angular(q, qa, sset, C.U64_MAX)
        dev.append(lib.smb_last_kernel_ms(1))
    lib.smb_set_profiling(False)
    dev_ms = statistics.median(dev)
    qbytes = 16 * len(q)
    if len(q) > C.SPLIT_MAX:                         # directory (about 2 u32 per key) and bitmap (8 bits per bucket)
        qbytes += 2 * 4 * len(q) + 2 * len(q)
    hbm = 16 * len(h) + qbytes
    entry.update(device_ms=round(dev_ms, 3), device_ms_spread=[round(min(dev), 3), round(max(dev), 3)], hbm_bytes=hbm,
                 hbm_tb_s=round(hbm / dev_ms / 1e9, 3), hbm_share=round(hbm / HBM_PEAK / (dev_ms / 1e3), 3),
                 min_ms_from_bytes=round(hbm / HBM_PEAK * 1e3, 3))
    call_ms, spread = median_ms(lambda: B.search_angular(q, qa, sset, C.U64_MAX), args.repeats)
    entry.update(call_ms=round(call_ms, 3), call_ms_spread=[round(x, 3) for x in spread])
    # Index.search_abund over signature objects
    del head, sigs
    if all_sigs is None:
        all_sigs = signatures_of(sset, "s")
    idx = LinearIndex(all_sigs, filename="db")
    t0 = time.perf_counter()
    res = idx.search_abund(query, threshold=0.08)
    entry["search_abund_first_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    ms, spread = median_ms(lambda: idx.search_abund(query, threshold=0.08), args.repeats)
    entry.update(search_abund_ms=round(ms, 3), search_abund_ms_spread=[round(x, 3) for x in spread],
                 search_abund_matches=len(res), speedup_vs_loop=round(loop_s * n / m / (ms / 1e3), 1),
                 first_call_speedup_vs_loop=round(loop_s * n / m / (entry["search_abund_first_ms"] / 1e3), 2))
    return entry, sset, query, all_sigs


def b200search(query, sigs, tmp):
    """workload 1's database as one .sig file and as a .zip (members of 5 000 signatures, stored): per format, the
    route `b200search` takes for each database argument -- load_file_as_index + select, then search_abund -- against
    the same load followed by the per-subject loop it replaces, and the command end to end"""
    from sourmash_b200.index import load_file_as_index
    from sourmash_b200.signature import save_signatures_to_json
    qpath = os.path.join(tmp, "q.sig")
    with open(qpath, "wb") as fh:
        save_signatures_to_json([query], fh)
    out = {"subjects": len(sigs)}
    for kind in ("sig", "zip"):
        path = os.path.join(tmp, "db." + kind)
        t0 = time.perf_counter()
        if kind == "sig":
            with open(path, "wb") as fh:
                save_signatures_to_json(sigs, fh)
        else:
            with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_STORED, allowZip64=True) as z:
                for i in range(0, len(sigs), 5000):
                    z.writestr("signatures/part%02d.sig" % (i // 5000), save_signatures_to_json(sigs[i:i + 5000]))
        entry = {"write_s": round(time.perf_counter() - t0, 1), "bytes": os.path.getsize(path)}
        for route in ("search_abund", "per_subject_loop"):
            t0 = time.perf_counter()
            db = load_file_as_index(path).select(ksize=31, moltype="DNA")
            t1 = time.perf_counter()
            if route == "search_abund":
                res = db.search_abund(query, threshold=0.08)
            else:                                      # Index.search_abund of the reference, subject by subject
                res = [(sc, s) for s, sc in ((s, query.similarity(s, downsample=True)) for s in db.signatures())
                       if sc >= 0.08]
                res.sort(key=lambda x: -x[0])
            t2 = time.perf_counter()
            entry[route] = {"load_s": round(t1 - t0, 2), "search_s": round(t2 - t1, 2), "total_s": round(t2 - t0, 2),
                            "matches": len(res)}
            del db, res
        cmd = [sys.executable, "-m", "sourmash_b200.plugin", "b200search", qpath, path, "-o", os.path.join(tmp, "o.csv")]
        t0 = time.perf_counter()
        r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
        entry["command_s"] = round(time.perf_counter() - t0, 2)
        if r.returncode != 0:
            raise SystemExit("b200search failed:\n" + r.stderr[-2000:])
        os.remove(path)
        out[kind] = entry
        print("b200search", kind, json.dumps(entry), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check-rows", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workloads", default="1,2,3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import search_abund_cases as C
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import lib
    if B.device_count() <= 0:
        raise SystemExit("no CUDA device: %s" % B.device_probe_error())
    result = {"gpu (name, power limit, max SM clock, SM clock at start)": gpu_info()}
    wanted = [int(x) for x in args.workloads.split(",")]
    db = db_sigs = None
    for which in wanted:
        if which == 3:
            db = db_sigs = None                        # workload 1 and 2's database is not needed any more
        t0 = time.perf_counter()
        data = C.bench_workload(which, db if which in (1, 2) else None)
        if which in (1, 2):
            db = data[2:]
        gen_s = time.perf_counter() - t0
        entry, sset, query, sigs = run_workload(which, data, args, B, C, lib, db_sigs if which in (1, 2) else None)
        if which in (1, 2):
            db_sigs = sigs
        entry["generate_s"] = round(gen_s, 1)
        if which == 1:
            with tempfile.TemporaryDirectory() as tmp:
                entry["b200search"] = b200search(query, sigs, tmp)
        result["workload %d" % which] = entry
        print("workload %d" % which, json.dumps(entry), file=sys.stderr, flush=True)
        del data, sset, sigs
    result["gpu (name, power limit, max SM clock, SM clock at end)"] = gpu_info()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
