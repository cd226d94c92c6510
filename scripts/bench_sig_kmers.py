"""`sig kmers` on one GPU: 2 x 10^6 reads of 150 bp (FASTQ, a few N, some lower case) sampled from 20 synthetic
genomes of 5 Mbp, matched against three queries built from two of the genomes:

    scaled=1000, k=31   about 10^4 hashes   shared-memory split table
    scaled=10,   k=31   about 10^6 hashes   global directory + bitmap
    num=1000,    k=31                       every valid window probed

First, for every query, kmers.match_records on the first 10^4 reads must equal the reference's per-record loop written
with this package's MinHash (add_sequence, intersection, seq_to_hashes per record); only then are times taken:

    device_ms       CUDA events around the match kernel (smb_set_profiling), median of the repeats after a warm-up
    match_ms        kmers.match_records from a resident RecordBatch (upload, kernels, sort, readback), median
    command_s       `python -m sourmash_b200.sigkmers --save-kmers --save-sequences --check-sequence --force` end to end
                    (scaled=1000 query; without --check-sequence, --save-kmers stops at the first matching read with an N,
                    as the reference's `sig kmers` does)
    loop_s_extrapolated   the per-record loop's time on 10^4 reads, scaled to all reads (not run on all of them)

Writes one JSON line to stdout and, with --out, to that file.

    python scripts/bench_sig_kmers.py [--reads 2000000] [--repeats 5] [--out profiles/h100/bench_sig_kmers.json]
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

READ_BP = 150


def gpu_info():
    "name, power limit, maximum SM clock and current SM clock of GPU 0 (read-only query)"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


def write_reads(directory, *, n_genomes=20, genome_bp=5_000_000, n_reads=2_000_000, seed=77):
    """The genomes (uint8 arrays) and the path of a FASTQ file of n_reads reads sampled from them: one N per ~500
    reads, every 16th read lower case."""
    from sourmash_b200.synth import synth_genome
    genomes = [synth_genome(genome_bp, seed=1000 + g) for g in range(n_genomes)]
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n_genomes, size=n_reads)
    pos = rng.integers(0, genome_bp - READ_BP, size=n_reads)
    reads = np.empty((n_reads, READ_BP), np.uint8)
    for g in range(n_genomes):
        sel = np.nonzero(src == g)[0]
        reads[sel] = genomes[g][pos[sel][:, None] + np.arange(READ_BP)]
    reads[rng.integers(0, n_reads, size=n_reads // 500), rng.integers(0, READ_BP, size=n_reads // 500)] = ord("N")
    reads[::16] |= 0x20                                           # lower case
    path = os.path.join(directory, "reads.fq")
    qual = b"I" * READ_BP
    with open(path, "wb") as fh:
        for i0 in range(0, n_reads, 100_000):
            block = reads[i0:i0 + 100_000]
            fh.write(b"".join(b"@read%d\n%s\n+\n%s\n" % (i0 + j, block[j].tobytes(), qual) for j in range(len(block))))
    return genomes, path


def write_subset(directory, recs):
    path = os.path.join(directory, "head.fa")
    with open(path, "w") as fh:
        for i, s in enumerate(recs):
            fh.write(">read%d\n%s\n" % (i, s))
    return path


def queries(genomes, *, scaled_small=1000, scaled_large=10, num=1000):
    "the merged k=31 sketches of the first two genomes"
    from sourmash_b200.minhash import MinHash
    out = []
    for tag, kw in (("scaled=%d" % scaled_small, dict(n=0, scaled=scaled_small)),
                    ("scaled=%d" % scaled_large, dict(n=0, scaled=scaled_large)),
                    ("num=%d" % num, dict(n=num, scaled=0))):
        q = MinHash(kw["n"], 31, scaled=kw["scaled"])
        for g in genomes[:2]:
            q.add_sequence(g.tobytes(), True)
        out.append((tag, q))
    return out


def per_record_loop(q, recs):
    "(key list, matched) of the reference's loop, one record at a time"
    qh = set(q.hashes)
    rows, matched = [], []
    for r, s in enumerate(recs):
        seq_mh = q.copy_and_clear()
        seq_mh.add_sequence(s, True)
        matched.append(bool(seq_mh.intersection(q)))
        for o, h in enumerate(q.copy_and_clear().seq_to_hashes(s.upper(), force=True, bad_kmers_as_zeroes=True)):
            if h and h in qh:
                rows.append((r, o, h))
    return rows, matched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2_000_000)
    ap.add_argument("--genome-bp", type=int, default=5_000_000)
    ap.add_argument("--check-reads", type=int, default=10_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import lib
    from sourmash_b200.kmers import match_records
    from sourmash_b200.signature import SourmashSignature, save_signatures_to_json
    from sourmash_b200.sketch import RecordBatch
    if B.device_count() <= 0:
        raise SystemExit("bench_sig_kmers needs a CUDA device")
    result = {"gpu (name, power limit, max SM clock, SM clock at start)": gpu_info(), "reads": args.reads, "read_bp": READ_BP, "k": 31, "queries": {}}
    with tempfile.TemporaryDirectory() as d:
        genomes, path = write_reads(d, genome_bp=args.genome_bp, n_reads=args.reads)
        rb = RecordBatch([path])
        n_windows = int(np.maximum(rb.lengths.astype(np.int64) - 31 + 1, 0).sum())
        result["windows"] = n_windows
        recs = [rb.sequence(i).decode() for i in range(args.check_reads)]
        head = RecordBatch([write_subset(d, recs)])
        for tag, q in queries(genomes):
            # parity first: the first check_reads reads against the per-record loop
            t0 = time.perf_counter()
            rows, matched = per_record_loop(q, recs)
            loop_s = time.perf_counter() - t0
            got = match_records(q, head)
            assert list(zip(got.records.tolist(), got.ordinals.tolist(), got.hashes.tolist())) == rows, tag
            assert got.matched.tolist() == matched, tag
            full = match_records(q, rb)                                   # warm-up, and the head must agree
            cut = int(np.searchsorted(full.records, args.check_reads))
            assert full.hashes[:cut].tolist() == got.hashes.tolist(), tag
            dev, host = [], []
            lib.smb_set_profiling(True)
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                match_records(q, rb)
                host.append((time.perf_counter() - t0) * 1e3)
                dev.append(float(lib.smb_last_kernel_ms(1)))
            lib.smb_set_profiling(False)
            entry = {"query_hashes": len(q), "matches": int(len(full.hashes)), "matched_reads": int(full.matched.sum()),
                     "device_ms": statistics.median(dev), "device_ms_all": dev,
                     "kmers_per_s": n_windows / (statistics.median(dev) * 1e-3),
                     "match_ms": statistics.median(host), "match_ms_all": host,
                     "loop_s_on_check_reads": loop_s,
                     "loop_s_extrapolated": loop_s * args.reads / args.check_reads}
            if tag.startswith("scaled=1000"):
                sig = os.path.join(d, "q.sig")
                with open(sig, "wb") as fh:
                    save_signatures_to_json([SourmashSignature(q, name="q")], fh)
                cmd = [sys.executable, "-m", "sourmash_b200.sigkmers", "--signatures", sig, "--sequences", path, "-k", "31",
                       "--save-kmers", os.path.join(d, "k.csv"), "--save-sequences", os.path.join(d, "s.fa"),
                       "--check-sequence", "--force"]        # reads with an N are reported and skipped
                t0 = time.perf_counter()
                r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
                entry["command_s"] = time.perf_counter() - t0
                assert r.returncode == 0, r.stderr[-2000:]
                entry["command_stderr_tail"] = r.stderr.strip().splitlines()[-4:]
            result["queries"][tag] = entry
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
