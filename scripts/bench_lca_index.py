"""`lca index` on one GPU, over the GTDB-sized synthetic set of tests/lca_index_cases.skewed_rows (seeded): --genomes
genomes, about --pairs (hash, genome) pairs, a quarter of each genome's hashes drawn from a shared pool with a
Zipf-like skew.

Parity first: the arrays of batch.lca_index must equal the numpy oracle (tests/lca_index_cases.np_oracle_arrays), and
the text of the first, the largest and the last key must equal the oracle's.  Then:

    group_format_device_ms  CUDA events (smb_set_profiling) around the build (sort, key order, idx, byte sizes) plus
                            every chunk's text kernel, median
    rows_to_file_s          batch.lca_index from the resident rows plus lca.write_database to an uncompressed file,
                            median (the file is written under a temporary directory)
    command_s               `python -m sourmash_b200.lca index` end to end from a .zip of the genomes' signatures and a
                            spreadsheet of their lineages, one run
    gzip_s                  host zlib (level 9, as the reference writes .gz) over the uncompressed file, one run: paid
                            the same by any writer of a .lca.json.gz
    loop_s_extrapolated     the reference's insert loop (a dict of sets, LCA_Database.insert) plus save_to_json's
                            json.dump, restated and timed on the first --loop-genomes genomes, scaled by pairs:
                            extrapolated, not run

Writes one JSON line to stdout and, with --out, to that file.

    python scripts/bench_lca_index.py [--repeats 3] [--out profiles/h100/bench_lca_index.json]
"""
import argparse
import gzip
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sig_kmers import gpu_info  # noqa: E402


def write_inputs(tmp, h, off):
    "a .zip of one scaled=1 k=31 signature per genome (name g<i>) and a spreadsheet giving each a species lineage"
    zpath, csv = os.path.join(tmp, "genomes.zip"), os.path.join(tmp, "tax.csv")
    with zipfile.ZipFile(zpath, "w", zipfile.ZIP_STORED) as z:
        for g in range(len(off) - 1):
            mins = h[int(off[g]):int(off[g + 1])].tolist()
            sig = [{"class": "sourmash_signature", "email": "", "hash_function": "0.murmur64", "filename": "",
                    "name": "g%d" % g, "license": "CC0",
                    "signatures": [{"num": 0, "ksize": 31, "seed": 42, "max_hash": 2**64 - 1, "mins": mins,
                                    "molecule": "DNA"}], "version": 0.4}]
            z.writestr("signatures/g%d.sig" % g, json.dumps(sig))
    with open(csv, "w") as fh:
        fh.write("identifiers,superkingdom,phylum,class,order,family,genus,species\n")
        for g in range(len(off) - 1):
            fh.write("g%d,Bacteria,p%d,c%d,o%d,f%d,g%d,s%d\n" % (g, g % 7, g % 31, g % 97, g % 401, g % 2003, g))
    return zpath, csv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=30_000)
    ap.add_argument("--pairs", type=int, default=30_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--loop-genomes", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from sourmash_b200 import batch as B
    from sourmash_b200 import lca as L
    from tests import lca_index_cases as C

    h, off = C.skewed_rows(seed=7, n_rows=args.genomes, n_pairs=args.pairs)
    sset = B.SketchSet.from_host(h, off)
    x = B.lca_index(sset)                                               # warm-up, and the parity check
    got = x.arrays()
    for a, b in zip(got, C.np_oracle_arrays(h, off)):
        assert np.array_equal(a, b)
    hashes, offsets, idx = got
    n = len(x)
    sizes = np.diff(offsets.astype(np.int64))
    whole = b"".join(bytes(c) for c in x.text_chunks(64 << 20))
    first = C.text_of_keys(hashes, offsets, idx, 0, 1, n)
    last = C.text_of_keys(hashes, offsets, idx, n - 1, n, n)
    big = int(np.argmax(sizes))
    assert whole.startswith(first) and whole.endswith(last)
    assert C.text_of_keys(hashes, offsets, idx, big, big + 1, n)[2:] in whole
    text_bytes = len(whole)
    del whole, got

    tmp = tempfile.mkdtemp(prefix="bench_lca_index_")
    dev, to_file = [], []
    for _ in range(args.repeats):
        B.set_profiling(True)
        y = B.lca_index(sset)
        ms = B.last_kernel_ms(1)
        for _chunk in y.text_chunks(256 << 20):
            ms += B.last_kernel_ms(1)
        B.set_profiling(False)
        dev.append(ms)
        del y
        path = os.path.join(tmp, "db.lca.json")
        if os.path.exists(path):
            os.remove(path)
        B.synchronize()
        t = time.perf_counter()
        y = B.lca_index(sset)
        L.write_database(path, 31, 1, "DNA", {}, y, {}, {}, {})
        to_file.append(time.perf_counter() - t)
        del y
    t = time.perf_counter()
    with open(path, "rb") as fh:
        gz_len = len(gzip.compress(fh.read(), compresslevel=9))
    gzip_s = time.perf_counter() - t

    zpath, csv = write_inputs(tmp, h, off)
    out = os.path.join(tmp, "cmd.lca.json")
    t = time.perf_counter()
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.lca", "index", csv, out, zpath, "--scaled", "1"],
                       capture_output=True, text=True, cwd=ROOT)
    command_s = time.perf_counter() - t
    assert r.returncode == 0, r.stderr[-2000:]
    assert "loaded %d hashes at ksize=31 scaled=1" % n in r.stderr, r.stderr[-2000:]

    m = args.loop_genomes                                               # the reference's loop on a subset
    t = time.perf_counter()
    d = {}
    for g in range(m):
        for hv in h[int(off[g]):int(off[g + 1])].tolist():
            d.setdefault(hv, set()).add(g)
    with open(os.path.join(tmp, "loop.json"), "w") as fh:
        json.dump({"hashval_to_idx": dict((k, list(v)) for k, v in d.items())}, fh)
    loop_s = time.perf_counter() - t
    loop_pairs = int(off[m])

    res = {
        "gpu": gpu_info(),
        "genomes": args.genomes, "pairs": int(len(h)), "distinct_hashes": n, "max_genomes_per_hash": int(sizes.max()),
        "text_bytes": text_bytes, "gzip_bytes": gz_len,
        "group_format_device_ms": statistics.median(dev), "rows_to_file_s": statistics.median(to_file),
        "command_s": command_s, "gzip_s": gzip_s,
        "loop_genomes_timed": m, "loop_pairs_timed": loop_pairs, "loop_s_timed": loop_s,
        "loop_s_extrapolated": loop_s * len(h) / max(loop_pairs, 1),
        "parity": "arrays equal the numpy oracle; first, largest and last key's text equal the oracle's",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
