"""`lca classify` / `lca summarize`'s per-hash work on one GPU, over the GTDB-sized synthetic setting of
tests/lca_cases.synth_lca (seeded): 10^5 lineages, 10^7 (hash, genome) pairs in two databases, 1 000 queries of about
5 000 hashes.

Parity first: the counts of 8 queries must equal the oracle (the reference's gather_assignments +
count_lca_for_assignments restated in tests/lca_cases.py).  Then:

    table_build_ms    batch.lca_table from the host arrays (upload, sort, fold, compaction, one readback), median
    table_device_ms   CUDA events around the table build's device work (smb_set_profiling), median
    counts_device_ms  CUDA events around lca_counts' device work for the whole batch, median
    counts_e2e_ms     lca.ranked_counts from a resident batch: device work, copy-out and the per-query ordering, median
    loop_per_query_s  the reference's per-query loop (tests/lca_cases.oracle_counts: a dict hash -> [idx] per database,
                      a set of lineages and a dictionary tree per hash), timed on --loop-queries queries
    loop_batch_s_extrapolated  loop_per_query_s times the batch size: extrapolated, not run

Writes one JSON line to stdout and, with --out, to that file.

    python scripts/bench_lca.py [--repeats 5] [--loop-queries 5] [--out profiles/h100/bench_lca.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sig_kmers import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--loop-queries", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from sourmash_b200 import batch as B
    from sourmash_b200 import lca as L
    from tests import lca_cases as C
    dbs, queries = C.synth_lca(seed=1)
    tax = L.Taxonomy(dbs)
    hashes = np.concatenate([db.hashes for db in dbs])
    nodes = np.concatenate([tax.nodes_of(i, db) for i, db in enumerate(dbs)])
    off = np.concatenate([[0], np.cumsum([len(q) for q in queries])]).astype(np.uint64)
    sset = B.SketchSet.from_host(np.concatenate(queries), off)

    table = B.lca_table(hashes, nodes, tax.parent, tax.depth)               # warm-up, and the table checked below
    ranked = L.ranked_counts(table, sset, len(queries), False)
    for i, want in enumerate(C.synth_oracle(dbs, queries[:8])):
        assert [(tuple(tax.lineage(n)), c) for n, c in ranked[i]] == want, i

    build, build_dev, counts_dev, e2e = [], [], [], []
    B.set_profiling(True)
    for _ in range(args.repeats):
        B.synchronize()
        t = time.perf_counter()
        t2 = B.lca_table(hashes, nodes, tax.parent, tax.depth)
        build.append((time.perf_counter() - t) * 1e3)
        build_dev.append(B.last_kernel_ms(1))
        del t2
        B.lca_counts(table, sset, weights=False)
        counts_dev.append(B.last_kernel_ms(1))
    B.set_profiling(False)
    for _ in range(args.repeats):
        B.synchronize()
        t = time.perf_counter()
        L.ranked_counts(table, sset, len(queries), False)
        e2e.append((time.perf_counter() - t) * 1e3)

    dicts = []                                       # the reference's loaded form: hash -> [idx], idx -> lineage
    for db in dbs:
        d = {}
        for h, x in zip(db.hashes.tolist(), db.idx.tolist()):
            d.setdefault(h, []).append(x)
        dicts.append((d, {x: db.lid_to_lineage[db.idx_to_lid[x]] for x in db.idx_to_lid}))
    t = time.perf_counter()
    for i in range(args.loop_queries):
        want = C.oracle_counts(queries[i], dicts)
        assert want == [(tuple(tax.lineage(n)), c) for n, c in ranked[i]], i
    per_query = (time.perf_counter() - t) / args.loop_queries

    res = {
        "gpu": gpu_info(),
        "lineages": len(dbs[0].lid_to_lineage), "trie_nodes": len(tax.parent), "db_pairs": int(len(hashes)),
        "table_hashes": len(table), "queries": len(queries), "query_hashes": int(off[-1]),
        "count_rows": int(sum(len(r) for r in ranked)),
        "table_build_ms": statistics.median(build), "table_device_ms": statistics.median(build_dev),
        "counts_device_ms": statistics.median(counts_dev), "counts_e2e_ms": statistics.median(e2e),
        "loop_queries_timed": args.loop_queries, "loop_per_query_s": per_query,
        "loop_batch_s_extrapolated": per_query * len(queries),
        "parity": "8 queries equal the oracle; %d equal the reference loop" % args.loop_queries,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
