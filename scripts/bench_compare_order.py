#!/usr/bin/env python
"""compare_jaccard_device on two 10 000-sketch sets where counting rows in label order cannot help, so that its cost
(labels, the sort by label, the indirection of the count kernel) shows up undiluted:

    family_contiguous  the benchmark's set (synth_sketches(10 000), 100 families at a stride of 100) with its rows
                       permuted family-major, slot (r mod 100) * 100 + r / 100: index order already is family order
    own_pools          synth_sketches(10 000, n_families=10 000): nearly every row draws from a pool of its own

The sets are drawn once; each measurement is a subprocess on the library of one checkout.  With --against TREE (another
built checkout, e.g. the parent commit) it alternates with this tree --rounds times.  Every line carries the tree ("this" or
"against"), the set, the median and least ms per call over --steps calls (CUDA events, after warm-up) and a hash of the matrix, which
must agree between the trees.

    python scripts/bench_compare_order.py --against PARENT_TREE [--rounds 3] > profiles/h100/bench_compare_order.txt
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sets():
    from sourmash_b200.synth import synth_sketches
    h, off = synth_sketches(10_000)
    rows = [h[int(off[i]):int(off[i + 1])] for i in range(10_000)]
    order = np.empty(10_000, np.int64)
    r = np.arange(10_000)
    order[(r % 100) * 100 + r // 100] = r
    fam = [rows[i] for i in order]
    off_f = np.zeros(10_001, np.uint64)
    off_f[1:] = np.cumsum([len(x) for x in fam])
    yield "family_contiguous", np.concatenate(fam), off_f
    yield "own_pools", *synth_sketches(10_000, n_families=10_000)


def measure(tree, steps, data):
    sys.path.insert(0, tree)
    import torch
    from sourmash_b200 import batch as B
    torch.cuda.set_device(0)
    B.set_device(0)
    s = torch.cuda.current_stream()
    B.set_stream(s.cuda_stream)
    z = np.load(data)
    for name in ("family_contiguous", "own_pools"):
        h, off = z[name + "_h"], z[name + "_off"]
        n = len(off) - 1
        sset = B.SketchSet.from_host(h, off)
        d_out = torch.empty((n, n), dtype=torch.float64, device="cuda")
        for _ in range(3):
            B.compare_jaccard_device(sset, d_out.data_ptr())
        ms = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            B.compare_jaccard_device(sset, d_out.data_ptr())
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        digest = hashlib.sha256(d_out.cpu().numpy().tobytes()).hexdigest()[:16]
        print(json.dumps({"tree": "this" if tree == ROOT else "against", "set": name, "ms_median": round(statistics.median(ms), 3),
                          "ms_min": round(min(ms), 3), "steps": steps, "matrix_sha256_16": digest}), flush=True)
        del sset, d_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--data", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--against", default=None, help="another built checkout to alternate with")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if args.data:
        measure(os.path.abspath(args.tree), args.steps, args.data)
        return
    sys.path.insert(0, ROOT)
    with tempfile.TemporaryDirectory() as td:        # the sets are drawn once, for every run
        data = os.path.join(td, "sets.npz")
        np.savez(data, **{name + k: v for name, h, off in sets() for k, v in (("_h", h), ("_off", off))})
        trees = [ROOT] if not args.against else [os.path.abspath(args.against), ROOT]
        if args.against:
            smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                 capture_output=True, text=True)
            print(json.dumps({"gpu": smi.stdout.strip()}), flush=True)
        for _ in range(args.rounds if args.against else 1):
            for tree in trees:
                subprocess.check_call([sys.executable, os.path.abspath(__file__), "--tree", tree, "--steps", str(args.steps),
                                       "--data", data])


if __name__ == "__main__":
    main()
