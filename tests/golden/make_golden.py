#!/usr/bin/env python
"""Generate the golden parity fixtures in this directory from the reference's own test data.

Run once with the reference checkout (oracle/reference.py: BASELINE.json's reference_path, or SMB_REFERENCE):

    SMB_REFERENCE=<checkout> python tests/golden/make_golden.py

Outputs (committed):
  golden_arrays_1.npz, golden_arrays_2.npz   uint64 hash arrays pulled verbatim out of the reference's .sig fixtures
  golden_meta.json    md5sums, parameters and known-answer values quoted from the reference tests
  ecoli_k12.part1.fna.gz, ecoli_k12.part2.fna.gz   data/GCF_000005845.2_ASM584v2_genomic.fna.gz (BASELINE config 1
                      input) as two gzip members, split at a line; their concatenation is the genome's .fna.gz
  genome-s10.fa.gz    byte copy of tests/test-data/genome-s10.fa.gz (multi-record FASTA, num=500 golden sig)
  ecoli.faa, ecoli.genes.fna   byte copies of the protein / gene inputs of the known-good protein tests

Nothing here imports the reference's code (it cannot be built in this image: no Rust toolchain);
the .sig files are plain JSON written by the reference and are the pinned expected outputs.
"""
import gzip
import json
import os
import shutil
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle.reference import checkout  # noqa: E402

REF = checkout()
TD = os.path.join(REF, "tests", "test-data")
HERE = os.path.dirname(os.path.abspath(__file__))


def load_sig(path):
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rt") as fh:
        return json.load(fh)


def sketches(path):
    for rec in load_sig(path):
        for s in rec["signatures"]:
            yield rec, s


arrays = {}
meta = {"source": "sourmash-bio/sourmash tests/test-data + data/ (reference commit 6ae9cd32)"}

# --- E. coli K-12 golden signature (BASELINE config 1) -------------------------------------
ecoli = {}
for rec, s in sketches(os.path.join(TD, "GCF_000005845.2_ASM584v2_genomic.fna.gz.sig")):
    k = s["ksize"]
    arrays[f"ecoli_k{k}"] = np.array(s["mins"], dtype=np.uint64)
    ecoli[str(k)] = {"md5sum": s["md5sum"], "max_hash": s["max_hash"], "seed": s["seed"],
                     "num": s["num"], "n": len(s["mins"])}
meta["ecoli"] = ecoli
with gzip.open(os.path.join(REF, "data", "GCF_000005845.2_ASM584v2_genomic.fna.gz"), "rb") as fh:
    lines = fh.read().split(b"\n")
for i, part in enumerate((b"\n".join(lines[:len(lines) // 2]) + b"\n", b"\n".join(lines[len(lines) // 2:]))):
    with open(os.path.join(HERE, "ecoli_k12.part%d.fna.gz" % (i + 1)), "wb") as fh:
        with gzip.GzipFile(fileobj=fh, mode="wb", compresslevel=9, mtime=0, filename="") as g:
            g.write(part)

# --- 47.fa / 63.fa (k=31, scaled=1000): tests/test_prefetch.py:272, test_index_protocol.py:217-269
for name in ("47", "63"):
    for rec, s in sketches(os.path.join(TD, f"{name}.fa.sig")):
        assert s["ksize"] == 31 and s["max_hash"] == 18446744073709552
        arrays[f"s{name}"] = np.array(s["mins"], dtype=np.uint64)
        meta[f"s{name}_md5"] = s["md5sum"]
meta["s47_s63"] = {"common": 2529, "union": 7886, "n47": 5177, "n63": 5238,
                   "jaccard": 2529 / 7886}

# --- demo/*.sig (num=500, k=31) and the exact 7x7 matrix of tests/test_compare.py:49-61 ------
demo_files = sorted(f for f in os.listdir(os.path.join(TD, "demo")) if f.endswith(".sig"))
meta["demo_files"] = demo_files
for i, f in enumerate(demo_files):
    (rec, s), = list(sketches(os.path.join(TD, "demo", f)))
    assert s["num"] == 500 and s["ksize"] == 31
    arrays[f"demo{i}"] = np.array(s["mins"], dtype=np.uint64)
meta["demo_matrix"] = [
    [1.0, 0.356, 0.078, 0.086, 0.0, 0.0, 0.0],
    [0.356, 1.0, 0.072, 0.078, 0.0, 0.0, 0.0],
    [0.078, 0.072, 1.0, 0.074, 0.0, 0.0, 0.0],
    [0.086, 0.078, 0.074, 1.0, 0.0, 0.0, 0.0],
    [0.0, 0.0, 0.0, 0.0, 1.0, 0.382, 0.364],
    [0.0, 0.0, 0.0, 0.0, 0.382, 1.0, 0.386],
    [0.0, 0.0, 0.0, 0.0, 0.364, 0.386, 1.0],
]

# --- scaled100 / n10000 E. coli vs Salmonella: tests/test_jaccard.py:175-264 -----------------
for tag, sub in (("scaled100", "scaled100"), ("n10000", "n10000")):
    for short, fn in (("ecoli", "GCF_000005845.2_ASM584v2_genomic.fna.gz.sig.gz"),
                      ("salmonella", "GCF_000006945.1_ASM694v1_genomic.fna.gz.sig.gz")):
        recs = list(sketches(os.path.join(TD, sub, fn)))
        rec, s = recs[0]          # load_signatures(...)[0].minhash in the reference test
        arrays[f"{tag}_{short}"] = np.array(s["mins"], dtype=np.uint64)
        meta[f"{tag}_{short}"] = {"ksize": s["ksize"], "max_hash": s["max_hash"],
                                  "num": s["num"], "md5sum": s["md5sum"], "n": len(s["mins"])}
meta["scaled100_jaccard"] = {"100": 0.01644, "1000": 0.01874, "10000": 0.01, "100000": 0.01}
meta["n10000_jaccard"] = {"10000": 0.0183, "1000": 0.011, "100": 0.01, "10": 0.0}

# --- genome-s10.fa.gz (multi-record FASTA) and its num=500 DNA sketches ----------------------
shutil.copyfile(os.path.join(TD, "genome-s10.fa.gz"), os.path.join(HERE, "genome-s10.fa.gz"))
s10 = {}
for rec, s in sketches(os.path.join(TD, "genome-s10.fa.gz.sig")):
    if s["molecule"].lower() != "dna":
        # protein sketches of the same genome (six-frame translation, num=500): k stored x3
        arrays[f"s10_prot_k{s['ksize']}"] = np.array(s["mins"], dtype=np.uint64)
        meta.setdefault("genome_s10_protein", {})[str(s["ksize"])] = {
            "num": s["num"], "md5sum": s["md5sum"], "seed": s["seed"], "molecule": s["molecule"], "n": len(s["mins"])}
        continue
    key = f"s10_k{s['ksize']}"
    arrays[key] = np.array(s["mins"], dtype=np.uint64)
    s10[str(s["ksize"])] = {"num": s["num"], "md5sum": s["md5sum"], "seed": s["seed"],
                            "max_hash": s.get("max_hash", 0), "n": len(s["mins"])}
meta["genome_s10"] = s10

# --- the scaled_siglist of tests/test_compare.py:28-40 (ANI matrices :94-190): byte copies ------
for f in ("2.fa.sig", "2+63.fa.sig", "63.fa.sig"):
    shutil.copyfile(os.path.join(TD, f), os.path.join(HERE, f))
meta["compare_ani_k31"] = {   # np.testing.assert_array_almost_equal(..., decimal=3) in the reference
    "order": ["2.fa.sig", "2+63.fa.sig", "47.fa.sig", "63.fa.sig"],
    "jaccard": [[1.0, 0.978, 0.0, 0.0], [0.978, 1.0, 0.96973012, 0.99262776],
                [0.0, 0.96973012, 1.0, 0.97697011], [0.0, 0.99262776, 0.97697011, 1.0]],
    "containment": [[1, 0.966, 0.0, 0.0], [1, 1.0, 0.97715525, 1.0],
                    [0.0, 0.96377054, 1.0, 0.97678608], [0.0, 0.98667513, 0.97715525, 1.0]],
    "max_containment": [[1.0, 1.0, 0.0, 0.0], [1.0, 1.0, 0.97715525, 1.0],
                        [0.0, 0.97715525, 1.0, 0.97715525], [0.0, 1.0, 0.97715525, 1.0]],
    "avg_containment": [[1.0, 0.983, 0.0, 0.0], [0.983, 1.0, 0.97046289, 0.99333757],
                        [0.0, 0.97046289, 1.0, 0.97697067], [0.0, 0.99333757, 0.97697067, 1.0]]}

# --- two reference-written .sig files, byte copies, for the JSON loader tests ----------------
shutil.copyfile(os.path.join(TD, "47.fa.sig"), os.path.join(HERE, "47.fa.sig"))
shutil.copyfile(os.path.join(TD, "genome-s10.fa.gz.sig"), os.path.join(HERE, "genome-s10.fa.gz.sig"))

# --- protein-family fixtures (SURVEY §8 f4): tests/test_sourmash_sketch.py:1340-1376 ---------
# ecoli.faa (2 protein records) and ecoli.genes.fna (the 2 genes) are the inputs of the
# reference's known-good tests; benchmark.input_prot.sig / benchmark.prot.sig are their expected
# num=500, k=7 (ksize 21) protein sketches (input protein / six-frame translation).
shutil.copyfile(os.path.join(TD, "ecoli.faa"), os.path.join(HERE, "ecoli.faa"))
shutil.copyfile(os.path.join(TD, "ecoli.genes.fna"), os.path.join(HERE, "ecoli.genes.fna"))
prot = {}
for tag, fn in (("input_prot", "benchmark.input_prot.sig"), ("translate_prot", "benchmark.prot.sig"),
                ("benchmark_dna", "benchmark.dna.sig")):
    (rec, s), = list(sketches(os.path.join(TD, fn)))
    arrays[f"bench_{tag}"] = np.array(s["mins"], dtype=np.uint64)
    prot[tag] = {"name": rec["name"], "ksize": s["ksize"], "num": s["num"], "seed": s["seed"],
                 "molecule": s["molecule"], "md5sum": s["md5sum"], "n": len(s["mins"])}
meta["protein_benchmarks"] = prot
# 2 x 2 similarities of tests/test_sourmash_compute.py:810-860 (round(., 3)), k=21 (7 residues), num=500
meta["protein_2x2"] = {"aa1_trans1": 0.0, "aa2_trans1": 0.166, "aa1_trans2": 0.174, "aa2_trans2": 0.0}

# --- gather fixtures: tests/test_index_protocol.py:1057-1097 (12 genomes + their combined query,
# k=21 / 31 / 51 scaled sketches); byte copies of the reference-written .sig files ------------
os.makedirs(os.path.join(HERE, "gather"), exist_ok=True)
for f in sorted(os.listdir(os.path.join(TD, "gather"))):
    if f.endswith(".sig"):
        shutil.copyfile(os.path.join(TD, "gather", f), os.path.join(HERE, "gather", f))
meta["gather_k21_expected"] = [  # (first word of the match name, new hashes covered), in pick order
    ["NC_003198.1", 487], ["NC_000853.1", 192], ["NC_011978.1", 169], ["NC_002163.1", 157],
    ["NC_003197.2", 152], ["NC_009486.1", 92], ["NC_006905.1", 76], ["NC_011080.1", 59],
    ["NC_011274.1", 42], ["NC_006511.1", 31], ["NC_011294.1", 7], ["NC_004631.1", 2]]

# --- known-answer values quoted from the reference's tests ----------------------------------
meta["kat"] = {
    "hash_murmur_ACG_42": 1731421407650554201,            # tests/test_minhash.py:1239-1262
    "n1_k4_ATGC": [12415348535738636339],                  # tests/test_minhash.py:98-112
    "max_hash_scaled_100": 184467440737095520,             # src/core/tests/minhash.rs:177-180
    "max_hash_scaled_1000": 18446744073709552,
    "merge_k10_num20": {                                   # src/core/tests/minhash.rs:29-54
        "a": ["TGCCGCCCAGCA", "GTCCGCCCAGTGA"], "b": ["TGCCGCCCAGCA", "GTCCGCCCAGTGG"],
        "merged": [2996412506971915891, 4448613756639084635, 8373222269469409550,
                   9390240264282449587, 11085758717695534616, 11668188995231815419,
                   11760449009842383350, 14682565545778736889]},
    "invalid_dna_k3": {"AAANNCCCTN": 3, "NAAA": 1},        # src/core/tests/minhash.rs:56-66
    # tests/test_minhash.py:390-454: residues are re-encoded before hashing
    "dayhoff_CADHIFC": "abcdefa", "dayhoff_CADHIF*": "abcdef*", "hp_ANA": "hph", "hp_AN*": "hp*",
    # tests/test_minhash.py:313-358, src/core/tests/minhash.rs:153-175, signature.rs:1031-1039
    "AGYYG_k2": {"protein": 4, "dayhoff": 4, "hp": 1}, "ACTGAC_translate_k2": 2,
    "AGY_k2_protein": 2, "AGY_k1_protein": 3,
    # tests/test_minhash.py:361-370
    "translate_codon": {"TCT": "S", "TC": "S", "T": "X"},
}

names = sorted(arrays, key=lambda k: -arrays[k].nbytes)         # two archives of about equal size: each under 1 MB
parts, sizes = ({}, {}), [0, 0]
for k in names:
    i = 0 if sizes[0] <= sizes[1] else 1
    parts[i][k] = arrays[k]
    sizes[i] += arrays[k].nbytes
np.savez_compressed(os.path.join(HERE, "golden_arrays_1.npz"), **parts[0])
np.savez_compressed(os.path.join(HERE, "golden_arrays_2.npz"), **parts[1])
with open(os.path.join(HERE, "golden_meta.json"), "w") as fh:
    json.dump(meta, fh, indent=1)
print("wrote", len(arrays), "arrays")
