"""kmers.match_records on the GPU: the brute-force cases of tests/sig_kmers_cases.py, and the benchmark's workload
(reads sampled from synthetic genomes) at 10^5 reads against the per-record loop written with this package's MinHash,
on both probe paths and for a num sketch; and the `b200sigkmers` command on those reads."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sig_kmers_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu


def test_gpu_match_cases(tmp_path):
    from sourmash_b200.kmers import match_records
    from sourmash_b200.sketch import RecordBatch
    rng = np.random.default_rng(7)
    for i, (tag, q, recs, is_protein) in enumerate(C.cases(rng)):
        d = tmp_path / str(i)
        d.mkdir()
        res = match_records(q, RecordBatch(C.write_records(str(d), recs)), is_protein=is_protein)
        C.assert_same(res, C.brute(q, recs, is_protein=is_protein), tag)


def test_gpu_match_reads_both_probe_paths_and_num(tmp_path):
    "10^5 reads of the benchmark's workload; the per-record loop runs on the first 2 000 of them"
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import bench_sig_kmers as bench
    from sourmash_b200.kmers import match_records
    from sourmash_b200.sketch import RecordBatch
    genomes, path = bench.write_reads(str(tmp_path), n_genomes=4, genome_bp=500_000, n_reads=100_000)
    rb = RecordBatch([path])
    recs = [rb.sequence(i).decode() for i in range(2000)]
    sub = bench.write_subset(str(tmp_path), recs)
    for tag, q in bench.queries(genomes, scaled_small=1000, scaled_large=10, num=1000):
        full = match_records(q, rb)
        head = match_records(q, RecordBatch([sub]))
        C.assert_same(head, C.brute(q, recs), tag)
        cut = np.searchsorted(full.records, 2000)
        assert full.records[:cut].tolist() == head.records.tolist(), tag
        assert full.hashes[:cut].tolist() == head.hashes.tolist(), tag
        assert full.matched[:2000].tolist() == head.matched.tolist(), tag
        assert full.matched.any(), tag


def test_gpu_command_on_reads(tmp_path):
    "python -m sourmash_b200.sigkmers on 2 x 10^4 reads: the CSV rows are the matches of the matched reads"
    import csv
    import subprocess
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import bench_sig_kmers as bench
    from sourmash_b200.kmers import match_records
    from sourmash_b200.signature import SourmashSignature, save_signatures_to_json
    from sourmash_b200.sketch import RecordBatch
    genomes, path = bench.write_reads(str(tmp_path), n_genomes=4, genome_bp=200_000, n_reads=20_000)
    _, q = bench.queries(genomes, scaled_small=100)[0]
    sig = str(tmp_path / "q.sig")
    with open(sig, "wb") as fh:
        save_signatures_to_json([SourmashSignature(q, name="q")], fh)
    out = str(tmp_path / "k.csv")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.sigkmers", "--signatures", sig, "--sequences", path,
                        "--save-kmers", out, "--check-sequence", "--force"], capture_output=True, text=True, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    res = match_records(q, RecordBatch([path]), skip_invalid=True)
    keep = res.matched & ~res.has_invalid
    want = [int(h) for rec, h in zip(res.records, res.hashes) if keep[rec]]
    with open(out, newline="") as fh:
        got = [int(row["hashval"]) for row in csv.DictReader(fh)]
    assert got == want and len(got) > 100
    assert "found %d distinct matching hashes" % len(res.found) in r.stderr
