"""kmers.match_records end to end with the EMULATED build (emul_lib.py) against the reference's per-record loop written
with this package's MinHash (tests/sig_kmers_cases.py).  Run as a script by tests/test_sig_kmers_emulated.py.

    python tests/host_emul/sig_kmers_checks.py [name ...]
"""
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emulated_boot  # noqa: E402

LIB = emulated_boot.install()

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402
from sourmash_b200.kmers import match_records  # noqa: E402
from sourmash_b200.sketch import RecordBatch  # noqa: E402
from tests import sig_kmers_cases as C  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


@check
def match_vs_per_record_loop():
    rng = np.random.default_rng(7)
    with tempfile.TemporaryDirectory() as d:
        disagree = 0
        for tag, q, recs, is_protein in C.cases(rng):
            rb = RecordBatch(C.write_records(d, recs))
            assert len(rb) == len(recs)
            res = match_records(q, rb, is_protein=is_protein)
            C.assert_same(res, C.brute(q, recs, is_protein=is_protein), tag)
            if q.num:
                hit = np.zeros(len(recs), bool)
                hit[res.records] = True
                disagree += int((hit & ~res.matched).sum())
        assert disagree > 0, "no num case where a probe hit fails the record test"


@check
def match_large_query_and_overflow():
    "Q above the shared-memory table (global directory), and scaled = 1 with every window a match (staging overflow)"
    rng = np.random.default_rng(11)
    recs = C.dna_records(rng, 40)
    with tempfile.TemporaryDirectory() as d:
        rb = RecordBatch(C.write_records(d, recs))
        q = C.query_from(recs, "DNA", 31, rng, scaled=1, extra=20000, take=40)
        assert len(q) > 16382
        C.assert_same(match_records(q, rb), C.brute(q, recs), "global directory")
        big = ["".join(rng.choice(list("ACGT"), size=3000)) for _ in range(3)]
        q = C.query_from(big, "DNA", 21, rng, scaled=1, extra=0, take=3)
        rb = RecordBatch(C.write_records(d, big, parts=1))
        res = match_records(q, rb)
        assert len(res.hashes) > 2 * 512
        C.assert_same(res, C.brute(q, big), "every window")


@check
def match_launches_do_not_grow_with_records():
    rng = np.random.default_rng(3)
    recs = C.dna_records(rng, 60)
    q = C.query_from(recs, "DNA", 31, rng, scaled=2)
    counts = []
    with tempfile.TemporaryDirectory() as d:
        for n in (10, 60):
            rb = RecordBatch(C.write_records(d, recs[:n]))
            before = B.kernel_launches()
            match_records(q, rb)
            counts.append(B.kernel_launches() - before)
    assert counts[0] == counts[1], counts


@check
def match_input_errors():
    rng = np.random.default_rng(5)
    recs = C.dna_records(rng, 4)
    with tempfile.TemporaryDirectory() as d:
        rb = RecordBatch(C.write_records(d, recs, parts=1))
        q = C.query_from(recs, "DNA", 31, rng, scaled=2)
        try:
            match_records(q, rb, is_protein=True)
            raise AssertionError("protein input into a DNA sketch was accepted")
        except ValueError as exc:
            assert "cannot add protein sequence to DNA MinHash" in str(exc)
        empty = C.make_query("DNA", 31, scaled=2)
        res = match_records(empty, rb)
        assert len(res.hashes) == 0 and not res.matched.any()


@check
def match_overflow_rerun_and_skipped_records():
    """A record repeating one matched k-mer thousands of times overflows the first match buffer (rerun at the exact
    size); skip_invalid leaves records with invalid DNA out of found, for scaled and num queries."""
    rng = np.random.default_rng(13)
    with tempfile.TemporaryDirectory() as d:
        # the homopolymer k-mer with the smallest hash, and the largest scaled that keeps it: the first buffer holds
        # the expected probes (1/scaled of the windows) + 4 |Q| + 4096 matches, every window of the record matches
        h, base, k = min((C.make_query("DNA", k, scaled=1).seq_to_hashes(b * k)[0], b, k) for b in "ACGT" for k in (21, 25, 31, 33))
        scaled = 2**64 // h
        assert scaled >= 2
        rep = [base * 40000, "".join(rng.choice(list("ACGT"), size=300))]
        q = C.make_query("DNA", k, scaled=scaled)
        q.add_sequence(rep[0], True)
        assert list(q.hashes) == [h]
        rb = RecordBatch(C.write_records(d, rep, parts=1))
        res = match_records(q, rb)
        n_windows = 40000 - k + 1 + 300 - k + 1
        assert len(res.hashes) > n_windows / scaled + 4 + 4096
        C.assert_same(res, C.brute(q, rep), "overflow")
        recs = C.dna_records(rng, 30)
        rb = RecordBatch(C.write_records(d, recs))
        for q in (C.query_from(recs, "DNA", 21, rng, scaled=2), C.query_from(recs, "DNA", 21, rng, num=40)):
            res = match_records(q, rb, skip_invalid=True)
            _, matched, invalid, _ = C.brute(q, recs)
            found = q.copy_and_clear()
            for r, s in enumerate(recs):
                if matched[r] and not invalid[r]:
                    seq_mh = q.copy_and_clear()
                    seq_mh.add_sequence(s, True)
                    found += seq_mh.intersection(q)
            assert invalid[matched].any()
            assert res.found.tolist() == sorted(found.hashes), (q.num, len(res.found), len(found))


@check
def match_num_launches_do_not_grow_with_records():
    rng = np.random.default_rng(4)
    recs = C.dna_records(rng, 60)
    q = C.query_from(recs, "DNA", 21, rng, num=40)
    counts = []
    with tempfile.TemporaryDirectory() as d:
        for n in (15, 60):
            rb = RecordBatch(C.write_records(d, recs[:n]))
            before = B.kernel_launches()
            match_records(q, rb)
            counts.append(B.kernel_launches() - before)
    assert counts[0] == counts[1], counts


def _reference_loop(query_mh, files, kmers_csv, seqs_fa, *, is_protein=False):
    """The record loop of sig/__main__.py:1193-1256 with this package's MinHash and the sequences read one file at a
    time: the files it writes and the summary counts."""
    import csv
    found = query_mh.copy_and_clear()
    n_seqs = n_bp = n_kmers = n_found = 0
    with open(kmers_csv, "w", newline="") as kfp, open(seqs_fa, "wt") as sfp:
        w = csv.DictWriter(kfp, fieldnames=["sequence_file", "sequence_name", "kmer", "hashval"])
        w.writeheader()
        qh = query_mh.hashes
        for f in files:
            rb = RecordBatch([f])
            for name, i in zip(rb.names(), range(len(rb))):
                seq = rb.sequence(i).decode()
                seq_mh = query_mh.copy_and_clear()
                if is_protein:
                    seq_mh.add_protein(seq)
                else:
                    seq_mh.add_sequence(seq, True)
                if seq_mh.intersection(query_mh):
                    sfp.write(f">{name}\n{seq}\n")
                    n_found += 1
                    for kmer, h in seq_mh.kmers_and_hashes(seq, force=False, is_protein=is_protein):
                        if h in qh:
                            found.add_hash(h)
                            n_kmers += 1
                            w.writerow(dict(sequence_file=f, sequence_name=name, kmer=kmer, hashval=h))
                    found += seq_mh.intersection(query_mh)
                n_seqs += 1
                n_bp += len(seq)
    return n_seqs, n_bp, n_found, n_kmers, len(found)


@check
def command_writes_what_the_loop_writes():
    "b200sigkmers --save-kmers --save-sequences against the reference's loop: byte-identical files, same summary"
    import contextlib
    import io
    from sourmash_b200 import sigkmers
    from sourmash_b200.signature import SourmashSignature, save_signatures_to_json
    rng = np.random.default_rng(21)
    dna = [r.replace("N", "A") for r in C.dna_records(rng, 30)]          # invalid DNA would stop the reference's loop
    prot = C.protein_records(rng, 20)
    with tempfile.TemporaryDirectory() as d:
        for tag, q, recs, extra in (("dna scaled", C.query_from(dna, "DNA", 21, rng, scaled=2), dna, []),
                                    ("dna num", C.query_from(dna, "DNA", 31, rng, num=30), dna, []),
                                    ("translate", C.query_from(dna, "dayhoff", 5, rng, scaled=2), dna, ["--translate"]),
                                    ("protein", C.query_from(prot, "protein", 6, rng, scaled=2, is_protein=True), prot, [])):
            files = C.write_records(d, recs)
            sig = os.path.join(d, "q.sig")
            with open(sig, "wb") as fh:
                save_signatures_to_json([SourmashSignature(q, name="q")], fh)
            want = _reference_loop(q, files, os.path.join(d, "want.csv"), os.path.join(d, "want.fa"),
                                   is_protein=q.moltype != "DNA" and not extra)
            err = io.StringIO()
            with contextlib.redirect_stderr(err):
                assert sigkmers.main(["--signatures", sig, "--sequences", *files,
                                      "--save-kmers", os.path.join(d, "got.csv"),
                                      "--save-sequences", os.path.join(d, "got.fa")] + extra) == 0
            for a, b in (("want.csv", "got.csv"), ("want.fa", "got.fa")):
                with open(os.path.join(d, a), "rb") as fa, open(os.path.join(d, b), "rb") as fb:
                    assert fa.read() == fb.read(), (tag, b)
            text = err.getvalue()
            n_seqs, n_bp, n_found, n_kmers, n_distinct = want
            assert f"searched {n_seqs} sequences from {len(files)} files, containing a total of " \
                   f"{sigkmers.format_bp(n_bp)}." in text, (tag, text)
            assert f"matched and saved a total of {n_found} sequences" in text, (tag, text)
            assert f"matched and saved a total of {n_kmers} k-mers." in text, (tag, text)
            assert f"found {n_distinct} distinct matching hashes" in text, (tag, text)


if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        t0 = time.time()
        CHECKS[name]()
        print("ok  %s (%.1f s)" % (name, time.time() - t0), flush=True)
    print("sig kmers checks passed")
