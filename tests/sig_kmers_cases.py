"""Cases of `sig kmers` matching (kmers.match_records) and their brute force: the reference's per-record loop
(src/sourmash/sig/__main__.py:1206-1256) written with this package's MinHash, one record at a time.  Used by the
emulated-library checks (tests/host_emul/sig_kmers_checks.py) and by tests/test_gpu_sig_kmers.py."""
import gzip
import os

import numpy as np

from sourmash_b200.minhash import MinHash


def random_records(rng, n, lo, hi, *, alphabet="ACGTacgtN", weights=None):
    w = np.asarray(weights if weights is not None else [1.0] * len(alphabet), float)
    w /= w.sum()
    letters = np.array(list(alphabet))
    return ["".join(rng.choice(letters, p=w, size=int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def write_records(directory, recs, *, parts=3):
    """The records spread over FASTA, FASTQ and gzipped FASTA files; returns the paths in record order."""
    paths = []
    chunks = np.array_split(np.arange(len(recs)), parts)
    for pi, idx in enumerate(chunks):
        kind = ("fa", "fq", "fa.gz")[pi % 3]
        path = os.path.join(directory, "part%d.%s" % (pi, kind))
        text = ""
        for i in idx.tolist():
            s = recs[i]
            text += ("@r%d x\n%s\n+\n%s\n" % (i, s, "I" * len(s))) if kind == "fq" else (">r%d x\n%s\n" % (i, s))
        if kind.endswith(".gz"):
            with gzip.open(path, "wt") as fh:
                fh.write(text)
        else:
            with open(path, "w") as fh:
                fh.write(text)
        paths.append(path)
    return paths


def make_query(moltype, k, *, scaled=0, num=0, seed=42):
    return MinHash(num, k, scaled=scaled, seed=seed, is_protein=moltype == "protein", dayhoff=moltype == "dayhoff",
                   hp=moltype == "hp")


def brute(query_mh, recs, *, is_protein=False):
    """(records, ordinals, hashes) of every window whose hash is in the query, per-record matched / has_invalid, and
    the found hashes -- one record at a time, as the reference's loop sees them."""
    qh = set(query_mh.hashes)
    rows, matched, invalid = [], [], []
    found = query_mh.copy_and_clear()
    dna = query_mh.moltype == "DNA"
    for r, s in enumerate(recs):
        seq_mh = query_mh.copy_and_clear()
        if is_protein:
            seq_mh.add_protein(s)
        else:
            seq_mh.add_sequence(s, True)
        common = seq_mh.intersection(query_mh)
        matched.append(bool(common))
        if common:
            found += common
        invalid.append(dna and len(s) >= query_mh.ksize and any(c not in "ACGT" for c in s.upper()))
        # kmers_and_hashes order: DNA windows by position (invalid ones as 0); protein-family windows as
        # seq_to_hashes(force=False) lists them (translated: frame 0 forward, frame 0 reverse, frame 1 forward, ...)
        if dna:
            hv = query_mh.copy_and_clear().seq_to_hashes(s.upper(), force=True, bad_kmers_as_zeroes=True)
        else:
            hv = query_mh.copy_and_clear().seq_to_hashes(s.upper(), is_protein=is_protein)
        for o, h in enumerate(hv):
            if h and h in qh and (not query_mh.scaled or h <= query_mh._max_hash):
                rows.append((r, o, h))
    return rows, np.array(matched, bool), np.array(invalid, bool), np.array(sorted(found.hashes), np.uint64)


def assert_same(res, want, tag):
    rows, matched, invalid, found = want
    got = list(zip(res.records.tolist(), res.ordinals.tolist(), res.hashes.tolist()))
    assert got == rows, (tag, len(got), len(rows), [g for g in got if g not in rows][:3], [w for w in rows if w not in got][:3])
    assert res.matched.tolist() == matched.tolist(), (tag, np.nonzero(res.matched != matched)[0][:5])
    assert res.has_invalid.tolist() == invalid.tolist(), (tag, np.nonzero(res.has_invalid != invalid)[0][:5])
    assert res.found.tolist() == found.tolist(), (tag, len(res.found), len(found))


def dna_records(rng, n=24):
    """Mixed case, N runs, records shorter than k, empty records, records of only N, a repeated k-mer and a palindrome."""
    recs = random_records(rng, n, 0, 260, weights=[.2, .2, .2, .2, .04, .04, .04, .04, .04])
    recs += ["", "N" * 80, "ACGT" * 3, "ACGTACGTAC" * 12, "ACGTTAACGTTAACGT" * 8, "GAATTC" * 20 + "nnnn" + "acgt" * 15]
    return recs


def protein_records(rng, n=20):
    return random_records(rng, n, 0, 200, alphabet="ACDEFGHIKLMNPQRSTVWYacdX*")


def query_from(recs, moltype, k, rng, *, scaled=0, num=0, is_protein=False, extra=50, take=6):
    """A query holding the hashes of a few of the records plus random hashes that match nothing."""
    q = make_query(moltype, k, scaled=scaled, num=num)
    for s in recs[:take]:
        if is_protein:
            q.add_protein(s)
        else:
            q.add_sequence(s, True)
    mx = q._max_hash if scaled else 2**64 - 1
    q.add_many(rng.integers(1, max(mx // 2, 2), size=extra, dtype=np.uint64))
    return q


def cases(rng):
    """(tag, query, records, is_protein) for the moltype x k combinations."""
    dna = dna_records(rng)
    prot = protein_records(rng)
    out = []
    for k in (21, 31, 51, 17):
        out.append(("dna k=%d scaled=2" % k, query_from(dna, "DNA", k, rng, scaled=2), dna, False))
    out.append(("dna k=31 scaled=1", query_from(dna, "DNA", 31, rng, scaled=1), dna, False))
    out.append(("dna k=21 num=40", query_from(dna, "DNA", 21, rng, num=40), dna, False))
    # a record that holds all of the query's k-mers among many more: probe hits, but its bottom num misses them
    a = random_records(rng, 1, 120, 120, alphabet="ACGT")[0]
    long_recs = [a, random_records(rng, 1, 2000, 2000, alphabet="ACGT")[0] + a, dna[0]]
    out.append(("dna k=21 num=5 hits without a match", query_from([a], "DNA", 21, rng, num=5, extra=0, take=1),
                long_recs, False))
    for mol in ("protein", "dayhoff", "hp"):
        out.append(("%s residues" % mol, query_from(prot, mol, 7, rng, scaled=2, is_protein=True), prot, True))
        out.append(("%s translate" % mol, query_from(dna, mol, 5, rng, scaled=2), dna, False))
    out.append(("protein num=30", query_from(prot, "protein", 6, rng, num=30, is_protein=True), prot, True))
    return out
