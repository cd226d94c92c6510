"""`sourmash scripts b200sigkmers`: the k-mers and sequences that carry a sketch's hashes, hashed and matched on a GPU.

The reference's `sourmash sig kmers` (src/sourmash/sig/__main__.py:1087-1304) merges the given signatures into one
query sketch and then walks every record of every sequence file in Python: a sketch of the record, its intersection
with the query, and for a matching record a hash of every k-mer and a set lookup.  Here all records are read natively
(``sketch.RecordBatch``) and matched in one library call (``kmers.match_records``); Python only writes the outputs of
the matching records.  The options, the files written and the messages follow the reference:

    sourmash scripts b200sigkmers --signatures q.sig --sequences reads.fq.gz --save-kmers k.csv --save-sequences s.fa

``--save-kmers`` writes one CSV row per k-mer occurrence of a matching record (sequence_file, sequence_name, kmer,
hashval), ``--save-sequences`` the matching records as FASTA.  Sequences are FASTA / FASTQ, plain, gzip or bzip2.
Signatures are read from .sig / .sig.gz JSON files, named on the command line or listed in --from-file; unlike the
reference, .zip collections, directories and picklists are not accepted.  Also ``python -m sourmash_b200.sigkmers ...``.
"""
import argparse
import csv
import gzip
import os
import sys

import numpy as np

from .plugin import CommandLinePlugin, _select_args


def _notify(args, msg):
    if not getattr(args, "quiet", False):
        print("\r\033[K", end="", file=sys.stderr)
        print(msg, file=sys.stderr)


def _error(msg):
    print("\r\033[K", end="", file=sys.stderr)
    print(msg, file=sys.stderr)


def format_bp(bp):
    "search.py:667-678"
    bp = float(bp)
    if bp < 500:
        return f"{bp:.0f} bp"
    elif bp <= 500e3:
        return f"{round(bp / 1e3, 1):.1f} kbp"
    elif bp < 500e6:
        return f"{round(bp / 1e6, 1):.1f} Mbp"
    elif bp < 500e9:
        return f"{round(bp / 1e9, 1):.1f} Gbp"
    return "???"


def merge_query(args):
    """The merged query sketch of --signatures / --from-file, flat (sig/__main__.py:1113-1141); exits like the
    reference on incompatible signatures and when there is none."""
    from .signature import load_signatures_from_json
    files = list(args.signatures)
    if args.from_file:
        with open(args.from_file) as fh:
            files += [line.strip() for line in fh if line.strip()]
    query_mh, n = None, 0
    for loc in files:
        for sig in load_signatures_from_json(loc, select_moltype=args.moltype):
            if args.ksize is not None and sig.minhash.ksize != args.ksize:     # k in residues for protein families
                continue
            n += 1
            if query_mh is None:
                query_mh = sig.minhash.copy_and_clear().flatten()
            try:
                query_mh.merge(sig.minhash.flatten())
            except (TypeError, ValueError) as exc:
                _error(f"ERROR when merging signature '{sig}' ({sig.md5sum()[:8]}) from file {loc}")
                _error(str(exc))
                raise SystemExit(-1)
    if not n:
        _error("no signatures in query!?")
        raise SystemExit(-1)
    _notify(args, f"loaded and merged {n} signatures")
    return query_mh


class Command_B200SigKmers(CommandLinePlugin):
    command = "b200sigkmers"
    description = "retrieve the k-mers and sequences that carry a sketch's hashes, on a GPU (sig kmers)"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("--signatures", nargs="*", default=[])
        p.add_argument("-f", "--force", action="store_true", help="continue past invalid sequences")
        p.add_argument("--from-file", help="a text file containing a list of files to load signatures from")
        _select_args(p)
        p.set_defaults(moltype=None)              # like the reference: any moltype unless one is asked for
        p.add_argument("--sequences", nargs="+", required=True, help="FASTA/FASTQ/bz2/gz files with sequences")
        p.add_argument("--save-kmers", help="save k-mers and hash values to a CSV file")
        p.add_argument("--save-sequences", help="save sequences with matching hashes to a FASTA file")
        p.add_argument("--translate", action="store_true",
                       help="translate DNA k-mers into amino acids (for protein, dayhoff, and hp sketches)")
        p.add_argument("--check-sequence", action="store_true",
                       help="complain if input sequence is invalid (NOTE: only checks DNA)")

    def main(self, args):
        super().main(args)
        from .kmers import kmer_strings, match_records
        from .sketch import RecordBatch
        query_mh = merge_query(args)
        if query_mh.moltype == "DNA" and args.translate:
            _error("ERROR: cannot use --translate with DNA sketches.")
            raise SystemExit(-1)
        if not query_mh:
            _notify(args, "ERROR: no hashes in query signature!?")
            raise SystemExit(-1)
        is_protein = query_mh.moltype != "DNA" and not args.translate
        _notify(args, "")
        _notify(args, "merged signature has the following properties:")
        _notify(args, f"k={query_mh.ksize} molecule={query_mh.moltype} num={query_mh.num} scaled={query_mh.scaled} "
                      f"seed={query_mh.seed}")
        _notify(args, f"total hashes in merged signature: {len(query_mh)}")
        _notify(args, "")
        _notify(args, "now processing sequence files for matches!")

        kmer_fp = kmer_w = seq_fp = None
        if args.save_kmers:
            kmer_fp = gzip.open(args.save_kmers, "wt", newline="") if args.save_kmers.endswith(".gz") \
                else open(args.save_kmers, "w", newline="")
            kmer_w = csv.DictWriter(kmer_fp, fieldnames=["sequence_file", "sequence_name", "kmer", "hashval"])
            kmer_w.writeheader()
        if args.save_sequences:
            seq_fp = open(args.save_sequences, "wt", encoding="utf-8")
        try:
            return self._run(args, query_mh, is_protein, kmer_w, seq_fp, RecordBatch, match_records, kmer_strings)
        except SystemExit:
            # The reference's `sig kmers` leaves its outputs unflushed when it exits with -1 on invalid DNA
            # (--check-sequence without --force): the files keep only what the io buffers had written out (whole 8 KB
            # blocks).  The same io objects got the same writes here; their unwritten rest goes nowhere.
            for fp in (kmer_fp, seq_fp):
                if fp is not None:
                    devnull = os.open(os.devnull, os.O_WRONLY)
                    os.dup2(devnull, fp.fileno())
                    os.close(devnull)
            raise
        finally:
            for fp in (kmer_fp, seq_fp):      # after a ValueError (--save-kmers on invalid DNA) the reference's are flushed
                if fp is not None:
                    fp.close()

    @staticmethod
    def _run(args, query_mh, is_protein, kmer_w, seq_fp, RecordBatch, match_records, kmer_strings):
        rb = RecordBatch(args.sequences)
        # check_sequence: add_sequence(seq, force=False) raises on a record with an invalid DNA k-mer; such a record
        # is skipped (--force) and adds nothing to found_mh
        check = args.check_sequence and query_mh.moltype == "DNA"
        res = match_records(query_mh, rb, is_protein=is_protein, skip_invalid=check)
        names = rb.names()
        lengths = rb.lengths.astype(np.int64)
        invalid = res.has_invalid if check else np.zeros(len(rb), bool)
        first = np.searchsorted(res.records, np.arange(len(rb) + 1)) if len(rb) else np.zeros(1, np.int64)
        found = set(res.found.tolist())
        n_seqs = n_bp = n_kmers = n_found_seqs = n_bp_saved = 0
        threshold = 1e6
        for fi, filename in enumerate(args.sequences):
            _notify(args, f"opening sequence file '{filename}'")
            recs = np.nonzero(rb.files == fi)[0]
            # records with something to do: a match, an error, or the bp count crossing a progress mark
            cum = n_bp + np.cumsum(np.where(invalid[recs], 0, lengths[recs]))
            marks = np.floor(cum / 1e6) > np.floor(np.concatenate(([n_bp], cum[:-1])) / 1e6)
            busy = np.nonzero(res.matched[recs] | invalid[recs] | marks)[0]
            before = np.concatenate(([0], np.cumsum(lengths[recs])))   # bp of the file's records before position j
            last = -1                                                  # position of the last busy record
            for j in busy.tolist():
                n_seqs += j - last - 1                                 # the quiet records in between
                n_bp += int(before[j] - before[last + 1])
                last = j
                i = int(recs[j])
                name = names[i]
                if invalid[i]:
                    seqname = name if len(name) <= 40 else name[:37] + "..."
                    seq = rb.sequence(i).decode("utf-8", "replace")
                    L, k = len(seq), query_mh.ksize
                    bad = next(p for p in range(L) if seq[p].upper() not in "ACGT")
                    w = max(bad - k + 1, 0)
                    _notify(args, f"ERROR in sequence '{seqname}', file '{filename}'")
                    _notify(args, f"invalid DNA character in input k-mer: {seq[w:w + k].upper()}")
                    if args.force:
                        _notify(args, "(continuing)")
                        continue
                    raise SystemExit(-1)
                if res.matched[i]:
                    seq = rb.sequence(i).decode("utf-8", "replace")
                    if seq_fp is not None:
                        seq_fp.write(f">{name}\n{seq}\n")
                        n_found_seqs += 1
                        n_bp_saved += len(seq)
                    if kmer_w is not None:
                        if query_mh.moltype == "DNA" and res.has_invalid[i]:
                            # kmers_and_hashes(seq, force=False) raises here, as in the reference
                            list(query_mh.copy_and_clear().kmers_and_hashes(seq, force=False, is_protein=is_protein))
                        lo, hi = int(first[i]), int(first[i + 1])
                        hashes = res.hashes[lo:hi].tolist()
                        for kmer, h in zip(kmer_strings(query_mh, seq, res.ordinals[lo:hi].tolist(), is_protein=is_protein),
                                           hashes):
                            kmer_w.writerow(dict(sequence_file=filename, sequence_name=name, kmer=kmer, hashval=h))
                        n_kmers += hi - lo
                        found.update(hashes)                            # found_mh.add_hash(hashval)
                n_seqs += 1
                n_bp += int(lengths[i])
                if n_bp >= threshold:
                    _notify(args, f"... searched {n_bp} from {fi + 1} files so far")
                    while n_bp >= threshold:
                        threshold += 1e6
            n_seqs += len(recs) - last - 1
            n_bp += int(before[len(recs)] - before[last + 1])
        if not n_seqs:
            _notify(args, "ERROR: no sequences searched!?")
            raise SystemExit(-1)
        _notify(args, "DONE.")
        _notify(args, f"searched {n_seqs} sequences from {len(args.sequences)} files, containing a total of "
                      f"{format_bp(n_bp)}.")
        if seq_fp is not None:
            _notify(args, f"matched and saved a total of {n_found_seqs} sequences with {format_bp(n_bp_saved)}.")
        if kmer_w is not None:
            _notify(args, f"matched and saved a total of {n_kmers} k-mers.")
        cont = len(found) / len(query_mh)
        _notify(args, f"found {len(found)} distinct matching hashes ({cont*100:.1f}%)")
        if kmer_w is None and seq_fp is None:
            _notify(args, "NOTE: see --save-kmers or --save-sequences for output options.")
        return 0


def main(argv=None):
    parser = argparse.ArgumentParser(prog="python -m sourmash_b200.sigkmers", description=Command_B200SigKmers.description)
    cmd = Command_B200SigKmers(parser)
    return cmd.main(parser.parse_args(argv))


if __name__ == "__main__":
    sys.exit(main())
