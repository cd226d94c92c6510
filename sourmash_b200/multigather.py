"""`sourmash scripts b200multigather`: gather many query sketches against one set of databases on a GPU.

The reference's `sourmash multigather` (commands.py:1124-1386, cli/multigather.py) loads the databases once and runs
one gather per query, each with its own prefetch and its own rounds.  Here the databases become one resident
SketchSet, loaded once, and the rounds of all queries run together on the device (gather.gather_many ->
batch.multigather).  The options and the files written follow the reference:

    sourmash scripts b200multigather --query q1.sig q2.sig --db refs/*.sig -k 31 [--output-dir out] [-U]

writes, per query, ``<base>.csv`` (the gather CSV), ``<base>.matches.sig`` (the matches in pick order) and, when there
was a match, ``<base>.unassigned.sig`` (the query hashes no match took, with the query's abundances).  ``<base>`` is
the basename of the file the query was sketched from (its md5sum when there is none; ``-U`` appends the md5sum).  As
in the reference, the databases are selected against the FIRST query, and ``--estimate-ani-ci`` is accepted but adds
no columns.  Also ``python -m sourmash_b200.multigather ...``.
"""
import argparse
import os
import sys

import numpy as np

from .plugin import CommandLinePlugin, _expand, _notify


def _error(msg):
    print(msg, file=sys.stderr)


class Command_B200Multigather(CommandLinePlugin):
    command = "b200multigather"
    description = "gather many query sketches against the same databases on a GPU (multigather)"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("--query", nargs="*", default=[], action="append", help="query signature")
        p.add_argument("--query-from-file", help="file containing list of signature files to query")
        p.add_argument("--db", nargs="+", action="append", help="database .sig / .sig.gz files, directories or .zip collections")
        p.add_argument("-k", "--ksize", type=int, default=None, help="k-mer size (as stored in the .sig)")
        p.add_argument("--moltype", choices=["DNA", "protein", "dayhoff", "hp"], default="DNA")
        p.add_argument("--scaled", type=float, default=0, help="downsample the queries to this scaled")
        p.add_argument("--threshold-bp", type=float, default=5e4, help="threshold (in bp) for reporting results")
        p.add_argument("--ignore-abundance", action="store_true", help="do NOT use k-mer abundances if present")
        p.add_argument("--estimate-ani-ci", action="store_true",
                       help="accepted like the reference's multigather, which writes no confidence intervals")
        p.add_argument("--force-allow-overwrite-output", action="store_true", help="allow output files to be overwritten")
        p.add_argument("--output-dir", "--outdir", help="write the output files to this directory")
        p.add_argument("-U", "--output-add-query-md5sum", action="store_true",
                       help="add the md5sum of each query to the output file names")
        p.add_argument("-E", "--extension", type=str, default=".sig", help="extension of the unassigned signature file")

    def main(self, args):
        super().main(args)
        from .gather import gather_many, write_gather_csv
        from .signature import load_signatures_from_json, save_signatures_to_json
        from .sigset import SignatureSet
        if not args.db:
            _error("Error! must specify at least one database with --db")
            raise SystemExit(-1)
        if not args.query and not args.query_from_file:
            _error("Error! must specify at least one query signature with --query")
            raise SystemExit(-1)
        db_args = [x for sub in args.db for x in sub]
        inp_files = [x for sub in args.query for x in sub]
        if args.query_from_file:
            with open(args.query_from_file) as fh:
                inp_files += [line.strip() for line in fh if line.strip()]
        moltype = "DNA" if args.moltype == "DNA" else args.moltype
        queries = [q for f in inp_files for q in load_signatures_from_json(f, ksize=args.ksize, select_moltype=moltype)]
        if not queries:
            raise ValueError("no query signatures loaded")
        # the databases, selected against the first query and loaded once
        first = queries[0].minhash
        files, _origin = _expand(db_args)
        db = SignatureSet.from_files(files)
        rows = db.select(ksize=first.ksize if first.is_dna else first.ksize * 3, moltype=args.moltype)
        rows = rows[db.max_hash[rows] != 0]
        rows = rows[db.seed[rows] == first.seed]
        if len(rows) == 0:
            raise ValueError("no compatible scaled signatures in the databases")
        db_scaled = max(round((2**64 - 1) / int(m)) for m in db.max_hash[rows])
        sset = db.to_sketchset(rows, scaled=db_scaled)
        where = [os.path.abspath(p) if p.endswith(".zip") else p for p in files]
        meta = dict(names=[db.name(i) for i in rows], md5s=[db.md5sum(i) for i in rows],
                    locations=[where[int(db.file[i])] for i in rows])
        # the queries that are searched, in order (skip rules of commands.py:1171-1190)
        todo = []
        for query in queries:
            if not query.minhash.scaled:
                _error("query signature needs to be created with --scaled; skipping")
                continue
            if args.scaled and int(args.scaled) != query.minhash.scaled:
                with query.update() as query:
                    query.minhash = query.minhash.downsample(scaled=int(args.scaled))
            if not len(query.minhash):
                _error("no query hashes!? skipping to next..")
                continue
            cmp_scaled = max(query.minhash.scaled, db_scaled)
            qmh = query.minhash.downsample(scaled=cmp_scaled) if cmp_scaled > query.minhash.scaled else query.minhash
            todo.append((query, qmh))
        results = gather_many([qmh for _, qmh in todo], sset, threshold_bp=args.threshold_bp,
                              ignore_abundance=args.ignore_abundance, db_scaled=db_scaled,
                              query_names=[q.name for q, _ in todo], query_filenames=[q.filename for q, _ in todo],
                              query_origs=[(len(q.minhash), q.minhash.scaled, q.md5sum()) for q, _ in todo], **meta)
        used = set()
        n = 0
        for (query, qmh), found in zip(todo, results):
            base = self._output_base(args, query, used)
            matches = db.signatures(np.asarray([rows[g.row] for g in found], dtype=rows.dtype))
            with open(base + ".matches.sig", "wb") as fp:
                save_signatures_to_json(matches, fp)
            with open(base + ".csv", "w", newline="") as fp:
                write_gather_csv(found, fp)
            _notify(args, f"found {len(found)} matches total for '{query.name}'")
            if not found:
                _notify(args, "nothing found... skipping.")
                continue
            with open(base + ".unassigned" + args.extension, "wb") as fp:
                save_signatures_to_json([self._unassigned(query, qmh, sset, [g.row for g in found],
                                                          query.minhash.track_abundance and not args.ignore_abundance)], fp)
            n += 1
        _notify(args, f"conducted gather searches on {n} signatures")
        return 0

    @staticmethod
    def _output_base(args, query, used):
        "output file name stem of a query, and the guard against two queries writing the same files (commands.py:1237-1266)"
        if not query.filename or query.filename == "-":
            base = query.md5sum()
        elif args.output_add_query_md5sum:
            base = os.path.basename(query.filename) + "." + query.md5sum()
        else:
            base = os.path.basename(query.filename)
        if args.output_dir:
            base = os.path.join(args.output_dir, base)
        if base in used:
            _error(f"ERROR: detected overwritten outputs! '{base}' has already been used. Failing.")
            if args.force_allow_overwrite_output:
                _error("continuing because --force-allow-overwrite was specified")
            else:
                _error("Consider using '-U/--output-add-query-md5sum' to build unique outputs")
                _error("and/or '--force-allow-overwrite-output'")
                raise SystemExit(-1)
        used.add(base)
        return base

    @staticmethod
    def _unassigned(query, qmh, sset, picked, is_abundance):
        """The query hashes (at the comparison's scaled) that no match took -- the reference's remaining query plus its
        noident hashes -- re-inflated with the query's abundances when they count (commands.py:1342-1355)."""
        from .batch import max_hash_for_scaled
        taken = sset.take_rows(np.asarray(picked, dtype=np.uint32)).rows()
        cut = np.uint64(max_hash_for_scaled(qmh.scaled))
        mh = qmh.flatten().to_mutable()
        for r in taken:
            mh.remove_many(r[r <= cut])
        if is_abundance:
            mh = mh.inflate(query.minhash)
        from .signature import SourmashSignature
        return SourmashSignature(mh)         # a new signature, without name or filename, as GatherDatabases leaves it


def main(argv=None):
    parser = argparse.ArgumentParser(prog="python -m sourmash_b200.multigather", description=Command_B200Multigather.description)
    cmd = Command_B200Multigather(parser)
    return cmd.main(parser.parse_args(argv))


if __name__ == "__main__":
    sys.exit(main())
