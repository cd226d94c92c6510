"""`sourmash scripts` commands backed by the GPU paths -- the reference's plugin route.

sourmash discovers command-line extensions through the ``sourmash.cli_script`` entry-point
group (sourmash/src/sourmash/plugins.py:8-12,91-186: a class with ``command``,
``description``, ``__init__(subparser)`` and ``main(args)``; the branchwater plugin uses the same
hook).  With this package installed next to sourmash (see the entry points in pyproject.toml):

    sourmash scripts b200sketch  genomes/*.fa.gz -p k=21,k=31,k=51,scaled=1000 -o all.sig
    sourmash scripts b200compare sigs/*.sig -k 31 -o cmp.npy --csv cmp.csv
    sourmash scripts b200gather  metagenome.sig refs/*.sig --threshold-bp 50000 -o gather.csv
    sourmash scripts b200prefetch metagenome.sig refs/*.sig --threshold-bp 50000 -o prefetch.csv

The classes also run without sourmash (``python -m sourmash_b200.plugin <command> ...``): the base
class falls back to a local twin of ``sourmash.plugins.CommandLinePlugin``.
Outputs follow the reference's commands: ``compare -o`` writes the numpy matrix plus
``<out>.labels.txt`` and ``--csv`` the labelled matrix (commands.py:253-292); gather / prefetch
write the reference's CSV columns (search.py:364-388,480-523).
"""
import argparse
import csv
import sys

import numpy as np

try:                                                    # pragma: no cover - depends on the host install
    from sourmash.plugins import CommandLinePlugin
except Exception:                                       # sourmash itself is optional here
    class CommandLinePlugin:
        "Local twin of sourmash.plugins.CommandLinePlugin (plugins.py:91-111): -q and -d."
        command = None
        description = None

        def __init__(self, parser):
            parser.add_argument("-q", "--quiet", action="store_true", help="suppress non-error output")
            parser.add_argument("-d", "--debug", action="store_true", help="provide debugging output")

        def main(self, args):
            pass


def _notify(args, msg):
    if not getattr(args, "quiet", False):
        print(msg, file=sys.stderr)


def parse_param_string(text):
    """'k=21,k=31,scaled=1000,abund' -> dict(ksizes, scaled, num, seed, track_abundance); the
    `-p` mini-language of `sourmash sketch` (command_sketch.py:33-87)."""
    out = {"ksizes": [], "scaled": None, "num": None, "seed": 42, "track_abundance": False}
    for item in filter(None, (t.strip() for t in text.split(","))):
        if item == "abund":
            out["track_abundance"] = True
        elif item == "noabund":
            out["track_abundance"] = False
        elif item.startswith("k="):
            out["ksizes"].append(int(item[2:]))
        elif item.startswith("scaled="):
            out["scaled"] = int(float(item[7:]))
        elif item.startswith("num="):
            out["num"] = int(item[4:])
        elif item.startswith("seed="):
            out["seed"] = int(item[5:])
        else:
            raise ValueError(f"unknown component '{item}' in params string")
    if out["scaled"] and out["num"]:
        raise ValueError("cannot set both num and scaled in a single minhash")
    return out


class Command_B200Sketch(CommandLinePlugin):
    command = "b200sketch"
    description = "sketch FASTA/FASTQ files (dna, protein or translated) on a GPU"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("filenames", nargs="+", help="FASTA / FASTQ files, plain or gzip")
        p.add_argument("-p", "--param-string", default=None, help="e.g. k=21,k=31,k=51,scaled=1000,abund")
        p.add_argument("--moltype", choices=["dna", "protein", "dayhoff", "hp"], default="dna")
        p.add_argument("--input-is-protein", action="store_true", help="records are residues (sketch protein); "
                       "default for a protein-family moltype is six-frame translation (sketch translate)")
        p.add_argument("--singleton", action="store_true", help="one signature per record")
        p.add_argument("--name-from-first", action="store_true")
        p.add_argument("--merge", "--name", dest="merge", default=None, metavar="NAME",
                       help="one signature named NAME from all records of all files")
        p.add_argument("--check-sequence", action="store_true", help="fail on invalid DNA instead of skipping")
        p.add_argument("-o", "--output", required=True, help=".sig (or .sig.gz) file for all signatures")

    def main(self, args):
        super().main(args)
        from .signature import save_signatures_to_json
        from .sketch import sketch_fasta_files
        protein = args.moltype != "dna"
        default = "k=10,scaled=200" if protein else "k=31,scaled=1000"          # command_sketch.py:25-30
        P = parse_param_string(args.param_string or default)
        if not P["ksizes"]:
            P["ksizes"] = [10] if protein else [31]
        scaled, num = P["scaled"], P["num"]
        if not scaled and not num:
            scaled = 200 if protein else 1000
        sigs = sketch_fasta_files(args.filenames, ksizes=P["ksizes"], scaled=scaled or 0, num=num or 0, seed=P["seed"],
                                  track_abundance=P["track_abundance"], singleton=args.singleton,
                                  name_from_first=args.name_from_first, check_sequence=args.check_sequence,
                                  moltype=args.moltype, input_is_protein=args.input_is_protein, merge=args.merge)
        compression = 1 if args.output.endswith(".gz") else 0
        with open(args.output, "wb") as fp:
            save_signatures_to_json(sigs, fp, compression=compression)
        _notify(args, f"saved {len(sigs)} signature(s) to '{args.output}'")
        return 0


def _select_args(p):
    p.add_argument("-k", "--ksize", type=int, default=None, help="k-mer size (as stored in the .sig)")
    p.add_argument("--moltype", choices=["DNA", "protein", "dayhoff", "hp"], default="DNA")
    p.add_argument("--scaled", type=int, default=None, help="downsample to this scaled")


class Command_B200Compare(CommandLinePlugin):
    command = "b200compare"
    description = "all-vs-all Jaccard comparison of .sig files on a GPU"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("signatures", nargs="+", help=".sig / .sig.gz files or .zip collections")
        _select_args(p)
        p.add_argument("-o", "--output", default=None, help="numpy matrix (+ <output>.labels.txt)")
        p.add_argument("--csv", default=None, help="labelled matrix as CSV")
        p.add_argument("--ignore-abundance", action="store_true", help="Jaccard also for sketches with abundances (default: angular similarity)")
        p.add_argument("--containment", action="store_true", help="containment matrix")
        p.add_argument("--max-containment", action="store_true", help="max-containment matrix")
        p.add_argument("--avg-containment", action="store_true", help="average-containment matrix")
        p.add_argument("--estimate-ani", "--ani", dest="estimate_ani", action="store_true", help="ANI estimated from the chosen measure")
        p.add_argument("--distance-matrix", action="store_true", help="1 - similarity")

    _matrix = staticmethod(lambda args: _compare_matrix(args))

    def main(self, args):
        super().main(args)
        matrix, labels = self._matrix(args)
        if args.distance_matrix:
            matrix = 1 - matrix
            _notify(args, f"max distance in matrix: {np.max(matrix):.3f}")
        else:
            _notify(args, f"min similarity in matrix: {np.min(matrix):.3f}")
        if args.output:                                                  # commands.py:253-262
            with open(args.output + ".labels.txt", "w") as fp:
                fp.write("\n".join(labels))
            with open(args.output, "wb") as fp:
                np.save(fp, matrix)
        if args.csv:                                                     # commands.py:283-292
            with open(args.csv, "w", newline="") as fp:
                w = csv.writer(fp)
                w.writerow(labels)
                for i in range(len(labels)):
                    w.writerow([str(matrix[i][j]) for j in range(len(labels))])
        return 0


def _compare_matrix(args):
    """The matrix `sourmash compare` computes for these flags (commands.py:100-214).  Flat sketches, or --ignore-abundance:
    parsed natively and compared in one pass (sigset.compare_signature_files).  Abundance sketches (angular similarity), the
    containment matrices and ANI: signature objects built in one call, brought to the coarsest scaled like there, then the
    batched functions of compare.py."""
    from . import compare as C
    from .sigset import SignatureSet, compare_signature_files
    kinds = [args.containment, args.max_containment, args.avg_containment]
    if sum(kinds) > 1:
        print("ERROR: cannot specify more than one containment argument!", file=sys.stderr)
        raise SystemExit(-1)
    files, _origin = _expand(args.signatures)
    ss = SignatureSet.from_files(files)
    rows = ss.select(ksize=args.ksize, moltype=args.moltype)
    if len(rows) == 0:
        raise ValueError("no signatures match the selection")
    is_scaled = bool((ss.max_hash[rows] != 0).all())
    if any(kinds) and not is_scaled:
        print("must use scaled signatures with --containment, --max-containment, and --avg-containment", file=sys.stderr)
        raise SystemExit(-1)
    if args.estimate_ani and not is_scaled:
        print("must use scaled signatures with --estimate-ani", file=sys.stderr)
        raise SystemExit(-1)
    keeps_abundance = bool(ss.has_abund[rows].any()) and not args.ignore_abundance
    if not (any(kinds) or args.estimate_ani or keeps_abundance):
        return compare_signature_files(files, ksize=args.ksize, moltype=args.moltype, scaled=args.scaled)
    if len(set(int(x) for x in ss.ksize[rows])) != 1:
        raise ValueError("multiple k-mer sizes loaded; please specify one with ksize")
    sigs = ss.signatures(rows)
    labels = [str(x) for x in sigs]
    if is_scaled:
        coarsest = max([int(x.minhash.scaled) for x in sigs] + [int(args.scaled or 0)])
        down = []
        for x in sigs:
            if x.minhash.scaled != coarsest:
                with x.update() as x:
                    x.minhash = x.minhash.downsample(scaled=coarsest)
            down.append(x)
        sigs = down
    if args.containment:
        return C.compare_serial_containment(sigs, return_ani=args.estimate_ani), labels
    if args.max_containment:
        return C.compare_serial_max_containment(sigs, return_ani=args.estimate_ani), labels
    if args.avg_containment:
        return C.compare_serial_avg_containment(sigs, return_ani=args.estimate_ani), labels
    return C.compare_all_pairs(sigs, args.ignore_abundance, return_ani=args.estimate_ani), labels


def _expand(paths):
    """Files behind the arguments, and the argument each came from: a directory stands for the .sig / .sig.gz files below it, in
    the reference's traversal order (traverse_find_sigs, sourmash_args.py:275-295) -- one database, many locations."""
    import os
    files, origin = [], []
    for k, p in enumerate(paths):
        if os.path.isdir(p):
            for root, _dirs, names in os.walk(p):
                for name in sorted(names):
                    if name.endswith((".sig", ".sig.gz")):
                        files.append(os.path.join(root, name))
                        origin.append(k)
        else:
            files.append(p)
            origin.append(k)
    return files, origin


def _load_query_and_db(args):
    from .signature import load_signatures_from_json
    from .sigset import SignatureSet
    moltype = None if args.moltype == "DNA" else args.moltype
    queries = list(load_signatures_from_json(args.query, ksize=args.ksize, select_moltype=moltype or "DNA"))
    if len(queries) != 1:
        raise ValueError(f"need exactly one query sketch in '{args.query}' (found {len(queries)}); select with -k")
    query = queries[0]
    given_mh = query.minhash
    if args.scaled and int(args.scaled) > query.minhash.scaled:        # --scaled: the query itself is downsampled first, and that
        with query.update() as query:                                  # sketch is "the query" of the reports (commands.py: gather)
            query.minhash = query.minhash.downsample(scaled=int(args.scaled))
    files, origin = _expand(args.databases)
    db = SignatureSet.from_files(files)
    rows = db.select(ksize=query.minhash.ksize if query.minhash.is_dna else query.minhash.ksize * 3,
                     moltype=args.moltype)
    rows = rows[db.max_hash[rows] != 0]
    rows = rows[db.seed[rows] == query.minhash.seed]      # check_compatible: ksize, molecule AND seed (minhash.rs:886-912)
    if len(rows) == 0:
        raise ValueError("no compatible scaled signatures in the databases")
    scaled = max(int(args.scaled or 0), query.minhash.scaled,
                 max(round((2**64 - 1) / int(m)) for m in db.max_hash[rows]))
    qmh = query.minhash.downsample(scaled=scaled) if scaled > query.minhash.scaled else query.minhash
    sset = db.to_sketchset(rows, scaled=scaled)
    meta = dict(names=[db.name(i) for i in rows], md5s=[db.md5sum(i) for i in rows],
                filenames=[db.filename(i) for i in rows], query_name=query.name, query_filename=query.filename)
    # where each row was loaded from: the `filename` column of the reference's search / gather CSVs (the match's location)
    import os
    where = [os.path.abspath(p) if p.endswith(".zip") else p for p in files]               # a zip collection reports its absolute path
    meta["locations"] = [where[int(db.file[i])] for i in rows]
    meta["groups"] = [origin[int(db.file[i])] for i in rows]                                # the database (argument) of every row
    # the sketches as given: the reports quote their sizes and the query's md5, the comparisons run at `scaled`
    meta["query_orig"] = (len(query.minhash), query.minhash.scaled, query.md5sum())
    meta["match_orig"] = (db.n_mins[rows].astype(np.int64), db.python_scaled()[rows].astype(np.int64))
    # what the signature outputs need: the database rows as loaded, the query after --scaled and as given
    src = _Loaded(db, rows, query, given_mh)
    return qmh, sset, meta, src


class _Loaded:
    "The loaded side of a search: row r of the compared set is signature ``rows[r]`` of ``db``."
    def __init__(self, db, rows, query, given_mh):
        self.db, self.rows, self.query, self.given_mh = db, rows, query, given_mh

    def signatures(self, rows):
        "the signatures behind rows of the compared set, as loaded (not downsampled), in the given order"
        return self.db.signatures(self.rows[np.asarray(rows, dtype=np.int64)]) if len(rows) else []


_COLLECTION_TARGETS = ((".zip", "a .zip collection"), (".sqldb", "a SQLite database"), ("/", "a directory"))


def _check_sig_targets(*targets):
    """Signature outputs go to a .sig file (gzip JSON for a path ending in .gz) or to stdout for ``-``, as the reference's
    SaveSignatures_SigFile writes them (save_load.py:406-445); collections are refused before anything is loaded."""
    for t in targets:
        for suffix, what in _COLLECTION_TARGETS:
            if t and t.endswith(suffix):
                print(f"ERROR: cannot save signatures to {what} ('{t}'); write a .sig or .sig.gz file, or - for stdout",
                      file=sys.stderr)
                raise SystemExit(-1)


def _save_sigs(path, sigs):
    from .signature import save_signatures_to_json
    if path == "-":
        save_signatures_to_json(sigs, sys.stdout)
        sys.stdout.flush()
        return
    gz = path.endswith(".gz")
    with open(path, "wb" if gz else "w", encoding=None if gz else "utf-8") as fp:
        save_signatures_to_json(sigs, fp, compression=1 if gz else 0)


def _sketch_of(template, hashes, abund_from=None):
    """A sketch with ``template``'s parameters holding ``hashes`` (sorted, unique).  With ``abund_from`` (a sketch with
    abundances that holds every hash): ``flat.inflate(abund_from)`` -- the abundances taken from it, and its max_hash
    kept, because the reference's inflate discards its own downsample (minhash.py:1071-1087) -- built from arrays."""
    from ._ffi import rustcall
    from ._lowlevel import ffi, lib
    hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
    if abund_from is None:
        mh = template._blank_like(track_abundance=False)
        mh.add_many(hashes)
        return mh
    mh = abund_from._blank_like()
    src = abund_from._mins_array()
    abunds = np.ascontiguousarray(abund_from._abunds_array()[np.searchsorted(src, hashes)], dtype=np.uint64)
    rustcall(lib.kmerminhash_set_abundances, mh._get_objptr(), ffi.cast("uint64_t *", hashes.ctypes.data),
             ffi.cast("uint64_t *", abunds.ctypes.data), len(hashes), True)
    return mh


class Command_B200Gather(CommandLinePlugin):
    command = "b200gather"
    description = "min-set-cover of a query sketch by database sketches on a GPU (gather CSV)"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("query", help="query .sig")
        p.add_argument("databases", nargs="+", help="database .sig / .sig.gz files or .zip collections")
        _select_args(p)
        p.add_argument("--threshold-bp", type=float, default=50000.0)
        p.add_argument("--ignore-abundance", action="store_true")
        p.add_argument("--estimate-ani-ci", action="store_true")
        p.add_argument("-o", "--output", default=None, help="CSV of the matches")
        p.add_argument("--save-matches", default=None, help="save the picked signatures (.sig, .sig.gz or -)")
        p.add_argument("--save-prefetch", default=None, help="save the signatures of the prefetch stage")
        p.add_argument("--save-prefetch-csv", default=None, help="prefetch CSV of the prefetch stage")
        p.add_argument("--output-unassigned", default=None, help="save the query hashes no match took")

    def main(self, args):
        super().main(args)
        from .gather import gather_databases, write_gather_csv
        _check_sig_targets(args.save_matches, args.save_prefetch, args.output_unassigned)
        qmh, sset, meta, src = _load_query_and_db(args)
        match_orig = meta.pop("match_orig")
        groups = meta.pop("groups")
        stats = {}
        rows = gather_databases(qmh, sset, threshold_bp=args.threshold_bp, ignore_abundance=args.ignore_abundance,
                                estimate_ani_ci=args.estimate_ani_ci, stats=stats, **meta)
        if args.save_prefetch or args.save_prefetch_csv:
            self._save_prefetch(args, qmh, sset, meta, match_orig, groups, stats, src)
        if args.save_matches:                               # the picks, in pick order (commands.py:1043-1045)
            _notify(args, f"saving all matches to '{args.save_matches}'")
        for g in rows:
            _notify(args, f"{g.intersect_bp / 1e3:9.1f} kbp {g.f_orig_query * 100:6.1f}% {g.f_match * 100:6.1f}%  {g.name}")
        if args.save_matches and rows:                      # nothing picked: the reference's empty saver writes no file
            # the counter of a database holds the last of the signatures that share an md5 (index/__init__.py:777-794)
            last = {}
            for r in self._passing(stats).tolist():
                last[(groups[r], meta["md5s"][r])] = r
            _save_sigs(args.save_matches, src.signatures([last.get((groups[g.row], meta["md5s"][g.row]), g.row)
                                                          for g in rows]))
        _notify(args, f"found {len(rows)} matches total")
        if args.output and rows:                            # no matches: the reference leaves without creating the file
            with open(args.output, "w", newline="") as fp:
                write_gather_csv(rows, fp, estimate_ani_ci=args.estimate_ani_ci)
        if args.output_unassigned:
            self._save_unassigned(args, qmh, sset, rows, stats, src)
        return 0

    @staticmethod
    def _passing(stats):
        "rows of the compared set at or above the prefetch threshold (none when the threshold is unattainable)"
        if stats["counts0"] is None:                        # no database yields a counter (commands.py:909-914)
            return np.zeros(0, dtype=np.int64)
        return np.nonzero(stats["counts0"].astype(np.int64) >= max(1, stats["min_count"]))[0]

    @classmethod
    def _prefetch_rows(cls, groups, md5s, stats):
        """Rows of the prefetch stage as the reference's save_prefetch holds them (commands.py:894-922): database argument
        after argument, and inside one the rows at or above the threshold collapsed by md5 -- CounterGather.add keys a
        dict by md5, so the entry keeps the first duplicate's place and the last one's signature (index/__init__.py:777-794)."""
        by_group = {}
        for r in cls._passing(stats).tolist():
            by_group.setdefault(groups[r], {})[md5s[r]] = r
        return [r for k in sorted(by_group) for r in by_group[k].values()]

    def _save_prefetch(self, args, qmh, sset, meta, match_orig, groups, stats, src):
        from .gather import prefetch_database, write_prefetch_csv
        rows = self._prefetch_rows(groups, meta["md5s"], stats)
        if args.save_prefetch:
            _save_sigs(args.save_prefetch, src.signatures(rows))
        if args.save_prefetch_csv:
            res = []
            if rows:                                        # PrefetchResult of the flattened query (commands.py:924-934)
                pm = {k: v for k, v in meta.items() if k != "locations"}
                flat = qmh.flatten() if qmh.track_abundance else qmh
                by_row = {d["row"]: d for d in prefetch_database(flat, sset, args.threshold_bp, counts=stats["counts0"],
                                                                 estimate_ani_ci=args.estimate_ani_ci,
                                                                 match_orig=match_orig, **pm)}
                res = [by_row[r] for r in rows]
            with open(args.save_prefetch_csv, "w", newline="") as fp:
                write_prefetch_csv(res, fp, estimate_ani_ci=args.estimate_ani_ci)

    @classmethod
    def _save_unassigned(cls, args, qmh, sset, rows, stats, src):
        """The query hashes that no pick took: the remaining query plus the prefetch's noident hashes
        (commands.py:1094-1112), named as GatherDatabases names its query (search.py:826-827,918-920).  Without a pick
        that is the whole query at its own scaled (after --scaled).  After a pick the remaining query is at the comparison
        scaled and noident at the query's; when a database coarser than the query makes these differ, the reference's
        `remaining_mh += noident_mh` fails on the two scaled values, and so does this (an empty noident is not merged)."""
        from . import batch as B
        from .signature import SourmashSignature
        noident = np.zeros(0, dtype=np.uint64)
        if rows:
            q, left = stats["q_hashes"], stats["q_hashes"][stats["alive"]]
            if qmh.scaled != src.query.minhash.scaled:
                full = src.query.minhash._mins_array()       # q is its prefix: the hashes <= the comparison's max_hash
                held = B.query_covered(q, sset, cls._passing(stats))
                noident = np.concatenate([q[~held], full[len(q):]])
        else:
            left = src.query.minhash._mins_array()
        if not len(left) and not len(noident):
            _notify(args, "no unassigned hashes to save with --output-unassigned!")
            return
        _notify(args, f"saving unassigned hashes to '{args.output_unassigned}'")
        if len(noident):                                    # two max_hash values: merge raises, as in the reference
            _sketch_of(qmh, left).merge(_sketch_of(src.query.minhash, noident))
        abund = qmh.track_abundance and not args.ignore_abundance
        mh = _sketch_of(qmh if rows else src.query.minhash, left, abund_from=src.query.minhash if abund else None)
        if rows:
            sig = SourmashSignature(mh)
        else:
            sig = SourmashSignature(mh, name=src.query.name or "", filename=src.query.filename or "")
        _save_sigs(args.output_unassigned, [sig])


class Command_B200Prefetch(CommandLinePlugin):
    command = "b200prefetch"
    description = "all database sketches overlapping a query by a threshold, on a GPU (prefetch CSV)"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("query", help="query .sig")
        p.add_argument("databases", nargs="+", help="database .sig / .sig.gz files or .zip collections")
        _select_args(p)
        p.add_argument("--threshold-bp", type=float, default=50000.0)
        p.add_argument("--estimate-ani-ci", action="store_true")
        p.add_argument("-o", "--output", default=None, help="CSV of the matches")
        p.add_argument("--save-matches", default=None, help="save the matching database signatures (.sig, .sig.gz or -)")
        p.add_argument("--save-matching-hashes", default=None, help="save the query hashes found in the matches")
        p.add_argument("--save-unmatched-hashes", default=None, help="save the query hashes no match holds")

    def main(self, args):
        super().main(args)
        from .gather import prefetch_database, write_prefetch_csv
        _check_sig_targets(args.save_matches, args.save_matching_hashes, args.save_unmatched_hashes)
        if args.output:
            open(args.output, "w").close()                  # created before the search, as in the reference (empty if it fails)
        qmh, sset, meta, src = _load_query_and_db(args)
        meta.pop("locations")                              # prefetch reports the filename stored in the match (match_filename)
        meta.pop("groups")
        if qmh.track_abundance:                             # prefetch works on the flattened query (commands.py: prefetch)
            qmh = qmh.flatten()
        if args.save_matches:
            _notify(args, f"saving all matching database signatures to '{args.save_matches}'")
        res = prefetch_database(qmh, sset, args.threshold_bp, estimate_ani_ci=args.estimate_ani_ci, **meta)
        _notify(args, f"total of {len(res)} matching signatures")
        if args.save_matches:                               # every match as loaded, in CSV order (commands.py:1631)
            _save_sigs(args.save_matches, src.signatures([d["row"] for d in res]))
        if args.output:
            with open(args.output, "w", newline="") as fp:
                write_prefetch_csv(res, fp, estimate_ani_ci=args.estimate_ani_ci)
        if args.save_matching_hashes or args.save_unmatched_hashes:
            self._save_hashes(args, qmh, sset, [d["row"] for d in res], src)
        return 0

    @staticmethod
    def _save_hashes(args, qmh, sset, rows, src):
        """The query hashes the matches hold ("known") and the rest ("unknown"), the reference's ident_mh / noident_mh
        (commands.py:1602-1622,1674-1712): the flattened query at the comparison's scaled, split by one device pass over
        the matches; with no match, at the query's own scaled (after --scaled), all of it unknown."""
        from . import batch as B
        from .signature import SourmashSignature
        if rows:
            template = qmh
            q = qmh._mins_array()
            covered = B.query_covered(q, sset, rows)
        else:
            template = src.query.minhash.flatten()
            q = template._mins_array()
            covered = np.zeros(len(q), dtype=bool)
        given = src.given_mh if src.given_mh.track_abundance else None
        name = src.query.name
        for path, mask, tag, what in ((args.save_matching_hashes, covered, "known", "matched"),
                                      (args.save_unmatched_hashes, ~covered, "unknown", "unmatched")):
            if not path:
                continue
            hashes = q[mask]
            _notify(args, f"saving {len(hashes)} {what} hashes to '{path}'")
            mh = _sketch_of(template, hashes, abund_from=given)
            _save_sigs(path, [SourmashSignature(mh, name=f"{name}-{tag}" if name else "")])


class Command_B200Search(CommandLinePlugin):
    command = "b200search"
    description = "search a query sketch against database sketches on a GPU (search CSV)"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("query", help="query .sig")
        p.add_argument("databases", nargs="+", help="database .sig / .sig.gz files or .zip collections")
        _select_args(p)
        p.add_argument("-t", "--threshold", type=float, default=0.08, help="minimum score to report (default 0.08)")
        p.add_argument("--containment", action="store_true", help="score by containment of the query")
        p.add_argument("--max-containment", action="store_true", help="score by max containment")
        p.add_argument("--best-only", action="store_true", help="report only the best match")
        p.add_argument("--ignore-abundance", action="store_true", help="search an abundance query by its hashes only")
        p.add_argument("-n", "--num-results", type=int, default=3, help="matches to print (0: all; the CSV has all)")
        p.add_argument("--estimate-ani-ci", action="store_true")
        p.add_argument("-o", "--output", default=None, help="CSV of the matches")
        p.add_argument("--save-matches", default=None, help="save the signature of every match (.sig, .sig.gz or -)")

    def main(self, args):
        super().main(args)
        from .gather import write_search_csv
        if args.containment and args.max_containment:
            raise ValueError("--containment and --max-containment are mutually exclusive")
        _check_sig_targets(args.save_matches)
        res = self._abundance_search(args)                 # None: a flat query, or --ignore-abundance
        if res is None:
            res = self._flat_search(args)
        _notify(args, f"{len(res)} matches above threshold {args.threshold:0.3f}")
        shown = res if not args.num_results else res[:args.num_results]
        if args.best_only:                                         # commands.py: --best-only prints one match; the CSV has all
            shown = res[:1]
        for d in shown:
            _notify(args, f"{d['similarity'] * 100:6.1f}%       {d.get('name') or d.get('md5', '')}")
        if args.output:
            with open(args.output, "w", newline="") as fp:
                write_search_csv(res, fp, estimate_ani_ci=args.estimate_ani_ci)
        if args.save_matches:                                      # every result row's match, in CSV order (commands.py:737-743)
            _notify(args, f"saving all matched signatures to \"{args.save_matches}\"")
            _save_sigs(args.save_matches, [d["match"] for d in res])
        return 0

    @staticmethod
    def _abundance_search(args):
        """A query with abundances, kept: angular similarity against subjects with abundances, database by database, one entry
        per md5, best first (commands.py:652-684 -> search_databases_with_abund_query, search.py:723-748 -> Index.search_abund);
        containment searches and flat subjects are errors there, and here."""
        from .index import load_file_as_index
        from .signature import load_signatures_from_json
        moltype = None if args.moltype == "DNA" else args.moltype
        queries = list(load_signatures_from_json(args.query, ksize=args.ksize, select_moltype=moltype or "DNA"))
        if len(queries) != 1 or not queries[0].minhash.track_abundance or args.ignore_abundance:
            return None
        query = queries[0]
        if args.containment or args.max_containment:
            print("ERROR: cannot do containment searches on an abund signature; maybe specify --ignore-abundance?", file=sys.stderr)
            raise SystemExit(-1)
        ksize = query.minhash.ksize
        found, seen = [], set()
        try:
            for path in args.databases:
                db = load_file_as_index(path).select(ksize=ksize, moltype=args.moltype)
                for score, match, location in db.search_abund(query, threshold=args.threshold):
                    if match.md5sum() not in seen:
                        seen.add(match.md5sum())
                        found.append((score, match, location))
        except TypeError as exc:
            print(f"ERROR: {exc}", file=sys.stderr)
            raise SystemExit(-1)
        found.sort(key=lambda x: -x[0])
        return [{"similarity": score, "md5": match.md5sum(), "filename": location, "name": match.name,
                 "query_filename": query.filename, "query_name": query.name, "query_md5": query.md5sum()[:8], "ani": None,
                 "match": match}
                for score, match, location in found]

    @staticmethod
    def _flat_search(args):
        from .gather import search_database
        qmh, sset, meta, src = _load_query_and_db(args)
        meta.pop("match_orig")
        res = search_database(qmh.flatten() if qmh.track_abundance else qmh, sset, threshold=args.threshold,
                              do_containment=args.containment, do_max_containment=args.max_containment,
                              best_only=args.best_only, estimate_ani_ci=args.estimate_ani_ci, **meta)   # `groups`: one database per argument
        if args.save_matches:
            for d, match in zip(res, src.signatures([d["row"] for d in res])):
                d["match"] = match
        return res


COMMANDS = [Command_B200Sketch, Command_B200Compare, Command_B200Search, Command_B200Gather, Command_B200Prefetch]


def build_parser():
    "Stand-alone equivalent of `sourmash scripts` (plugins.py:160-186 add_cli_scripts)."
    parser = argparse.ArgumentParser(prog="python -m sourmash_b200.plugin")
    sub = parser.add_subparsers(dest="cmd", required=True)
    objs = {}
    for cls in COMMANDS:
        sp = sub.add_parser(cls.command, description=cls.description)
        objs[cls.command] = cls(sp)
    return parser, objs


def main(argv=None):
    parser, objs = build_parser()
    args = parser.parse_args(argv)
    return objs[args.cmd].main(args)


if __name__ == "__main__":
    sys.exit(main())
