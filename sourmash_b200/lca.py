"""`sourmash scripts b200lcaclassify | b200lcasummarize | b200lcaindex`: taxonomic classification against LCA
databases, each hash's lowest common ancestor found on the GPU, and building those databases.

The reference's `sourmash lca classify` and `lca summarize` (src/sourmash/lca/command_classify.py,
command_summarize.py) look every query hash up in every database and build a dictionary tree of its lineages to find
its LCA (gather_assignments / count_lca_for_assignments, lca/lca_utils.py:186-225): one Python tree per query hash.
Here a hash's LCA, which depends on the databases alone, is computed once per command for every database hash
(``batch.lca_table``), and a batch of queries then costs one probe per hash and one count per (query, LCA node)
(``batch.lca_counts``).  The host sees only those few rows per query and does the rest as the reference does: the
threshold and majority logic and the tree walk of classify, the aggregation up to the root of summarize.

Databases are the reference's JSON format (.lca.json, .lca.json.gz, LCA_Database.load, lca/lca_db.py:296-410); the
large "hashval_to_idx" table is parsed natively into arrays.  SQLite LCA databases (.sqldb) are refused.

    sourmash scripts b200lcaclassify --db db1.lca.json db2.lca.json.gz --query q1.sig q2.sig -o out.csv
    sourmash scripts b200lcasummarize --db db.lca.json --query metagenome.sig --ignore-abundance -o out.csv
    sourmash scripts b200lcaindex taxonomy.csv db.lca.json genomes/ -C 3 --split-identifiers --report report.txt

`lca index` (src/sourmash/lca/command_index.py) inserts every (hash, genome) pair into a dict of sets and json.dumps
it.  Here the spreadsheet and the per-signature loop run over metadata only; the kept sketches go to the device once,
where every hash's genomes are grouped in the reference's key order and the "hashval_to_idx" text is written in key
ranges of bounded size (``batch.lca_index``), spliced into what Python's json writes for the other members.  Each idx
list is ascending, where the reference writes CPython's set order (the same whenever every idx is below 8).  A
--from-file list is read in file order; the reference reads it into a set (load_pathlist_from_file,
sourmash_args.py:380-399), so with several entries its idx order follows the string hash seed.  Every input file is
parsed once, before the per-signature loop, where the reference streams them file by file: a file that fails to parse
stops the command before an error the reference would report for an earlier file (--fail-on-missing-taxonomy, a num
sketch).  -F sql and picklists are refused.

Also ``python -m sourmash_b200.lca classify|summarize|index ...``.  The command classes are not yet declared as
``sourmash.cli_script`` entry points in pyproject.toml, whose declared list the test suite pins to the six existing
commands; ``sourmash scripts ...`` finds them once they are.  Report lines, CSV columns and exit codes are the
reference's; -d/--debug is accepted but prints no debugging output.
"""
import argparse
import csv
import gzip
import json
import os
import sys
from collections import OrderedDict

import numpy as np

from . import batch as B
from .minhash import _get_max_hash_for_scaled
from .plugin import CommandLinePlugin, _expand
from .sigkmers import _error

TAXLIST = ("superkingdom", "phylum", "class", "order", "family", "genus", "species", "strain")
_SQLITE_MAGIC = b"SQLite format 3\x00"


class LcaDatabase:
    """One LCA database as arrays: ``hashes`` / ``idx`` (one pair per listed idx), ``idx_to_lid``, ``lid_to_lineage``
    (lid -> the 8 names of taxlist order, '' where a rank is empty), ``ksize`` (residues for protein moltypes),
    ``scaled``, ``moltype``, ``filename``."""

    @classmethod
    def load(cls, db_name):
        "LCA_Database.load's checks and messages, with hashval_to_idx parsed natively"
        if not os.path.isfile(db_name):
            raise ValueError(f"'{db_name}' is not a file and cannot be loaded as an LCA database")
        with open(db_name, "rb") as fh:
            head = fh.read(len(_SQLITE_MAGIC))
        if head == _SQLITE_MAGIC:
            raise ValueError(f"'{db_name}' is a SQLite LCA database; only JSON LCA databases (.lca.json, "
                             ".lca.json.gz) are supported")
        with (gzip.open if db_name.endswith(".gz") else open)(db_name, "rb") as fh:
            raw = fh.read()
        if not raw[:1] == b"{":
            raise ValueError(f"'{db_name}' is not an LCA database file.")
        from .exceptions import SourmashError
        load_d = {}
        try:
            hashes, idx, (begin, end) = B.lca_parse_hashvals(raw)
            load_d = json.loads(raw[:begin] + b"{}" + raw[end:] if begin >= 0 else raw)
        except (SourmashError, ValueError):              # the native scanner's errors, JSONDecodeError, bad UTF-8
            pass
        if not load_d:
            raise ValueError("cannot parse database file '{}' as JSON; invalid format.")
        version = db_type = None
        try:
            version = load_d.get("version")
            db_type = load_d.get("type")
        except AttributeError:
            pass
        if db_type != "sourmash_lca":
            raise ValueError(f"database file '{db_name}' is not an LCA db.")
        version = float(version)
        if version < 2.0 or "lid_to_lineage" not in load_d:
            raise ValueError("Error! This is an old-style LCA DB. You'll need to rebuild or download a newer one.")
        if begin < 0:
            raise KeyError("hashval_to_idx")
        db = cls()
        db.ksize = int(load_d["ksize"])
        db.scaled = int(load_d["scaled"])
        db.moltype = load_d.get("moltype", "DNA")
        if db.moltype != "DNA":
            assert db.ksize % 3 == 0
            db.ksize = int(db.ksize / 3)
        db.lid_to_lineage = {}
        for k, v in load_d["lid_to_lineage"].items():
            ranks = dict((x[0], x[1]) for x in v)
            db.lid_to_lineage[int(k)] = tuple(ranks.get(rank, "") or "" for rank in TAXLIST)
        db.idx_to_lid = {int(k): v for k, v in load_d["idx_to_lid"].items()}
        db.hashes, db.idx = hashes, idx
        db.filename = db_name
        return db


def load_databases(filenames, scaled=None):
    """load_databases (lca_db.py:721-760): (dbs, ksize, scaled, moltype, max_hash).  ``max_hash`` is the cut of the
    hashes of databases finer than ``scaled`` (downsample_scaled keeps hash < max_hash_for_scaled), or None."""
    ksize_vals, scaled_vals, moltype_vals = set(), set(), set()
    dbs, cut = [], None
    for db_name in filenames:
        _notify_end(f"... loading database {db_name}", "\r")
        db = LcaDatabase.load(db_name)
        ksize_vals.add(db.ksize)
        if len(ksize_vals) > 1:
            raise Exception("multiple ksizes, quitting")
        if scaled and scaled > db.scaled:
            db.scaled = scaled
            cut = _get_max_hash_for_scaled(scaled) - 1
        scaled_vals.add(db.scaled)
        moltype_vals.add(db.moltype)
        if len(moltype_vals) > 1:
            raise Exception("multiple moltypes, quitting")
        dbs.append(db)
    ksize, scaled, moltype = ksize_vals.pop(), scaled_vals.pop(), moltype_vals.pop()
    _notify_end(f"loaded {len(dbs)} LCA databases. ksize={ksize}, scaled={scaled} moltype={moltype}", "\n")
    return dbs, ksize, scaled, moltype, cut


_QUIET = [False]


def _notify_end(msg, end):
    if not _QUIET[0]:
        print("\r\033[K", end="", file=sys.stderr)
        print(msg, end=end, file=sys.stderr)


class Taxonomy:
    """One trie over the lineages of every database (build_tree, lca_utils.py:137-162): ranks with an empty name are
    skipped, equal lineages are one node, a lineage of empty names is the root (node 0).  ``parent``, ``depth``,
    ``rank`` (index into TAXLIST), ``name`` per node; ``nodes_of(db)``: the node of each of the db's (hash, idx)
    pairs, batch.LCA_NO_NODE for an idx without a lineage."""

    def __init__(self, dbs):
        self.parent, self.depth, self.rank, self.name = [0], [0], [-1], [""]
        self._child = {}
        self._node_of_lineage = {}
        self._db_nodes = []
        for db in dbs:
            lid_node = {lid: self._insert(lin) for lid, lin in db.lid_to_lineage.items()}
            n_idx = max([int(db.idx.max()) + 1 if len(db.idx) else 0] + [i + 1 for i in db.idx_to_lid])
            idx_node = np.full(max(n_idx, 1), B.LCA_NO_NODE, dtype=np.uint32)
            for i, lid in db.idx_to_lid.items():
                if lid is not None:
                    idx_node[i] = lid_node[lid]
            self._db_nodes.append(idx_node)

    def _insert(self, names):
        node = self._node_of_lineage.get(names)
        if node is not None:
            return node
        cur = 0
        for r, name in enumerate(names):
            if not name:
                continue
            key = (cur, r, name)
            nxt = self._child.get(key)
            if nxt is None:
                nxt = len(self.parent)
                self._child[key] = nxt
                self.parent.append(cur)
                self.depth.append(self.depth[cur] + 1)
                self.rank.append(r)
                self.name.append(name)
            cur = nxt
        self._node_of_lineage[names] = cur
        return cur

    def nodes_of(self, i, db):
        return self._db_nodes[i][db.idx]

    def lineage(self, node):
        "the (rank, name) pairs from the root down to node"
        out = []
        while node:
            out.append((TAXLIST[self.rank[node]], self.name[node]))
            node = self.parent[node]
        return out[::-1]


def build_table(dbs, tax, cut=None):
    "the LCA node of every distinct hash of the databases, on the device"
    hashes = np.concatenate([db.hashes for db in dbs]) if dbs else np.zeros(0, np.uint64)
    nodes = np.concatenate([tax.nodes_of(i, db) for i, db in enumerate(dbs)]) if dbs else np.zeros(0, np.uint32)
    return B.lca_table(hashes, nodes, tax.parent, tax.depth, 2**64 - 1 if cut is None else cut)


def ranked_counts(table, sset, n_queries, use_abunds):
    """per query, its [(node, count)] in Counter.most_common() order: count descending, then the order in which the
    query's ascending hashes first produced each node"""
    q, node, count, first = B.lca_counts(table, sset, weights=use_abunds)
    order = np.lexsort((first, -count.astype(np.int64), q))
    bounds = np.searchsorted(q[order], np.arange(n_queries + 1)).tolist()
    nodes, counts = node[order].tolist(), count[order].tolist()
    return [list(zip(nodes[a:b], counts[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]


def zip_lineage(lineage, truncate_empty=False):
    "zip_lineage (lca_utils.py:76-116) of (rank, name) pairs: the names in taxlist order, '' where absent"
    pairs = list(lineage) + [None] * (len(TAXLIST) - len(lineage))
    if truncate_empty:
        while pairs and pairs[-1] is None:
            pairs.pop()
    row = []
    for taxrank, pair in zip(TAXLIST, pairs):
        if pair is not None and pair[0] != taxrank:
            raise ValueError(f"incomplete lineage at {taxrank} - is {pair[0]} instead")
        row.append(pair[1] if pair is not None else "")
    return row


def classify_counts(tax, ranked, threshold, majority):
    "classify_signature's tree over the (node, count) rows of one query: (lineage pairs, status)"
    if ranked and majority:
        node, count = ranked[0]
        selected = [node] if count > threshold else []
    else:
        selected = []
        for node, count in ranked:
            if count < threshold:
                break
            selected.append(node)
    children = {}
    for node in selected:
        while node:
            children.setdefault(tax.parent[node], set()).add(node)
            node = tax.parent[node]
    if not children:
        return [], "nomatch"
    node = 0
    while len(children.get(node, ())) == 1:
        node = next(iter(children[node]))
    return tax.lineage(node), "found" if not children.get(node) else "disagree"


def summarize_counts(tax, ranked, threshold):
    "summarize's aggregated_counts over the (node, count) rows of one query: node -> count, in the reference's order"
    agg = OrderedDict()
    for node, count in ranked:
        if count < threshold:
            break
        if node == 0:
            agg[0] = agg.get(0, 0) + count
        while node:
            agg[node] = agg.get(node, 0) + count
            node = tax.parent[node]
    return agg


# ---------------------------------------------------------------------------------------------------- commands
def _check_files_exist(*files):
    missing = [f for f in files if not os.path.exists(f)]
    if missing:
        _error("Error! Could not find the following files. Make sure the file paths are specified correctly.\n{}"
               .format("\n".join(missing)))
    return not missing


def _pathlist(filename):
    "load_pathlist_from_file (sourmash_args.py:380-399); the reference returns a set, this keeps first occurrences"
    try:
        with open(filename) as fp:
            file_list = list(dict.fromkeys(x.rstrip("\r\n") for x in fp))
        if not file_list:
            raise ValueError("pathlist is empty")
        for checkfile in file_list:
            if not os.path.exists(checkfile):
                raise ValueError(f"file '{checkfile}' inside the pathlist does not exist")
    except OSError:
        raise ValueError(f"pathlist file '{filename}' does not exist")
    except UnicodeDecodeError:
        raise ValueError(f"cannot parse file '{filename}' as list of filenames")
    return file_list


def _load_queries(paths, ksize):
    """every sketch of the query files with the databases' ksize, in load order: (SignatureSet, rows, files)"""
    from .sigset import SignatureSet
    files, _ = _expand(paths)
    ss = SignatureSet.from_files(files)
    keep = np.where(ss.hash_function == 1, ss.ksize == ksize, ss.ksize == 3 * ksize)
    return ss, np.nonzero(keep)[0].astype(np.uint32), files


def _first_unscalable(ss, rows, scaled):
    "position of the first query whose downsample to ``scaled`` raises (a num sketch, or a coarser one), or None"
    qscaled = ss.python_scaled()[rows]
    bad = np.nonzero((ss.max_hash[rows] == 0) | (qscaled > np.uint64(scaled)))[0]
    return int(bad[0]) if len(bad) else None


def _query_counts(tax, table, ss, rows, scaled, use_abunds):
    """(rows, ranked counts, signatures) of the queries before the first one whose downsample raises; the signatures
    include that one, whose downsample the caller repeats to raise the reference's error after the earlier output"""
    stop = _first_unscalable(ss, rows, scaled)
    done = rows if stop is None else rows[:stop]
    ranked = []
    if len(done):
        sset = ss.to_sketchset(done, with_abunds=use_abunds).downsample(_get_max_hash_for_scaled(scaled))
        ranked = ranked_counts(table, sset, len(done), use_abunds)
    return done, ranked, ss.signatures(rows[:len(done) + (stop is not None)]) if len(rows) else []


def _common_args(p):
    p.add_argument("--db", nargs="+", action="append", help="databases to use to classify")
    p.add_argument("--query", nargs="*", default=[], action="append", help="query signatures to classify")
    p.add_argument("--query-from-file", help="file containing list of signature files to query")
    p.add_argument("--threshold", metavar="T", type=int, default=5,
                   help="minimum number of hashes needed for a taxonomic classification (default: 5)")


def _prepare(args):
    "the shared start of both commands: (dbs, ksize, scaled, taxonomy, table)"
    if not args.db:
        _error("Error! must specify at least one LCA database with --db")
        raise SystemExit(-1)
    _QUIET[0] = bool(args.quiet)
    args.db = [item for sublist in args.db for item in sublist]
    args.query = [item for sublist in args.query for item in sublist]
    if not _check_files_exist(*args.db):
        raise SystemExit(-1)
    dbs, ksize, scaled, _moltype, cut = load_databases(args.db, args.scaled)
    tax = Taxonomy(dbs)
    return dbs, ksize, scaled, tax, build_table(dbs, tax, cut)


class Command_B200LcaClassify(CommandLinePlugin):
    command = "b200lcaclassify"
    description = "classify genomes (lca classify): each hash's lowest common ancestor found on a GPU"

    def __init__(self, p):
        super().__init__(p)
        _common_args(p)
        p.add_argument("--majority", action="store_true", help="use majority vote classification instead of lca")
        p.add_argument("-o", "--output", metavar="FILE", default="-",
                       help="output CSV to the specified file; by default output to stdout")
        p.add_argument("--scaled", type=float)

    def main(self, args):
        super().main(args)
        _dbs, ksize, scaled, tax, table = _prepare(args)
        _notify_end("finding query signatures...", "\n")
        inp_files = list(args.query)
        if args.query_from_file:
            inp_files.extend(_pathlist(args.query_from_file))
        if not _check_files_exist(*inp_files):
            raise SystemExit(-1)
        if not inp_files:
            _error("Error! must specify at least one query signature with --query or --query-from-file")
            raise SystemExit(-1)
        _notify_end(f"outputting classifications to {args.output}", "\n")
        ss, rows, _files = _load_queries(inp_files, ksize)
        done, ranked, sigs = _query_counts(tax, table, ss, rows, scaled, False)
        out = sys.stdout if args.output == "-" else (
            gzip.open(args.output, "wt", newline="") if args.output.endswith(".gz") else
            open(args.output, "w", newline=""))
        try:
            w = csv.writer(out)
            w.writerow(["ID", "status"] + list(TAXLIST))
            for i in range(len(done)):
                lineage, status = classify_counts(tax, ranked[i], args.threshold, args.majority)
                w.writerow([str(sigs[i]), status] + zip_lineage(lineage))
            if len(sigs) > len(done):
                sigs[-1].minhash.downsample(scaled=scaled)            # raises the reference's error
            _notify_end(f"classified {len(rows)} signatures total", "\n")
        finally:
            if out is not sys.stdout:
                out.close()
        return 0


class Command_B200LcaSummarize(CommandLinePlugin):
    command = "b200lcasummarize"
    description = "summarize mixture (lca summarize): each hash's lowest common ancestor found on a GPU"

    def __init__(self, p):
        super().__init__(p)
        _common_args(p)
        p.add_argument("-o", "--output", metavar="FILE", help="CSV output")
        p.add_argument("--scaled", metavar="FLOAT", type=float, help="scaled value to downsample to")
        p.add_argument("--ignore-abundance", action="store_true",
                       help="ignore hash abundances in query signatures do not weight results")

    def main(self, args):
        super().main(args)
        if args.scaled:
            args.scaled = int(args.scaled)
        ignore = args.ignore_abundance
        _dbs, ksize, scaled, tax, table = _prepare(args)
        if ignore:
            _notify_end("Ignoring any k-mer abundances in query, since --ignore-abundance given.", "\n")
        _notify_end("finding query signatures...", "\n")
        inp_files = args.query
        if args.query_from_file:
            inp_files.extend(_pathlist(args.query_from_file))
        if not inp_files:
            _error("Error! must specify at least one query signature with --query")
            raise SystemExit(-1)
        if not _check_files_exist(*inp_files):
            raise SystemExit(-1)
        ss, rows, files = _load_queries(inp_files, ksize)
        done, ranked, sigs = _query_counts(tax, table, ss, rows, scaled, not ignore)
        _h, off, ab = ss.csr_host(_get_max_hash_for_scaled(scaled), with_abunds=True)
        off = off.astype(np.int64)
        sizes = np.diff(off)
        csum = np.concatenate([[0], np.cumsum(ab, dtype=np.uint64)])
        totals = csum[off[1:]] - csum[off[:-1]]
        csv_fp = open(args.output, "w", newline="") if args.output else None
        write_header = True
        try:
            for i in range(len(done)):
                r = int(done[i])
                sig, filename = sigs[i], files[int(ss.file[r])]
                if ignore and ss.has_abund[r]:
                    _notify_end("NOTE: discarding abundances in query, since --ignore-abundance", "\n")
                counts = summarize_counts(tax, ranked[i], args.threshold)
                total = float(sizes[r] if ignore else totals[r])
                md5 = sig.md5sum()
                for node, count in counts.items():
                    lineage = ";".join(zip_lineage(tax.lineage(node), truncate_empty=True)) if node else "(root)"
                    p = f"{count / total * 100.0:.1f}%"
                    if not args.quiet:
                        print(f"{p:5} {count:>5}   {lineage}   {filename}:{md5[:8]} {sig}".format(), file=sys.stdout)
                        sys.stdout.flush()
                if csv_fp:
                    w = csv.writer(csv_fp)
                    if write_header:
                        w.writerow(["count"] + list(TAXLIST) + ["filename", "sig_name", "sig_md5", "total_counts"])
                        write_header = False
                    for node, count in counts.items():
                        w.writerow([count] + zip_lineage(tax.lineage(node)) + [filename, sig.name, md5, total])
            if len(sigs) > len(done):
                if ignore and ss.has_abund[int(rows[len(done)])]:
                    _notify_end("NOTE: discarding abundances in query, since --ignore-abundance", "\n")
                sigs[-1].minhash.downsample(scaled=scaled)            # raises the reference's error
            _notify_end(f"loaded {len(rows)} signatures from {len(inp_files)} files total.", "\n")
        finally:
            if csv_fp:
                csv_fp.close()
        return 0


# ---------------------------------------------------------------------------------------------------- lca index
def filter_null(x):
    "filter_null (lca_utils.py:128-131)"
    return "unassigned" if x is None or x.strip() in ("[Blank]", "na", "null", "") else x


def load_taxonomy_assignments(filename, *, delimiter=",", start_column=2, use_headers=True, force=False,
                              split_identifiers=False, keep_identifier_versions=False):
    """load_taxonomy_assignments (lca/command_index.py:19-127): identifier -> lineage, a tuple of (rank, name, None)
    triples (LineagePair's fields, as json.dump writes them), and the number of non-empty rows"""
    fp = open(filename, newline="")
    r = csv.reader(fp, delimiter=delimiter)
    row_headers = ["identifiers"] + ["_skip_"] * (start_column - 2) + list(TAXLIST)
    if use_headers:
        _notify_end("examining spreadsheet headers...", "\n")
        first_row = next(iter(r))
        n_disagree = 0
        for column, value in zip(row_headers, first_row):
            if column == "_skip_":
                continue
            if column.lower() != value.lower():
                _notify_end(f"** assuming column '{value}' is {column} in spreadsheet", "\n")
                n_disagree += 1
                if n_disagree > 2:
                    _error("whoa, too many assumptions. are the headers right?")
                    _error("expecting {}".format(",".join(row_headers)))
                    if not force:
                        sys.exit(-1)
                    _notify_end("...continue, because --force was specified.", "\n")
    assignments = {}
    num_rows = n_species = 0
    for row in r:
        if row and row[0].strip():
            num_rows += 1
            lineage = [x for x in zip(row_headers, row) if x[0] != "_skip_"]
            ident = lineage[0][1]
            lineage = lineage[1:]
            if split_identifiers:
                ident = ident.split(" ")[0]
                if not keep_identifier_versions:
                    ident = ident.split(".")[0]
            lineage = [(a, filter_null(b), None) for (a, b) in lineage]
            while lineage and lineage[-1][1] == "unassigned":
                lineage = lineage[:-1]
            if lineage:
                if ident in assignments:
                    if assignments[ident] != tuple(lineage) and not force:
                        raise Exception(f"multiple lineages for identifier {ident}")
                else:
                    assignments[ident] = tuple(lineage)
                    if lineage[-1][0] in ("species", "strain"):
                        n_species += 1
    fp.close()
    if len(assignments) * 0.2 > n_species and len(assignments) > 50 and not force:
        _error("")
        _error("ERROR: fewer than 20% of lineages have species-level resolution!?")
        _error("({} species assignments found, of {} assignments total)".format(n_species, len(assignments)))
        _error("** If this is intentional, re-run the command with -f.")
        sys.exit(-1)
    return assignments, num_rows


def generate_report(record_duplicates, record_no_lineage, record_remnants, unused_lineages, unused_identifiers,
                    filename):
    """generate_report (lca/command_index.py:130-163).  The reference lists its sets in set iteration order, which
    varies with the string hash seed; here they are sorted."""
    with open(filename, "w") as fp:
        print(f"Duplicate signatures: {len(record_duplicates)}", file=fp)
        fp.write("\n".join(sorted(record_duplicates)))
        fp.write("\n")
        print(f"----\nUnused identifiers: {len(unused_identifiers)}", file=fp)
        fp.write("\n".join(sorted(unused_identifiers)))
        fp.write("\n")
        print(f"----\nNo lineage provided for these identifiers: {len(record_no_lineage)}", file=fp)
        fp.write("\n".join(record_no_lineage))
        fp.write("\n")
        print(f"----\nNo signatures found for these identifiers: {len(record_remnants)}", file=fp)
        fp.write("\n".join(sorted(record_remnants)))
        fp.write("\n")
        print(f"----\nUnused lineages: {len(unused_lineages)}", file=fp)
        for lineage in sorted(unused_lineages):
            fp.write(";".join(zip_lineage([p[:2] for p in lineage])))
            fp.write("\n")


def _index_files(paths, yield_all):
    """the files load_file_as_signatures reads for each argument, the argument each came from, and whether it is read
    loosely: a directory stands for its .sig / .sig.gz files, and with yield_all (-f) for every file below it, each
    skipped when it does not parse, as MultiIndex.load_from_directory(force=True) skips it (index/__init__.py:
    1033-1045).  The files are parsed once, by the caller."""
    if not yield_all:
        files, origin = _expand(paths)
        return files, origin, None
    files, origin, loose = [], [], []
    for k, p in enumerate(paths):
        if not os.path.isdir(p):
            files.append(p)
            origin.append(k)
            loose.append(False)
            continue
        for root, _dirs, names in os.walk(p):
            for name in sorted(names):
                files.append(os.path.join(root, name))
                origin.append(k)
                loose.append(True)
    return files, origin, loose


def write_database(path, ksize, scaled, moltype, lid_to_lineage, index, ident_to_name, ident_to_idx, idx_to_lid,
                   max_bytes=256 << 20):
    """save_to_json (lca_db.py:420-465): json serialises every member but "hashval_to_idx", whose text the device
    writes in key ranges of at most max_bytes, spliced in at its place; gzip (level 9) for a .gz name"""
    head = OrderedDict([("version", "2.1"), ("type", "sourmash_lca"), ("license", "CC0"),
                        ("ksize", ksize * 3 if moltype != "DNA" else ksize), ("scaled", scaled),
                        ("moltype", moltype), ("lid_to_lineage", lid_to_lineage)])
    tail = OrderedDict([("ident_to_name", ident_to_name), ("ident_to_idx", ident_to_idx),
                        ("idx_to_lid", idx_to_lid)])
    fp = gzip.open(path, "wb", compresslevel=9) if path.endswith(".gz") else open(path, "wb")
    with fp:
        fp.write(json.dumps(head)[:-1].encode("ascii") + b', "hashval_to_idx": ')
        index.write_text(fp, max_bytes)
        fp.write(b", " + json.dumps(tail)[1:].encode("ascii"))


class Command_B200LcaIndex(CommandLinePlugin):
    command = "b200lcaindex"
    description = "create LCA database (lca index): every hash's genomes grouped and the table written on a GPU"

    def __init__(self, p):
        from .sigsetops import _moltype_args
        super().__init__(p)
        p.add_argument("csv", help="taxonomy spreadsheet")
        p.add_argument("lca_db_out", help="output database name")
        p.add_argument("signatures", nargs="*",
                       help="signatures or directory of signatures to index (optional if provided via --from-file)")
        p.add_argument("--from-file", help="a text file containing a list of files to load signatures from")
        p.add_argument("--scaled", metavar="S", default=10000, type=float)
        p.add_argument("-C", "--start-column", metavar="C", default=2, type=int,
                       help="column at which taxonomic assignments start; default=2")
        p.add_argument("--tabs", action="store_true", help="input spreadsheet is tab-delimited; default is commas")
        p.add_argument("--no-headers", action="store_true", help="no headers present in taxonomy spreadsheet")
        p.add_argument("--split-identifiers", action="store_true", help="split names in signatures on whitespace")
        p.add_argument("--keep-identifier-versions", action="store_true", help="do not remove accession versions")
        p.add_argument("-f", "--force", action="store_true")
        p.add_argument("--report", help="output a report on anomalies, if any")
        p.add_argument("--require-taxonomy", action="store_true", help="ignore signatures with no taxonomy entry")
        p.add_argument("--fail-on-missing-taxonomy", action="store_true",
                       help="fail quickly if taxonomy is not available for an identifier")
        p.add_argument("-F", "--database-format", default="json", choices=["json", "sql"],
                       help="format of output database; only 'json' is supported")
        _moltype_args(p)

    def main(self, args):
        from .sigsetops import _moltype
        from .sigset import SignatureSet
        super().main(args)
        if args.start_column < 2:
            _error("error, --start-column cannot be less than 2")
            sys.exit(-1)
        _QUIET[0] = bool(args.quiet)
        args.scaled = int(args.scaled)
        if args.ksize is None:
            args.ksize = 31
        moltype = _moltype(args) or "DNA"
        if args.database_format != "json":
            _error("ERROR: SQLite LCA databases (-F sql) are not supported; write a JSON database "
                   "(.lca.json or .lca.json.gz)")
            sys.exit(-1)
        db_outfile = args.lca_db_out
        if not (db_outfile.endswith(".lca.json") or db_outfile.endswith(".lca.json.gz")):
            db_outfile += ".lca.json"
        if os.path.exists(db_outfile):
            _error(f"ERROR: output file {db_outfile} already exists. Not overwriting.")
            sys.exit(-1)
        _notify_end(f"saving to LCA DB: {format(db_outfile)}", "\n")
        _notify_end(f"Building LCA database with ksize={args.ksize} scaled={args.scaled} moltype={moltype}.", "\n")
        assignments, num_rows = load_taxonomy_assignments(
            args.csv, delimiter="\t" if args.tabs else ",", start_column=args.start_column,
            use_headers=not args.no_headers, force=args.force, split_identifiers=args.split_identifiers,
            keep_identifier_versions=args.keep_identifier_versions)
        distinct_lineages = set(assignments.values())
        _notify_end(f"{len(assignments)} distinct identities in spreadsheet out of {num_rows} rows.", "\n")
        _notify_end(f"{len(distinct_lineages)} distinct lineages in spreadsheet out of {num_rows} rows.", "\n")

        inp_files = list(args.signatures)
        if args.from_file:
            inp_files.extend(_pathlist(args.from_file))
        files, origin, loose = _index_files(inp_files, args.force)
        ss = SignatureSet.from_files(files, traverse_yield_all=args.force, loose=loose)
        code = {"DNA": 1, "protein": 2, "dayhoff": 3, "hp": 4}[moltype]
        want_k = args.ksize if moltype == "DNA" else 3 * args.ksize
        rows = np.nonzero((ss.hash_function == code) & (ss.ksize == want_k))[0]
        md5s = ss.md5sums() if len(rows) else []
        qscaled = ss.python_scaled()

        # the insert loop (command_index.py:248-329) over metadata: which rows become which idx
        md5_seen, kept = set(), []
        record_duplicates, record_no_lineage, record_remnants = set(), [], set(assignments)
        record_used_lineages, record_used_idents = set(), set()
        ident_to_name, ident_to_idx, idx_to_lid = {}, {}, {}
        lineage_to_lid, lid_to_lineage = {}, {}
        n_skipped = 0
        for r in rows.tolist():
            name, md5 = ss.name(r), md5s[r]
            if md5 in md5_seen:
                record_duplicates.add(name)
                continue
            md5_seen.add(md5)
            ident = name if name else ss.filename(r)
            orig_ident = ident
            if args.split_identifiers:
                ident = ident.split(" ")[0]
                if not args.keep_identifier_versions:
                    ident = ident.split(".")[0]
            lineage = assignments.get(ident)
            if lineage is None and args.require_taxonomy:
                if args.fail_on_missing_taxonomy:
                    _notify_end(f"ERROR: no taxonomy found for identifier '{ident}'", "\n")
                    if args.split_identifiers:
                        _notify_end(f"(Identifier extracted from name: '{orig_ident})')", "\n")
                    sys.exit(-1)
                n_skipped += 1
                continue
            shown = name or ss.filename(r) or md5[:8]                  # str(sig)
            db_ident = ident or shown                                   # insert's ident (lca_db.py:176-177)
            reason = None
            if ss.max_hash[r] == 0 or int(qscaled[r]) > args.scaled:
                reason = "cannot downsample signature; is it a scaled signature?"
            elif db_ident in ident_to_name:
                reason = f"signature '{db_ident}' is already in this LCA db."
            if reason:
                _error(f"ERROR: cannot insert signature '{shown}' (md5 {md5[:8]}, loaded from "
                       f"'{inp_files[origin[int(ss.file[r])]]}') into database.")
                _error(f"ERROR: {reason}")
                sys.exit(-1)
            ident_to_name[db_ident] = name
            idx = len(ident_to_idx)
            ident_to_idx[db_ident] = idx
            if lineage:
                lid = lineage_to_lid.setdefault(lineage, len(lineage_to_lid))
                lid_to_lineage.setdefault(lid, lineage)
                idx_to_lid[idx] = lid
                record_remnants.remove(ident)
                record_used_idents.add(ident)
                record_used_lineages.add(lineage)
            else:
                record_no_lineage.append(ident)
            kept.append(r)

        if n_skipped:
            _notify_end(f"... loaded {len(inp_files)} signatures; skipped {n_skipped} because of --require-taxonomy.",
                        "\n")
        else:
            _notify_end(f"... loaded {len(inp_files)} signatures.", "\n")
        if not inp_files:
            _error("ERROR: no signatures found. ??")
            sys.exit(1)
        index = None
        if kept:
            sset = ss.to_sketchset(np.asarray(kept, dtype=np.uint32)).downsample(_get_max_hash_for_scaled(args.scaled))
            index = B.lca_index(sset)
            del sset
        if index is None or len(index) == 0:
            _error("ERROR: no hash values found - are there any signatures?")
            sys.exit(1)
        _notify_end(f"loaded {len(index)} hashes at ksize={args.ksize} scaled={args.scaled}", "\n")
        _notify_end(f"{len(record_used_lineages)} assigned lineages out of {len(distinct_lineages)} distinct lineages "
                    "in spreadsheet.", "\n")
        unused_lineages = distinct_lineages - record_used_lineages
        _notify_end(f"{len(record_used_idents)} identifiers used out of {len(set(assignments))} distinct identifiers "
                    "in spreadsheet.", "\n")
        unused_identifiers = set(assignments) - record_used_idents

        write_database(db_outfile, args.ksize, args.scaled, moltype, lid_to_lineage, index, ident_to_name,
                       ident_to_idx, idx_to_lid)

        if record_duplicates or record_no_lineage or record_remnants or unused_lineages:
            if record_duplicates:
                _notify_end(f"WARNING: {len(record_duplicates)} duplicate signatures.", "\n")
            if record_no_lineage:
                _notify_end(f"WARNING: no lineage provided for {len(record_no_lineage)} signatures.", "\n")
            if record_remnants:
                _notify_end(f"WARNING: no signatures for {len(record_remnants)} spreadsheet rows.", "\n")
            if unused_lineages:
                _notify_end(f"WARNING: {len(unused_lineages)} unused lineages.", "\n")
            if unused_identifiers:
                _notify_end(f"WARNING: {len(unused_identifiers)} unused identifiers.", "\n")
            if args.report:
                _notify_end(f"generating a report and saving in '{args.report}'", "\n")
                generate_report(record_duplicates, record_no_lineage, record_remnants, unused_lineages,
                                unused_identifiers, args.report)
            else:
                _notify_end("(You can use --report to generate a detailed report.)", "\n")
        return 0


_COMMANDS = {"classify": Command_B200LcaClassify, "summarize": Command_B200LcaSummarize,
             "index": Command_B200LcaIndex}


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    parser = argparse.ArgumentParser(prog="python -m sourmash_b200.lca")
    sub = parser.add_subparsers(dest="op", required=True)
    cmds = {name: cls(sub.add_parser(name, description=cls.description)) for name, cls in _COMMANDS.items()}
    args = parser.parse_args(argv)
    return cmds[args.op].main(args)


if __name__ == "__main__":
    sys.exit(main())
