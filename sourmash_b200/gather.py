"""`sourmash gather` with its full per-match report, driven by the GPU gather session.

The reference (src/sourmash/search.py:763-949) runs one Python round per match: pick the best
counter, intersect, subtract, rebuild MinHash objects, and build a ``GatherResult``
(search.py:471-655) whose columns come from two ``FracMinHashComparison`` objects
(sketchcomparison.py:99-256).  Here the database, the query and the counters stay in HBM
(``batch.GatherSession``); each round returns the winning row and the hashes it newly covers,
and every report column is evaluated from those integers with the reference's own float
formulas (Python floats, same operation order).  Abundance-weighted columns (f_unique_weighted,
average / median / std abundance; search.py:596-620) use the query's abundances of exactly those
hashes, in ascending hash order like ``MinHash.hashes``.
"""
from dataclasses import dataclass

import math

import numpy as np

from . import batch as B
from . import distance_utils as DU
from .search import calc_threshold_from_bp

GATHER_COLUMNS = [  # search.py:480-513
    "intersect_bp", "f_orig_query", "f_match", "f_unique_to_query", "f_unique_weighted", "average_abund",
    "median_abund", "std_abund", "filename", "name", "md5", "f_match_orig", "unique_intersect_bp",
    "gather_result_rank", "remaining_bp", "query_filename", "query_name", "query_md5", "query_bp", "ksize",
    "moltype", "scaled", "query_n_hashes", "query_abundance", "query_containment_ani", "match_containment_ani",
    "average_containment_ani", "max_containment_ani", "potential_false_negative", "n_unique_weighted_found",
    "sum_weighted_found", "total_weighted_hashes"]
CI_COLUMNS = ["query_containment_ani_low", "query_containment_ani_high", "match_containment_ani_low",
              "match_containment_ani_high"]


@dataclass
class GatherRow:
    "One gather match; attribute names are the reference's CSV columns."
    row: int                       # row of the database SketchSet
    intersect_bp: int = 0
    f_orig_query: float = 0.0
    f_match: float = 0.0
    f_unique_to_query: float = 0.0
    f_unique_weighted: float = 0.0
    average_abund: float = None
    median_abund: float = None
    std_abund: float = None
    filename: str = None
    name: str = None
    md5: str = None
    f_match_orig: float = 0.0
    unique_intersect_bp: int = 0
    gather_result_rank: int = 0
    remaining_bp: int = 0
    query_filename: str = None
    query_name: str = None
    query_md5: str = None
    query_bp: int = 0
    ksize: int = 0
    moltype: str = "DNA"
    scaled: int = 0
    query_n_hashes: int = 0
    query_abundance: bool = False
    query_containment_ani: float = None
    match_containment_ani: float = None
    average_containment_ani: float = None
    max_containment_ani: float = None
    potential_false_negative: bool = False
    n_unique_weighted_found: int = None
    sum_weighted_found: int = 0
    total_weighted_hashes: int = 0
    query_containment_ani_low: float = None
    query_containment_ani_high: float = None
    match_containment_ani_low: float = None
    match_containment_ani_high: float = None

    def to_dict(self, estimate_ani_ci=False):
        cols = GATHER_COLUMNS + (CI_COLUMNS if estimate_ani_ci else [])
        return {c: getattr(self, c) for c in cols if getattr(self, c) is not None}


def _contained_by(common, size, scaled):
    "MinHash.contained_by from counts (minhash.py:819-841): bias-corrected, clamped to [0, 1]."
    if size == 0:
        return 0
    bias = 1.0 - (1.0 - 1.0 / scaled) ** float(size * scaled)
    c = common / (size * bias)
    return 1.0 if c >= 1 else 0.0 if c <= 0 else c


def _size_ok(n, scaled, cache):
    key = (n, scaled)
    if key not in cache:
        cache[key] = bool(DU.set_size_exact_prob(n * scaled, scaled, relative_error=0.20) >= 0.95)
    return cache[key]


@dataclass
class _GatherQuery:
    "One query of a gather, prepared the way GatherDatabases.__init__ prepares it (search.py:803-818)."
    mh: object
    q_hashes: np.ndarray               # the query that is searched (noident hashes taken out), ascending
    q_abunds: np.ndarray               # their abundances (ones when abundance is not tracked)
    track: bool
    noident_len: int
    noident_weight: int
    orig_len: int                      # orig_query_len, search.py:912
    total_weighted: int
    query_md5: str
    query_bp_scaled: int
    min_count: int                     # least overlap of a row that takes part at all
    query_name: str
    query_filename: str
    q_size_ok: bool
    cache: dict


def _prepare_query(query_mh, *, threshold_bp, ignore_abundance, noident_hashes, query_orig, query_name,
                   query_filename):
    """The searched query of a gather and everything its report columns need; None when no round can run (empty query,
    or a threshold the query as given cannot reach)."""
    if not query_mh.scaled:
        raise TypeError("query signature must be calculated with scaled")
    scaled = query_mh.scaled
    q_hashes = query_mh._mins_array()
    track = bool(query_mh.track_abundance) and not ignore_abundance
    q_abunds = query_mh._abunds_array() if track else np.ones(len(q_hashes), dtype=np.uint64)
    noident_len = noident_weight = 0
    if noident_hashes is not None and len(noident_hashes):
        noident = np.unique(np.asarray(noident_hashes, dtype=np.uint64))
        noident = noident[noident <= np.uint64(B.max_hash_for_scaled(scaled))]      # noident_mh.downsample(scaled)
        gone = np.isin(q_hashes, noident)
        noident_len = len(noident)
        # abundances come from the query; a noident hash that is not in the query has none (KeyError there)
        if int(gone.sum()) != noident_len:
            raise KeyError("noident hashes must be part of the query")
        noident_weight = int(q_abunds[gone].sum(dtype=object)) if track else noident_len
        q_hashes, q_abunds = q_hashes[~gone], q_abunds[~gone]
    search_len = len(q_hashes)
    if search_len == 0:
        return None
    orig_len = search_len + noident_len
    total_weighted = (int(q_abunds.sum(dtype=object)) if track else search_len) + noident_weight
    # query_orig = (number of hashes, scaled, md5sum) of the query AS GIVEN, when ``query_mh`` is a downsampled copy of it: the
    # reference reports the given query's md5 and multiplies the hash count (at the comparison's scaled) by the GIVEN scaled
    # for query_bp (GatherResult.build_gather_result, search.py:553-561; BaseResult.get_cmpinfo, :222-243)
    query_md5 = (query_orig[2] if query_orig else query_mh.md5sum())[:8]
    query_bp_scaled = int(query_orig[1]) if query_orig else scaled
    # which rows enter the rounds at all: the reference fills its counters by a prefetch of the query as given
    # (commands.py:906-911 -> CounterGather via Index.counter_gather); later rounds only ask count >= n_threshold_hashes
    min_count = 1
    if query_orig is not None and threshold_bp:
        try:                                                   # unattainable for the query as given: no database yields a counter
            calc_threshold_from_bp(threshold_bp, int(query_orig[1]), int(query_orig[0]))      # (commands.py:909-914)
        except ValueError:
            return None
        min_count = _min_count_of_given_query(threshold_bp, query_orig, orig_len)
    cache = {}
    return _GatherQuery(query_mh, q_hashes, q_abunds, track, noident_len, noident_weight, orig_len, total_weighted,
                        query_md5, query_bp_scaled, min_count, query_name, query_filename, _size_ok(orig_len, scaled, cache),
                        cache)


def _gather_row(p, r, rank, ab, remaining, left_weight, c0, m, *, estimate_ani_ci, names, md5s, filenames, locations):
    """The GatherResult columns of round ``rank`` (search.py:548-620): row ``r`` (``m`` hashes, ``c0`` shared with the
    searched query) took the hashes whose abundances are ``ab`` (ascending hash order) from ``remaining`` live hashes;
    ``left_weight`` is the weight of the live hashes after the round.  Python floats, the reference's operation order."""
    mh = p.mh
    scaled, ksize = mh.scaled, mh.ksize
    u = len(ab)
    g = GatherRow(row=int(r), gather_result_rank=rank, ksize=ksize, moltype=mh.moltype,
                  scaled=scaled, query_name=p.query_name, query_filename=p.query_filename, query_md5=p.query_md5,
                  query_bp=p.orig_len * p.query_bp_scaled, query_n_hashes=p.orig_len, total_weighted_hashes=p.total_weighted)
    g.name = names[r] if names is not None else None
    g.md5 = md5s[r] if md5s is not None else None
    # the location the match was loaded from wins, else the filename stored in the match (search.py:230-235)
    g.filename = locations[r] if locations is not None else (filenames[r] if filenames is not None else None)
    g.intersect_bp = c0 * scaled
    g.unique_intersect_bp = u * scaled
    g.f_orig_query = c0 / p.orig_len
    g.f_unique_to_query = u / p.orig_len
    g.f_match_orig = _contained_by(c0, m, scaled)              # match.contained_by(original query)
    g.f_match = _contained_by(u, m, scaled)                    # match.contained_by(remaining query)
    g.remaining_bp = (p.noident_len + remaining - u) * scaled
    if p.track:
        g.query_abundance = True
        g.n_unique_weighted_found = int(ab.sum(dtype=object))
        g.f_unique_weighted = g.n_unique_weighted_found / p.total_weighted
        vals = ab.tolist()
        g.average_abund, g.median_abund, g.std_abund = np.mean(vals), np.median(vals), np.std(vals)
    else:
        g.f_unique_weighted = g.f_unique_to_query
    g.sum_weighted_found = p.total_weighted - p.noident_weight - left_weight
    # ANI columns: FracMinHashComparison(original query, match) (search.py:389-420, sketchcomparison.py:162-236)
    ok = p.q_size_ok and _size_ok(m, scaled, p.cache)
    qc = DU.containment_to_distance(_contained_by(c0, p.orig_len, scaled), ksize, scaled,
                                    n_unique_kmers=p.orig_len * scaled, estimate_ci=estimate_ani_ci)
    mc = DU.containment_to_distance(g.f_match_orig, ksize, scaled, n_unique_kmers=m * scaled,
                                    estimate_ci=estimate_ani_ci)
    qc.size_is_inaccurate = mc.size_is_inaccurate = not ok
    g.query_containment_ani, g.match_containment_ani = qc.ani, mc.ani
    g.potential_false_negative = bool(qc.p_exceeds_threshold or mc.p_exceeds_threshold)
    if estimate_ani_ci:
        g.query_containment_ani_low, g.query_containment_ani_high = qc.ani_low, qc.ani_high
        g.match_containment_ani_low, g.match_containment_ani_high = mc.ani_low, mc.ani_high
    if qc.ani is not None and mc.ani is not None:
        g.average_containment_ani = (qc.ani + mc.ani) / 2
        g.max_containment_ani = max(qc.ani, mc.ani)
    return g


def gather_databases(query_mh, db, *, threshold_bp=0, ignore_abundance=False, estimate_ani_ci=False,
                     names=None, md5s=None, filenames=None, query_name="", query_filename="", max_rounds=None,
                     noident_hashes=None, locations=None, query_orig=None, stats=None):
    """Min-set-cover of ``query_mh`` by the rows of the GPU-resident SketchSet ``db`` (same ksize,
    seed and scaled as the query; use ``SketchSet.downsample`` / ``SignatureSet.to_sketchset``).
    Returns the list of GatherRow in pick order -- the reference's GatherDatabases loop with the
    columns of GatherResult.gatherresultdict.

    ``noident_hashes``: hashes of the query known to match nothing (what ``sourmash gather`` collects
    from its prefetch stage, commands.py:894-922,973): they are taken out of the query that is searched,
    but stay in the denominators -- query_bp, query_n_hashes, f_orig_query, f_unique_to_query,
    total_weighted_hashes -- and in remaining_bp (GatherDatabases.__init__ / __next__,
    search.py:803-818,910-944; GatherResult.build_gather_result, search.py:553-590).

    ``stats`` (a dict, optional) receives what the rounds leave behind: ``q_hashes`` (the searched query), ``alive``
    (the mask of its hashes no pick took), ``counts0`` (every row's overlap with it, the prefetch stage) and
    ``min_count`` (the least overlap of a row that takes part).  Without a round: ``counts0`` is None."""
    p = _prepare_query(query_mh, threshold_bp=threshold_bp, ignore_abundance=ignore_abundance,
                       noident_hashes=noident_hashes, query_orig=query_orig, query_name=query_name,
                       query_filename=query_filename)
    rows = []
    if stats is not None:
        stats.update(q_hashes=p.q_hashes if p is not None else query_mh._mins_array(), counts0=None, min_count=None)
        stats["alive"] = np.ones(len(stats["q_hashes"]), dtype=bool)
    if p is None or len(db) == 0:
        return rows
    scaled = query_mh.scaled
    q_hashes, q_abunds = p.q_hashes, p.q_abunds
    sizes = db.sizes()
    counts0 = B.one_vs_many(q_hashes, db)                     # |match ∩ original query| for every row
    alive = np.ones(len(q_hashes), dtype=bool)                 # hashes of the searched query not yet covered
    if stats is not None:
        stats.update(counts0=counts0, alive=alive, min_count=p.min_count)
    remaining = len(q_hashes)
    rowmap = None
    if p.min_count > 1:                                        # the session's min_count is a hint; the rule is enforced here
        rowmap = np.nonzero(counts0.astype(np.int64) >= p.min_count)[0].astype(np.uint32)
        if len(rowmap) == 0:
            return rows
        sess = B.GatherSession(q_hashes, db.take_rows(rowmap), min_count=1)
    else:
        sess = B.GatherSession(q_hashes, db, min_count=1)
    if max_rounds is None:
        max_rounds = len(db)
    while remaining > 0 and len(rows) < max_rounds:
        try:                                                   # search.py:15-37, per current query size
            _, n_threshold = calc_threshold_from_bp(threshold_bp, scaled, remaining)
        except ValueError:
            break
        best, r = sess.peek()
        if best == 0 or best < n_threshold:
            break
        isect = sess.intersect(r)                              # remaining query ∩ row r (ascending)
        if rowmap is not None:
            r = int(rowmap[r])                                 # row of the caller's database
        pos = np.searchsorted(q_hashes, isect)
        alive[pos] = False
        left = sess.apply(isect)
        left_weight = int(q_abunds[alive].sum(dtype=object)) if p.track else int(alive.sum())
        rows.append(_gather_row(p, r, len(rows), q_abunds[pos], remaining, left_weight, int(counts0[r]), int(sizes[r]),
                                estimate_ani_ci=estimate_ani_ci, names=names, md5s=md5s, filenames=filenames,
                                locations=locations))
        remaining = left
    return rows


def gather_many(query_mhs, db, *, threshold_bp=0, ignore_abundance=False, estimate_ani_ci=False, names=None, md5s=None,
                filenames=None, locations=None, query_names=None, query_filenames=None, max_rounds=None,
                noident_hashes=None, query_origs=None, db_scaled=None):
    """gather_databases() of every query in ``query_mhs`` against the one resident ``db``; returns one list of GatherRow
    per query, each equal to what gather_databases returns for that query alone.  The rounds of all queries at one
    scaled run together on the device (batch.multigather); the report columns come from the picks, the overlaps and
    the round that consumed each query hash, read back once.

    ``db`` is sketched at ``db_scaled`` (default: the smallest scaled of the queries); queries at a coarser scaled are
    compared with one downsampled copy of it per distinct scaled.  ``query_names``, ``query_filenames``,
    ``noident_hashes`` and ``query_origs`` hold one entry per query (see gather_databases)."""
    n = len(query_mhs)

    def each(v, default=None):
        return list(v) if v is not None else [default] * n
    qnames, qfiles, noidents, origs = each(query_names, ""), each(query_filenames, ""), each(noident_hashes), each(query_origs)
    out = [[] for _ in range(n)]
    preps = [_prepare_query(mh, threshold_bp=threshold_bp, ignore_abundance=ignore_abundance, noident_hashes=noidents[i],
                            query_orig=origs[i], query_name=qnames[i], query_filename=qfiles[i])
             for i, mh in enumerate(query_mhs)]
    by_scaled = {}
    for i, p in enumerate(preps):
        if p is None:
            continue
        try:                                                   # the first round's threshold check (search.py:15-37)
            calc_threshold_from_bp(threshold_bp, p.mh.scaled, len(p.q_hashes))
        except ValueError:
            continue
        by_scaled.setdefault(p.mh.scaled, []).append(i)
    if not by_scaled or len(db) == 0:
        return out
    if db_scaled is None:
        db_scaled = min(by_scaled)
    for scaled in sorted(by_scaled):
        if scaled < db_scaled:
            raise ValueError("a query at scaled=%d cannot be compared with a database at scaled=%d" % (scaled, db_scaled))
        sdb = db if scaled == db_scaled else db.downsample(B.max_hash_for_scaled(scaled))
        idx = by_scaled[scaled]
        # gather_databases' stop rule per round, best < threshold_bp / scaled, on integer counters
        threshold = max(1, math.ceil(float(threshold_bp) / scaled)) if threshold_bp else 1
        stats = {}
        res = B.multigather([preps[i].q_hashes for i in idx], sdb, thresholds=threshold,
                            min_counts=[preps[i].min_count for i in idx],
                            max_rounds=len(sdb) if max_rounds is None else max_rounds, stats=stats)
        sizes = sdb.sizes()
        for i, (rows, _, consumed), overlaps in zip(idx, res, stats["overlaps"]):
            p = preps[i]
            order = np.argsort(consumed, kind="stable")        # hashes grouped by round, ascending inside each round
            bounds = np.searchsorted(consumed[order], np.arange(len(rows) + 1, dtype=np.uint32))
            remaining = len(p.q_hashes)
            left_weight = int(p.q_abunds.sum(dtype=object)) if p.track else remaining
            for k, r in enumerate(rows.tolist()):
                ab = p.q_abunds[order[bounds[k]:bounds[k + 1]]]
                left_weight -= int(ab.sum(dtype=object)) if p.track else len(ab)
                out[i].append(_gather_row(p, r, k, ab, remaining, left_weight, int(overlaps[k]), int(sizes[r]),
                                          estimate_ani_ci=estimate_ani_ci, names=names, md5s=md5s, filenames=filenames,
                                          locations=locations))
                remaining -= len(ab)
    return out


PREFETCH_COLUMNS = [  # search.py:364-388
    "intersect_bp", "jaccard", "max_containment", "f_query_match", "f_match_query", "match_filename", "match_name",
    "match_md5", "match_bp", "query_filename", "query_name", "query_md5", "query_bp", "ksize", "moltype", "scaled",
    "query_n_hashes", "query_abundance", "query_containment_ani", "match_containment_ani",
    "average_containment_ani", "max_containment_ani", "potential_false_negative"]


def _min_count_of_given_query(threshold_bp, query_orig, query_len):
    """Smallest overlap (in hashes of the comparison) that passes the reference's prefetch threshold when the query was given at a
    finer scaled than the comparison runs at: Index.prefetch turns threshold_bp into a containment
    (threshold_bp / scaled) / len(query) with the GIVEN query's scaled and length (make_containment_query, search.py:77-88;
    calc_threshold_from_bp :15-37) and Index.find compares it with shared / len(query downsampled) (index/__init__.py:151-164)
    -- so the bar in base pairs moves with the sampling noise of the downsampled query.  Same float operations as there."""
    frac = (float(threshold_bp) / int(query_orig[1])) / int(query_orig[0])
    c = max(1, int(math.ceil(frac * query_len)))
    while c > 1 and (c - 1) / query_len >= frac:
        c -= 1
    while c / query_len < frac:
        c += 1
    return c


def prefetch_database(query_mh, db, threshold_bp, *, estimate_ani_ci=False, names=None, md5s=None, filenames=None,
                      query_name="", query_filename="", query_orig=None, match_orig=None, counts=None):
    """All rows of ``db`` sharing at least ``threshold_bp`` with the query, in database order, as
    dictionaries with the reference's prefetch columns (search.py:953-998 + PrefetchResult
    :357-470).  One pass of the one-vs-many kernel; everything else is per-match scalar work.  ``counts``: the overlaps
    of that pass when the caller already has them (gather's prefetch stage), so the pass is not run again."""
    if not query_mh.scaled:
        raise TypeError("query signature must be calculated with scaled")
    scaled, ksize = query_mh.scaled, query_mh.ksize
    q = query_mh._mins_array()
    nq = len(q)
    if nq == 0:
        raise ValueError("query is empty!?")
    if query_orig is not None:                                 # ValueError if unattainable (search.py:15-37), judged on the query as given
        calc_threshold_from_bp(threshold_bp, int(query_orig[1]), int(query_orig[0]))
    else:
        calc_threshold_from_bp(threshold_bp, scaled, nq)
    if counts is None:
        counts = B.one_vs_many(q, db)
    sizes = db.sizes()
    cache = {}
    q_ok = _size_ok(nq, scaled, cache)
    out = []
    # sizes of the sketches AS GIVEN (PrefetchResult.init_sigcomparison, search.py:401-416: query_bp / match_bp are
    # unique_dataset_hashes of the given sketches, query_n_hashes their given length; the comparison itself is at `scaled`):
    # query_orig = (n hashes, scaled, md5sum), match_orig = (n hashes per row, scaled per row)
    query_md5 = (query_orig[2] if query_orig else query_mh.md5sum())[:8]
    query_n, query_bp = (int(query_orig[0]), int(query_orig[0]) * int(query_orig[1])) if query_orig else (nq, nq * scaled)
    if query_orig is not None and threshold_bp:
        passing = counts.astype(np.int64) >= _min_count_of_given_query(threshold_bp, query_orig, nq)
    else:
        passing = counts.astype(np.int64) * scaled >= max(threshold_bp, 1)
    for r in np.nonzero(passing)[0]:
        c, m = int(counts[r]), int(sizes[r])
        qc_c, mc_c = _contained_by(c, nq, scaled), _contained_by(c, m, scaled)
        qc = DU.containment_to_distance(qc_c, ksize, scaled, n_unique_kmers=nq * scaled, estimate_ci=estimate_ani_ci)
        mc = DU.containment_to_distance(mc_c, ksize, scaled, n_unique_kmers=m * scaled, estimate_ci=estimate_ani_ci)
        qc.size_is_inaccurate = mc.size_is_inaccurate = not (q_ok and _size_ok(m, scaled, cache))
        d = {"row": int(r), "intersect_bp": c * scaled, "jaccard": c / max(1, nq + m - c),
             "max_containment": _contained_by(c, min(nq, m), scaled), "f_query_match": mc_c, "f_match_query": qc_c,
             "match_bp": int(match_orig[0][r]) * int(match_orig[1][r]) if match_orig is not None else m * scaled,
             "query_bp": query_bp, "ksize": ksize, "moltype": query_mh.moltype,
             "scaled": scaled, "query_n_hashes": query_n, "query_abundance": bool(query_mh.track_abundance),
             "query_name": query_name, "query_filename": query_filename, "query_md5": query_md5,
             "potential_false_negative": bool(qc.p_exceeds_threshold or mc.p_exceeds_threshold)}
        if names is not None:
            d["match_name"] = names[r]
        if md5s is not None:
            d["match_md5"] = md5s[r][:8]
        if filenames is not None:
            d["match_filename"] = filenames[r]
        if qc.ani is not None:
            d["query_containment_ani"] = qc.ani
        if mc.ani is not None:
            d["match_containment_ani"] = mc.ani
        if qc.ani is not None and mc.ani is not None:
            d["average_containment_ani"] = (qc.ani + mc.ani) / 2
            d["max_containment_ani"] = max(qc.ani, mc.ani)
        if estimate_ani_ci:
            d.update(query_containment_ani_low=qc.ani_low, query_containment_ani_high=qc.ani_high,
                     match_containment_ani_low=mc.ani_low, match_containment_ani_high=mc.ani_high)
        out.append(d)
    return out


def write_gather_csv(rows, fp, *, estimate_ani_ci=False):
    """Write GatherRow objects as the reference's `gather -o` CSV: same columns in the same order
    (search.py:480-523), empty cells for values that are None, query md5 shortened to 8 characters
    (prep_gather_result, search.py:633-637)."""
    import csv
    cols = GATHER_COLUMNS + (CI_COLUMNS if estimate_ani_ci else [])
    if not rows:
        return                                             # the reference writes the header with the first result: no results, empty file
    w = csv.DictWriter(fp, fieldnames=cols)
    w.writeheader()
    for g in rows:
        w.writerow(g.to_dict(estimate_ani_ci))


def write_prefetch_csv(results, fp, *, estimate_ani_ci=False):
    "Write prefetch_database() results as the reference's `prefetch -o` CSV (search.py:364-395)."
    import csv
    cols = PREFETCH_COLUMNS + (CI_COLUMNS if estimate_ani_ci else [])
    if not results:
        return                                             # no results: an empty file, like the reference
    w = csv.DictWriter(fp, fieldnames=cols, extrasaction="ignore")
    w.writeheader()
    for d in results:
        w.writerow({k: v for k, v in d.items() if v is not None})


SEARCH_COLUMNS = ["similarity", "md5", "filename", "name", "query_filename", "query_name", "query_md5", "ani"]  # search.py:292-303
SEARCH_CI_COLUMNS = ["ani_low", "ani_high"]


def search_database(query_mh, db, *, threshold=0.08, do_containment=False, do_max_containment=False, best_only=False,
                    estimate_ani_ci=False, names=None, md5s=None, filenames=None, query_name="", query_filename="",
                    location=None, locations=None, groups=None, query_orig=None):
    """`sourmash search` of a flat scaled query against the rows of the GPU-resident SketchSet ``db``
    (same ksize / seed / scaled as the query): Jaccard, containment of the query or max-containment
    at or above ``threshold``, best first, one entry per md5
    (search_databases_with_flat_query, search.py:686-733, over Index.find / JaccardSearch,
    index/__init__.py:115-170, search.py:91-169).  Returns dictionaries with the columns of
    SearchResult (search.py:283-355): ``ani`` from the containment handed in (containment), the
    bias-corrected max containment (max-containment) or the Jaccard value; the confidence interval
    only for the two containment searches, like the reference.  One launch of the one-vs-many kernel."""
    if do_containment and do_max_containment:
        raise TypeError("'do_containment' and 'do_max_containment' cannot both be True")
    if query_mh.track_abundance:
        raise TypeError("this search cannot be done with an abund signature")
    if not query_mh.scaled:
        raise TypeError("this search requires a scaled signature")
    scaled, ksize = query_mh.scaled, query_mh.ksize
    q = query_mh._mins_array()
    nq = len(q)
    counts = B.one_vs_many(q, db).astype(np.int64)
    sizes = db.sizes().astype(np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        if do_containment:
            score = counts / nq if nq else np.zeros(len(counts))
        elif do_max_containment:
            d = np.minimum(nq, sizes)
            score = np.where(d > 0, counts / np.maximum(d, 1), 0.0)
        else:
            tot = nq + sizes - counts
            score = np.where(tot > 0, counts / np.maximum(tot, 1), 0.0)
    # index order; best_only ratchets the threshold (JaccardSearchBestOnly.collect, search.py:163-169) -- inside one
    # database: the reference searches database after database, each with a search function of its own
    # (search_databases_with_flat_query, search.py:676-691), so with ``groups`` (database id of every row) the ratchet
    # starts again at every new database
    floor = float(threshold or 0)
    threshold = floor
    picked = []
    for r in range(len(counts)):
        if groups is not None and r and groups[r] != groups[r - 1]:
            threshold = floor
        s = float(score[r])
        if s and s >= threshold:
            if best_only:
                threshold = max(threshold, s)
            picked.append(r)
    seen, uniq = set(), []
    for r in picked:
        key = md5s[r] if md5s is not None else r
        if key not in seen:
            seen.add(key)
            uniq.append(r)
    uniq.sort(key=lambda r: -float(score[r]))                  # stable: ties keep database order
    cache = {}
    q_ok = _size_ok(nq, scaled, cache)
    query_md5 = (query_orig[2] if query_orig else query_mh.md5sum())[:8]      # the query as given (get_cmpinfo, search.py:222-243)
    ci = estimate_ani_ci and (do_containment or do_max_containment)
    out = []
    for r in uniq:
        c, m, s = int(counts[r]), int(sizes[r]), float(score[r])
        if do_containment:
            res = DU.containment_to_distance(s, ksize, scaled, n_unique_kmers=nq * scaled, estimate_ci=ci)
        elif do_max_containment:
            res = DU.containment_to_distance(_contained_by(c, min(nq, m), scaled), ksize, scaled,
                                             n_unique_kmers=min(nq, m) * scaled, estimate_ci=ci)
        else:
            res = DU.jaccard_to_distance(s, ksize, scaled, n_unique_kmers=round((nq + m) / 2 * scaled))
        if not (q_ok and _size_ok(m, scaled, cache)):
            res.size_is_inaccurate = True
        d = {"row": int(r), "similarity": s, "query_name": query_name, "query_filename": query_filename,
             "query_md5": query_md5, "ani": res.ani,
             "potential_false_negative": bool(res.p_exceeds_threshold)}
        if md5s is not None:
            d["md5"] = md5s[r]
        if names is not None:
            d["name"] = names[r]
        # BaseResult.get_cmpinfo (search.py:230-234): the location passed by the search wins, else the
        # filename stored in the match
        if locations is not None:                     # one location per row (several database files behind one SketchSet)
            d["filename"] = locations[r]
        else:
            d["filename"] = location if location is not None else (filenames[r] if filenames is not None else None)
        if ci:
            d["ani_low"], d["ani_high"] = res.ani_low, res.ani_high
        out.append(d)
    return out


def write_search_csv(results, fp, *, estimate_ani_ci=False):
    "Write search_database() results as the reference's `search -o` CSV (search.py:292-307)."
    import csv
    cols = SEARCH_COLUMNS + (SEARCH_CI_COLUMNS if estimate_ani_ci else [])
    if not results:
        return                                             # no results: an empty file, like the reference
    w = csv.DictWriter(fp, fieldnames=cols, extrasaction="ignore")
    w.writeheader()
    for d in results:
        w.writerow({k: v for k, v in d.items() if v is not None})
