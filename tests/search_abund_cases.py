"""Shared cases of the abundance-search tests (batch.search_angular, LinearIndex / ZipFileLinearIndex.search_abund):
sketch sets and indexes with every edge the angular pass has to get right, a numpy restatement of the per-row terms
(u64 sums that wrap, the score finalized with math.acos row by row), and the reference's per-subject loop
(Index.search_abund, src/sourmash/index/__init__.py:172-200) written with this package's MinHash."""
import math

import numpy as np

U64_MAX = np.iinfo(np.uint64).max
SPLIT_MAX = 16382                  # largest query that becomes the shared-memory split table (ANGULAR_SPLIT_MAX)


def csr(rows, abunds):
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    h = np.concatenate(rows).astype(np.uint64) if rows else np.zeros(0, np.uint64)
    a = np.concatenate(abunds).astype(np.uint64) if rows else np.zeros(0, np.uint64)
    return h, off, a


def score_of(prod, a_sq, b_sq):
    "the tail of KmerMinHash::angular_similarity on u64 terms, as the library's host code computes it"
    norm_a, norm_b = math.sqrt(float(int(a_sq))), math.sqrt(float(int(b_sq)))
    if norm_a == 0. or norm_b == 0.:
        return 0.0
    p = min(float(int(prod)) / (norm_a * norm_b), 1.0)
    return 1. - 2. * math.acos(p) / math.pi


def numpy_angular(qh, qa, h, off, ab, max_hash, block=1 << 24):
    """float64 score of every row of the CSR (h, off, ab) against the query, over the hashes <= max_hash of both:
    prod / bsq per row as wrapping u64 sums (a cumulative sum and differences at the row ends), blocks of rows at a
    time so that a database of 10^8 elements fits in host memory."""
    qh, qa = np.asarray(qh, np.uint64), np.asarray(qa, np.uint64)
    keep_q = qh <= np.uint64(max_hash)
    qh, qa = qh[keep_q], qa[keep_q]
    a_sq = int(np.sum(qa * qa, dtype=np.uint64)) if len(qa) else 0
    off = np.asarray(off, np.int64)
    n = len(off) - 1
    out = np.zeros(n, np.float64)
    r0 = 0
    while r0 < n:
        r1 = r0 + 1
        while r1 < n and off[r1 + 1] - off[r0] <= block:
            r1 += 1
        lo, hi = int(off[r0]), int(off[r1])
        x, s = h[lo:hi], ab[lo:hi]
        keep = x <= np.uint64(max_hash)
        if len(qh):
            pos = np.minimum(np.searchsorted(qh, x), len(qh) - 1)
            hit = keep & (qh[pos] == x)
            prod_el = np.where(hit, qa[pos] * s, np.uint64(0))
        else:
            prod_el = np.zeros(len(x), np.uint64)
        sq_el = np.where(keep, s * s, np.uint64(0))
        ends = off[r0 + 1:r1 + 1] - lo
        starts = off[r0:r1] - lo
        for name, el in (("prod", prod_el), ("bsq", sq_el)):
            cs = np.concatenate([[np.uint64(0)], np.cumsum(el, dtype=np.uint64)])
            tot = cs[ends] - cs[starts]                      # wraps, like the sums themselves
            if name == "prod":
                prod = tot
            else:
                bsq = tot
        for i in range(r1 - r0):
            out[r0 + i] = score_of(prod[i], a_sq, bsq[i])
        r0 = r1
    return out


def _row(rng, pool, k):
    return np.unique(rng.choice(pool, size=min(k, len(pool)), replace=False)).astype(np.uint64)


def set_cases(rng):
    """(tag, q_hashes, q_abunds, rows, abund_rows, max_hash) for batch.search_angular: an empty set, an empty query,
    empty rows, rows emptied by max_hash, a query cut to nothing, UINT64_MAX on both sides, identical rows (the min(., 1)
    clamp), abundances >= 2^32 (a*b and a*a wrap), a duplicated row, rows longer than a chunk and a query above the
    split-table limit."""
    pool = rng.integers(1, 2**63, size=60_000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    pool = np.unique(pool)
    ab = lambda r, hi=100: rng.integers(1, hi, size=len(r)).astype(np.uint64)   # noqa: E731
    out = []
    q = _row(rng, pool[:3000], 800)
    rows = [_row(rng, pool[:3000], int(rng.integers(0, 900))) for _ in range(9)]
    out.append(("empty set", q, ab(q), [], [], U64_MAX))
    out.append(("empty query", np.zeros(0, np.uint64), np.zeros(0, np.uint64), rows, [ab(r) for r in rows], U64_MAX))
    rows_e = [np.zeros(0, np.uint64)] + rows[:4] + [np.zeros(0, np.uint64)] + rows[4:]
    out.append(("empty rows", q, ab(q), rows_e, [ab(r) for r in rows_e], U64_MAX))
    cut = np.uint64(2**62)
    low = pool[pool <= cut]
    high = pool[pool > cut]
    rows_c = [_row(rng, high[:2000], 300), _row(rng, np.concatenate([low[:500], high[:500]]), 400),
              _row(rng, high[:2000], 50), np.zeros(0, np.uint64)]
    qc = _row(rng, np.concatenate([low[:500], high[:2000]]), 900)
    out.append(("rows emptied by max_hash", qc, ab(qc), rows_c, [ab(r) for r in rows_c], int(cut)))
    qh = _row(rng, high[:2000], 400)
    out.append(("query cut to nothing", qh, ab(qh), rows_c, [ab(r) for r in rows_c], int(cut)))
    top = np.array([U64_MAX - np.uint64(i) for i in range(8)], np.uint64)
    qt = np.unique(np.concatenate([q[:200], top[[0, 3, 5]]]))
    rows_t = [np.unique(np.concatenate([_row(rng, q, 100), top[[0]]])), np.unique(np.concatenate([q[:50], top[[1, 3]]])),
              top[[0]], _row(rng, q, 120)]
    out.append(("UINT64_MAX keys", qt, ab(qt), rows_t, [ab(r) for r in rows_t], U64_MAX))
    qa = ab(q)
    out.append(("identical rows", q, qa, [q.copy(), q.copy(), q[:10].copy()], [qa.copy(), qa * np.uint64(3), qa[:10].copy()],
                U64_MAX))
    big = lambda r: rng.integers(2**32, 2**63, size=len(r), dtype=np.uint64)     # noqa: E731
    out.append(("abundances >= 2^32", q, big(q), rows, [big(r) for r in rows], U64_MAX))
    rd = [rows[0], rows[1], rows[0], rows[2]]
    ad = [ab(rows[0])] * 2
    out.append(("duplicated row", q, ab(q), rd, [ad[0], ab(rows[1]), ad[1], ab(rows[2])], U64_MAX))
    long_rows = [_row(rng, pool[:20_000], k) for k in (5000, 1024, 1025, 3, 12_000)]
    ql = _row(rng, pool[:20_000], 6000)
    out.append(("rows longer than a chunk", ql, ab(ql), long_rows, [ab(r) for r in long_rows], U64_MAX))
    qb = _row(rng, pool, SPLIT_MAX + 500)
    rows_b = [_row(rng, pool, int(rng.integers(0, 4000))) for _ in range(12)] + [qb[:3000].copy()]
    out.append(("query above the split-table limit", qb, ab(qb), rows_b, [ab(r) for r in rows_b], U64_MAX))
    out.append(("query above the split-table limit, cut", qb, ab(qb), rows_b, [ab(r) for r in rows_b], int(cut)))
    qs = qb[:SPLIT_MAX]
    out.append(("query at the split-table limit", qs, ab(qs), rows_b, [ab(r) for r in rows_b], U64_MAX))
    return out


# ---------------------------------------------------------------- indexes of signatures
def minhash_of(hashes, abunds, *, scaled=0, num=0, ksize=31, seed=42, moltype="DNA"):
    from sourmash_b200.minhash import MinHash
    kw = {"is_protein": moltype == "protein", "dayhoff": moltype == "dayhoff", "hp": moltype == "hp"}
    mh = MinHash(num, ksize, scaled=scaled, seed=seed, track_abundance=abunds is not None, **kw)
    if abunds is None:
        mh.add_many([int(x) for x in hashes])
    else:
        mh.set_abundances({int(x): int(y) for x, y in zip(hashes, abunds)})
    return mh


def sig_of(hashes, abunds, name, **kw):
    from sourmash_b200.signature import SourmashSignature
    return SourmashSignature(minhash_of(hashes, abunds, **kw), name=name)


def _max_hash(scaled):
    from sourmash_b200 import batch as B
    return B.max_hash_for_scaled(scaled)


def index_cases(rng):
    """(tag, query signature, subject signatures, threshold) for search_abund.  The subjects mix groups: the query's
    scaled, a coarser scaled (the query is cut), a finer scaled (the subject is cut); num groups of the query's num and
    of other nums, with UINT64_MAX keys; identical sketches, ties, a duplicated subject, a large query."""
    pool = np.unique(rng.integers(1, 2**64 - 1, size=40_000, dtype=np.uint64))
    out = []

    def draw(scaled, k, sub=pool):
        mx = np.uint64(_max_hash(scaled)) if scaled else U64_MAX
        return _row(rng, sub[sub <= mx], k)

    ab = lambda r: rng.integers(1, 100, size=len(r)).astype(np.uint64)   # noqa: E731
    qh = draw(10, 2000)
    q = sig_of(qh, ab(qh), "q", scaled=10)
    subs = []
    for i in range(24):
        s = (10, 100, 2, 10, 1000)[i % 5]
        h = np.unique(np.concatenate([draw(s, int(rng.integers(0, 1500))), draw(s, 300, qh)]))
        subs.append(sig_of(h, ab(h), "s%d" % i, scaled=s))
    subs.insert(5, sig_of(qh, q.minhash._abunds_array(), "identical", scaled=10))
    subs.insert(9, subs[3])
    subs.append(sig_of(np.zeros(0, np.uint64), np.zeros(0, np.uint64), "empty", scaled=10))
    for thr in (0.0, 0.05, 0.3, 1.0):
        out.append(("mixed scaled, threshold %g" % thr, q, subs, thr))
    # ties: the same sketch under several names (and threshold 0 keeps every subject, in index order among equals)
    t = [sig_of(qh[:500], ab(qh[:500]), "t%d" % i, scaled=10) for i in range(2)]
    out.append(("ties", q, [t[0], subs[0], t[1], t[0], subs[1], t[1]], 0.0))
    # num groups, UINT64_MAX keys on both sides
    top = np.array([U64_MAX, U64_MAX - np.uint64(7)], np.uint64)
    nq = np.unique(np.concatenate([pool[:400], top]))
    qn = sig_of(nq, ab(nq), "qn", num=500)
    subs_n = []
    for i, num in enumerate((500, 500, 300, 1000, 500)):
        h = np.unique(np.concatenate([_row(rng, pool[:2000], min(num, 350)), top[:1 + i % 2]]))
        subs_n.append(sig_of(h, ab(h), "n%d" % i, num=num))
    out.append(("num groups with UINT64_MAX", qn, subs_n, 0.0))
    s1 = np.unique(np.concatenate([pool[:300], top[:1]]))
    q1 = sig_of(s1, ab(s1), "q1", scaled=1)
    out.append(("scaled 1 with UINT64_MAX", q1, [sig_of(s1, ab(s1), "a", scaled=1),
                                                 sig_of(s1[::2], ab(s1[::2]), "b", scaled=1)], 0.0))
    # abundances >= 2^32: the products and squares wrap
    big = lambda r: rng.integers(2**32, 2**63, size=len(r), dtype=np.uint64)   # noqa: E731
    out.append(("abundances >= 2^32", sig_of(qh, big(qh), "qbig", scaled=10),
                [sig_of(s.minhash._mins_array(), big(s.minhash._mins_array()), s.name, scaled=s.minhash.scaled)
                 for s in subs[:8]], 0.0))
    # a query above the split-table limit: the global-directory layout
    lh = draw(1, SPLIT_MAX + 3000)
    ql = sig_of(lh, ab(lh), "qlarge", scaled=1)
    subs_l = [sig_of(h, ab(h), "l%d" % i, scaled=s) for i, (s, h) in
              enumerate((s, np.unique(np.concatenate([draw(s, 2000), draw(s, 1500, lh)]))) for s in (1, 1, 3, 1, 2))]
    out.append(("query above the split-table limit", ql, subs_l, 0.0))
    return out


def error_cases(rng):
    """(tag, query, subjects, threshold): each raises in the reference's loop, at the subject named in the tag."""
    pool = np.unique(rng.integers(1, 2**60, size=5000, dtype=np.uint64))
    ab = lambda r: rng.integers(1, 50, size=len(r)).astype(np.uint64)   # noqa: E731

    def s(name, track=True, **kw):
        h = _row(rng, pool, 200)
        return sig_of(h, ab(h) if track else None, name, **kw)

    q = s("q", scaled=10)
    good = [s("g%d" % i, scaled=(10, 100)[i % 2]) for i in range(4)]
    out = [("flat query", s("qflat", track=False, scaled=10), good, 0.0),
           ("threshold None", q, good, None),
           ("flat subject at 2", q, good[:2] + [s("flat", track=False, scaled=10)] + good[2:], 0.0),
           ("ksize at 3", q, good[:3] + [s("k", scaled=10, ksize=21)] + good[3:], 0.0),
           ("moltype at 1", q, good[:1] + [s("p", scaled=10, ksize=10, moltype="protein")] + good[1:], 0.0),
           ("seed at 4", q, good + [s("seed", scaled=10, seed=7)], 0.0),
           ("num subject at 2", q, good[:2] + [s("num", num=300)] + good[2:], 0.0),
           ("scaled subject for a num query at 0", s("qn", num=300), [s("sc", scaled=10), s("n2", num=300)], 0.5),
           ("flat before incompatible", q, good[:1] + [s("flat", track=False, scaled=10), s("k", scaled=10, ksize=21)],
            0.0),
           ("incompatible before flat", q, good[:1] + [s("k", scaled=10, ksize=21), s("flat", track=False, scaled=10)],
            0.0)]
    return out


def reference_search_abund(query, subjects, threshold):
    "Index.search_abund of the reference (index/__init__.py:172-200) over (subject, location) pairs"
    if not query.minhash.track_abundance:
        raise TypeError("'search_abund' requires query signature with abundance information")
    if threshold is None:
        raise TypeError("'search_abund' requires 'threshold'")
    threshold = float(threshold)
    matches = []
    for subj, loc in subjects:
        if not subj.minhash.track_abundance:
            raise TypeError("'search_abund' requires subject signatures with abundance information")
        score = query.similarity(subj, downsample=True)
        if score >= threshold:
            matches.append((score, subj, loc))
    matches.sort(key=lambda x: -x[0])
    return matches


def outcome(fn):
    "('ok', [(score bits, name, md5, location)]) or ('raise', exception type name, message)"
    try:
        res = fn()
    except Exception as e:                                   # noqa: BLE001 -- the exception is what is compared
        return ("raise", type(e).__name__, str(e))
    return ("ok", [(np.float64(r[0]).tobytes(), r[1].name, r[1].md5sum(), r[2]) for r in res])


# ---------------------------------------------------------------- the benchmark's workloads
def bench_workload(which, db=None):
    """(q_hashes, q_abunds, hashes, offsets, abunds) of workload 1, 2 or 3 of scripts/bench_search_abund.py, at scaled
    1000 (synth.MAX_HASH_1000), abundances 1..99 from a seeded generator:
      1  50 000 genome-sized subjects (synth_sketches: ~5 000 hashes, 100 families) and a 10^4-hash query drawn from
         the first 200 subjects, so that every family has hits (the split-table layout)
      2  the same database and a 10^6-hash query: those 10^4 hashes plus uniform ones (the global directory)
      3  1 000 sample-sized subjects of ~2 x 10^5 hashes and a 2 x 10^5-hash query drawn from their pools (long rows)
    ``db``: the (hashes, offsets, abunds) of workload 1 or 2, to build the other one's query without generating it again."""
    from sourmash_b200.synth import MAX_HASH_1000, synth_sketches
    rng = np.random.default_rng(100 + which)
    if which in (1, 2):
        if db is None:
            h, off = synth_sketches(50_000)
            ab = np.random.default_rng(7).integers(1, 100, size=len(h)).astype(np.uint64)
        else:
            h, off, ab = db
        q = np.unique(rng.choice(h[:int(off[200])], size=10_000, replace=False))
        if which == 2:
            extra = rng.integers(1, MAX_HASH_1000, size=1_000_000 - len(q), dtype=np.uint64, endpoint=True)
            q = np.unique(np.concatenate([q, extra]))
    else:
        h, off = synth_sketches(1000, mean=200_000, sd=20_000, lo=150_000, hi=250_000, n_families=20, pool=250_000)
        ab = np.random.default_rng(7).integers(1, 100, size=len(h)).astype(np.uint64)
        q = np.unique(rng.choice(h[:int(off[20])], size=200_000, replace=False))
    qa = rng.integers(1, 100, size=len(q)).astype(np.uint64)
    return q, qa, h, off, ab
