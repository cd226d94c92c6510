"""Shared cases of the LCA table and counts (batch.lca_table / batch.lca_counts), and the oracle: the reference's
gather_assignments and count_lca_for_assignments (src/sourmash/lca/lca_utils.py:137-225) restated in plain Python over
lineage tuples, with Counter.most_common() order.  The reference's LCA test data are stored gzip-compressed under
tests/golden/refdata/lca; ``unpack_fixtures`` writes them out as the reference names them."""
import gzip
import os
from collections import Counter

import numpy as np

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refdata", "lca")
RANKS = ("superkingdom", "phylum", "class", "order", "family", "genus", "species", "strain")
DATABASES = ("delmont-1.lca.json", "delmont-2.lca.json", "dir1.lca.json", "dir2.lca.json", "both.lca.json",
             "47+63.lca.json")


def unpack_fixtures(dst):
    "every fixture decompressed into dst under its reference name, plus delmont-1.lca.json.gz as stored"
    os.makedirs(dst, exist_ok=True)
    for name in sorted(os.listdir(FIXTURES)):
        with gzip.open(os.path.join(FIXTURES, name)) as fh, open(os.path.join(dst, name[:-3]), "wb") as out:
            out.write(fh.read())
    with open(os.path.join(FIXTURES, "delmont-1.lca.json.gz"), "rb") as fh, \
            open(os.path.join(dst, "delmont-1.lca.json.gz"), "wb") as out:
        out.write(fh.read())
    return dst


def tree_of(lineages):
    "build_tree: nested dicts keyed by (rank, name), empty names skipped"
    tree = {}
    for lin in lineages:
        node = tree
        for rank, name in zip(RANKS, lin):
            if name:
                node = node.setdefault((rank, name), {})
    return tree


def walk(tree):
    "find_lca: descend while a node has one child; the path as (rank, name) pairs"
    path = []
    while len(tree) == 1:
        (key, tree), = tree.items()
        path.append(key)
    return tuple(path)


def oracle_counts(query, dbs, weights=None):
    """count_lca_for_assignments(gather_assignments(query, dbs), weights) for one query (ascending hashes):
    [(lca path, count)] in most_common() order.  A db is (hash -> [idx]) and idx -> lineage (8 names) or None."""
    assignments = {}
    for i, h in enumerate(query):
        for hash_to_idx, idx_lineage in dbs:
            lins = [idx_lineage.get(x) for x in hash_to_idx.get(int(h), [])]
            lins = [lin for lin in lins if lin is not None]
            if lins:
                assignments.setdefault(int(h), (i, set()))[1].update(lins)
    counts = Counter()
    for h, (i, lins) in assignments.items():
        counts[walk(tree_of(lins))] += 1 if weights is None else int(weights[i])
    return counts.most_common()


def random_dbs(rng, n_dbs=3, n_lineages=40, n_hashes=3000, pool=None):
    """databases over one random taxonomy: lineages with empty middle ranks, all-empty lineages, lineages that differ at
    superkingdom, idx without a lineage, and hashes shared between databases"""
    names = [["%s%d" % (r[:2], k) for k in range(3)] for r in RANKS]
    lineages = []
    for _ in range(n_lineages):
        depth = int(rng.integers(0, 9))
        lin = [names[r][int(rng.integers(0, 3))] if r < depth else "" for r in range(8)]
        if depth > 2 and rng.random() < 0.3:
            lin[int(rng.integers(1, depth - 1))] = ""
        lineages.append(tuple(lin))
    lineages.append(("",) * 8)
    if pool is None:
        pool = rng.integers(1, 2**64 - 1, size=n_hashes, dtype=np.uint64)
        pool[:3] = [2**64 - 1, 0, 1]
    dbs = []
    for _ in range(n_dbs):
        n_idx = int(rng.integers(5, 30))
        idx_lineage = {x: lineages[int(rng.integers(0, len(lineages)))] for x in range(n_idx) if rng.random() < 0.85}
        hash_to_idx = {}
        for h in rng.choice(pool, size=len(pool) // 2, replace=False):
            hash_to_idx[int(h)] = sorted(set(int(x) for x in rng.integers(0, n_idx, size=int(rng.integers(1, 4)))))
        dbs.append((hash_to_idx, idx_lineage))
    return dbs, pool


def fixture_dbs():
    "the reference's LCA fixtures as (hash -> [idx], idx -> lineage) pairs, read with json"
    import json
    out = []
    for name in DATABASES:
        with gzip.open(os.path.join(FIXTURES, name + ".gz"), "rt") as fh:
            d = json.load(fh)
        lid_lin = {int(k): tuple(dict((x[0], x[1]) for x in v).get(r, "") or "" for r in RANKS)
                   for k, v in d["lid_to_lineage"].items()}
        idx_lineage = {int(k): lid_lin[v] for k, v in d["idx_to_lid"].items()}
        hash_to_idx = {int(k): v for k, v in d["hashval_to_idx"].items()}
        out.append((hash_to_idx, idx_lineage))
    return out


def device_counts(dbs, queries, weights=None):
    """the same through the package: Taxonomy over the lineages, batch.lca_table, batch.lca_counts, then
    lca.ranked_counts' order; per query [(lca path, count)]"""
    from sourmash_b200 import batch as B
    from sourmash_b200 import lca as L

    class Db:
        pass
    objs = []
    for hash_to_idx, idx_lineage in dbs:
        db = Db()
        lins = sorted(set(idx_lineage.values()))
        lid = {lin: k for k, lin in enumerate(lins)}
        db.lid_to_lineage = {k: lin for lin, k in lid.items()}
        db.idx_to_lid = {x: lid[lin] for x, lin in idx_lineage.items()}
        pairs = [(h, x) for h, xs in hash_to_idx.items() for x in xs]
        db.hashes = np.array([p[0] for p in pairs], dtype=np.uint64)
        db.idx = np.array([p[1] for p in pairs], dtype=np.uint32)
        objs.append(db)
    tax = L.Taxonomy(objs)
    table = L.build_table(objs, tax)
    qs = [np.asarray(q, dtype=np.uint64) for q in queries]
    off = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.uint64)
    h = np.concatenate(qs) if qs else np.zeros(0, np.uint64)
    w = None if weights is None else np.concatenate(weights).astype(np.uint64)
    sset = B.SketchSet.from_host(h, off, w)
    ranked = L.ranked_counts(table, sset, len(qs), w is not None)

    def path(node):
        return tuple(tax.lineage(node))
    return [[(path(n), c) for n, c in r] for r in ranked], table, tax


class SynthDb:
    "an LcaDatabase's arrays without a file: hashes / idx pairs, idx_to_lid, lid_to_lineage"

    def __init__(self, hashes, idx, idx_to_lid, lid_to_lineage):
        self.hashes, self.idx, self.idx_to_lid, self.lid_to_lineage = hashes, idx, idx_to_lid, lid_to_lineage


def synth_lca(seed=1, n_lineages=100_000, n_pairs=10_000_000, n_queries=1000, query_len=5000, n_dbs=2):
    """A GTDB-sized synthetic setting (seeded): n_lineages genomes with 8-rank lineages drawn from a branching taxonomy
    (some strain names empty), n_pairs (hash, genome) pairs split over n_dbs databases (about 1 hash in 8 also held by
    another genome), and n_queries queries of query_len hashes, 90 % drawn from
    one genome's neighbourhood of the database and 10 % unknown.  Returns (dbs, queries)."""
    rng = np.random.default_rng(seed)
    fan = (4, 12, 4, 5, 6, 8, 6, 3)                          # children per rank: 4 * 12 * ... leaves
    codes = np.stack([rng.integers(0, f, size=n_lineages) for f in fan], axis=1)
    for r in range(1, 8):                                     # names are unique per path prefix
        codes[:, r] += codes[:, r - 1] * fan[r]
    lineages = [tuple("%s_%d" % (RANKS[r][:2], c[r]) if (r < 7 or c[r] % 3) else "" for r in range(8))
                for c in codes.tolist()]
    genome_of_pair = rng.integers(0, n_lineages, size=n_pairs).astype(np.uint32)
    hashes = rng.integers(1, 2**64 - 1, size=n_pairs, dtype=np.uint64)
    shared = rng.random(n_pairs) < 0.125                     # share the hash of a nearby earlier pair
    src = np.maximum(np.arange(n_pairs) - rng.integers(1, 1000, size=n_pairs), 0)
    hashes[shared] = hashes[src[shared]]
    dbs = []
    cuts = np.linspace(0, n_pairs, n_dbs + 1).astype(np.int64)
    for d in range(n_dbs):
        sl = slice(int(cuts[d]), int(cuts[d + 1]))
        idx_to_lid = {g: g for g in range(n_lineages)}
        dbs.append(SynthDb(hashes[sl].copy(), genome_of_pair[sl].copy(), idx_to_lid,
                           {g: lineages[g] for g in range(n_lineages)}))
    queries = []
    for _ in range(n_queries):
        start = int(rng.integers(0, max(n_pairs - 20 * query_len, 1)))
        known = rng.choice(hashes[start:start + 20 * query_len], size=int(query_len * 0.9), replace=False)
        unknown = rng.integers(1, 2**64 - 1, size=query_len - len(known), dtype=np.uint64)
        queries.append(np.unique(np.concatenate([known, unknown])))
    return dbs, queries


def synth_oracle(dbs, queries):
    "oracle_counts for each of ``queries`` against SynthDb databases, each hash's pairs found by searchsorted"
    sorted_dbs = []
    for db in dbs:
        o = np.argsort(db.hashes, kind="stable")
        sorted_dbs.append((db.hashes[o], db.idx[o], db))
    out = []
    for query in queries:
        query = np.asarray(query, dtype=np.uint64)
        assignments = {}
        for hs, ix, db in sorted_dbs:
            lo, hi = np.searchsorted(hs, query, "left"), np.searchsorted(hs, query, "right")
            for i in np.nonzero(hi > lo)[0].tolist():
                lins = assignments.setdefault(i, set())
                for x in ix[lo[i]:hi[i]].tolist():
                    lins.add(db.lid_to_lineage[db.idx_to_lid[x]])
        counts = Counter()
        for i in sorted(assignments):
            counts[walk(tree_of(assignments[i]))] += 1
        out.append(counts.most_common())
    return out
