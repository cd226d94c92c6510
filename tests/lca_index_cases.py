"""Shared cases of the LCA database build (batch.lca_index), and the oracle: the reference's insert loop
(LCA_Database.insert, src/sourmash/lca/lca_db.py:145-205) restated over numpy rows -- a dict of sets filled in row
order -- and serialised with json.dumps as save_to_json does (:456-458), with each idx list ascending where the
reference writes list(set).  The reference's spreadsheets and genome signatures for `lca index` are stored
gzip-compressed under tests/golden/refdata/lca_index; ``unpack_fixtures`` writes them out under their reference names."""
import gzip
import json
import os

import numpy as np

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refdata", "lca_index")
U64_MAX = 2**64 - 1


def unpack_fixtures(dst):
    "every fixture decompressed into dst, keeping the sub-directories (dir1/, dir2/, lca-root/)"
    for root, _dirs, names in os.walk(FIXTURES):
        for name in names:
            rel = os.path.relpath(os.path.join(root, name), FIXTURES)[:-3]
            os.makedirs(os.path.dirname(os.path.join(dst, rel)) or dst, exist_ok=True)
            with gzip.open(os.path.join(root, name)) as fh, open(os.path.join(dst, rel), "wb") as out:
                out.write(fh.read())
    return dst


def oracle(rows):
    """(hashes in key order, offsets, idx, text) of the insert loop over ``rows`` (row r is idx r, ascending hashes)"""
    hashval_to_idx = {}
    for idx, row in enumerate(rows):
        for h in row.tolist():
            hashval_to_idx.setdefault(h, set()).add(idx)
    hashes = np.array(list(hashval_to_idx), dtype=np.uint64)
    lists = [sorted(v) for v in hashval_to_idx.values()]
    offsets = np.concatenate([[0], np.cumsum([len(v) for v in lists])]).astype(np.uint64)
    idx = np.array([x for v in lists for x in v], dtype=np.uint32)
    text = json.dumps(dict(zip(hashval_to_idx, lists))).encode()
    return hashes, offsets, idx, text


def np_oracle_arrays(h, off):
    """oracle's arrays without a Python dict, for sets of 10^7-10^8 pairs: a stable sort by hash groups every key's
    rows ascending, np.unique's first occurrences give the keys' first-insertion order"""
    h = np.asarray(h, dtype=np.uint64)
    row = np.repeat(np.arange(len(off) - 1, dtype=np.uint32), np.diff(np.asarray(off, dtype=np.int64)))
    order = np.argsort(h, kind="stable")
    hs = h[order]
    uniq, first, counts = np.unique(hs, return_index=True, return_counts=True)
    first_flat = order[first]                                  # flat position of each key's first element
    key_order = np.argsort(first_flat, kind="stable")
    hashes = uniq[key_order]
    sizes = counts[key_order]
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    starts = first[key_order]
    take = np.repeat(starts - np.concatenate([[0], np.cumsum(sizes)[:-1]]), sizes) + np.arange(len(h))
    idx = row[order[take]]
    return hashes, offsets, idx


def text_of_keys(hashes, offsets, idx, k0, k1, n_keys):
    "the member's text of keys [k0, k1) as the chunks carry it: the opening brace at key 0, the closing one at n_keys"
    parts = []
    for k in range(k0, k1):
        a, b = int(offsets[k]), int(offsets[k + 1])
        parts.append('"%d": [%s]' % (int(hashes[k]), ", ".join(str(x) for x in idx[a:b].tolist())))
    text = ", ".join(parts)
    if k0 > 0:
        text = ", " + text
    return (("{" if k0 == 0 else "") + text + ("}" if k1 == n_keys else "")).encode()


def random_rows(rng, n_rows=40, pool=600):
    """rows over one pool of hashes: some hashes in many rows, many in none, empty rows, one row with every hash that
    any row holds, 0 and UINT64_MAX, more than 8 rows so that idx lists reach past 7"""
    values = rng.integers(1, U64_MAX, size=pool, dtype=np.uint64)
    values[:2] = [0, U64_MAX]
    popular = values[:20]
    rows = []
    for r in range(n_rows):
        kind = rng.random()
        if kind < 0.1:
            rows.append(np.zeros(0, np.uint64))
            continue
        n = int(rng.integers(1, 80))
        row = rng.choice(values[: pool // 2], size=n, replace=False)          # the other half is in no row
        if kind < 0.6:
            row = np.concatenate([row, popular[rng.random(len(popular)) < 0.7]])
        rows.append(np.unique(row))
    everything = np.unique(np.concatenate(rows))
    rows.insert(int(rng.integers(0, n_rows)), everything)
    return rows


def csr(rows):
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint64)
    h = np.concatenate(rows) if rows else np.zeros(0, np.uint64)
    return np.ascontiguousarray(h, dtype=np.uint64), off


def skewed_rows(seed, n_rows, n_pairs):
    """A GTDB-sized synthetic set (seeded): n_rows genomes, about n_pairs (hash, genome) pairs, ascending rows.  Row
    sizes are log-normal; a quarter of each row's hashes come from a shared pool drawn with a Zipf-like skew, so a
    few hashes are held by thousands of genomes and most by one."""
    rng = np.random.default_rng(seed)
    sizes = rng.lognormal(0.0, 0.6, size=n_rows)
    sizes = np.maximum((sizes / sizes.sum() * n_pairs).astype(np.int64), 1)
    pool = rng.integers(0, U64_MAX, size=max(n_pairs // 40, 1000), dtype=np.uint64, endpoint=True)
    pool[:2] = [0, U64_MAX]
    weights = 1.0 / np.arange(1, len(pool) + 1) ** 1.1
    weights /= weights.sum()
    total = int(sizes.sum())
    shared = rng.choice(pool, size=total // 4, p=weights)
    own = rng.integers(0, U64_MAX, size=total - len(shared), dtype=np.uint64, endpoint=True)
    flat = np.concatenate([shared, own])
    rng.shuffle(flat)
    row = np.repeat(np.arange(n_rows, dtype=np.int64), sizes)
    # sort by (row, hash) and drop repeats within a row
    order = np.lexsort((flat, row))
    flat, row = flat[order], row[order]
    keep = np.ones(len(flat), bool)
    keep[1:] = (flat[1:] != flat[:-1]) | (row[1:] != row[:-1])
    flat, row = flat[keep], row[keep]
    off = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n_rows))]).astype(np.uint64)
    return flat, off
