"""Shared cases of the set-operation tests (batch.combine, sigsetops): sketch sets with every edge the combine pass has
to get right, a numpy restatement of the three operations, and the reference's semantics written as a chain of
``MinHash.merge`` calls and Python set operations with this package's MinHash."""
import numpy as np

U64_MAX = np.iinfo(np.uint64).max


def _rows(rng, n, pool, mean, lo=0):
    "n sorted-unique rows drawn from a pool of hashes"
    out = []
    for _ in range(n):
        k = int(min(len(pool), max(lo, rng.poisson(mean))))
        out.append(np.unique(rng.choice(pool, size=k, replace=False)).astype(np.uint64))
    return out


def cases(rng):
    """(tag, rows, abund_rows or None): an empty set, one row, empty rows (row 0 among them), a sketch present twice,
    UINT64_MAX keys, dense small keys, long runs (every row holds most of the pool) and random sparse sets."""
    wide = rng.integers(1, 2**63, size=3000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    out = [("empty set", [], None),
           ("one empty row", [np.zeros(0, np.uint64)], None),
           ("one row", _rows(rng, 1, wide, 200), None)]
    r = _rows(rng, 6, wide[:300], 120)
    out.append(("empty rows", [np.zeros(0, np.uint64)] + r[:3] + [np.zeros(0, np.uint64)] + r[3:], None))
    r = _rows(rng, 5, wide[:200], 80)
    out.append(("same sketch twice", [r[0], r[1], r[0], r[2], r[3], r[4]], None))
    top = np.array([U64_MAX - np.uint64(i) for i in range(40)], np.uint64)
    out.append(("UINT64_MAX keys", _rows(rng, 7, np.concatenate([top, wide[:60]]), 50), None))
    out.append(("dense small keys", _rows(rng, 9, np.arange(1, 65, dtype=np.uint64), 30), None))
    core = wide[:50]
    out.append(("long runs", [np.unique(np.concatenate([core, c])) for c in _rows(rng, 600, wide[50:400], 5)], None))
    out.append(("all rows equal", [core.copy() for _ in range(40)], None))
    for i in range(3):
        n = int(rng.integers(2, 40))
        out.append(("random %d" % i, _rows(rng, n, wide[:int(rng.integers(100, 3000))], float(rng.integers(5, 200))),
                    None))
    with_ab = []
    for tag, rows, _ in out:
        with_ab.append((tag + " +abund", rows, [rng.integers(1, 1000, size=len(x)).astype(np.uint64) for x in rows]))
    return out + with_ab


def csr(rows, abunds=None):
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    h = np.concatenate(rows).astype(np.uint64) if rows else np.zeros(0, np.uint64)
    a = (np.concatenate(abunds).astype(np.uint64) if rows else np.zeros(0, np.uint64)) if abunds is not None else None
    return h, off, a


def numpy_combine(op, rows, abunds=None, num=0):
    "(hashes, abunds or None): np.unique over the whole set, run lengths, np.add.at for the sums"
    h, off, a = csr(rows, abunds)
    keys, inv, cnt = np.unique(h, return_inverse=True, return_counts=True)
    if op == "union":
        keep = np.ones(len(keys), bool)
    elif op == "all":
        keep = cnt == len(rows)
    else:
        row0 = np.zeros(len(keys), bool)
        row0[inv[:int(off[1]) if len(rows) else 0]] = True
        keep = (cnt == 1) & row0
    out = keys[keep]
    sums = None
    if op == "union" and a is not None:
        sums = np.zeros(len(keys), np.uint64)
        np.add.at(sums, inv, a)
        sums = sums[keep]
    if op == "union" and num and len(out) > num:
        out = out[:num]
        sums = sums[:num] if sums is not None else None
    return out, sums


def minhash_of(row, abund=None, *, num=0, scaled=1, ksize=31):
    from sourmash_b200.minhash import MinHash
    mh = MinHash(num, ksize, scaled=0 if num else scaled, track_abundance=abund is not None)
    if abund is not None:
        mh.set_abundances({int(x): int(y) for x, y in zip(row, abund)})
    else:
        mh.add_many([int(x) for x in row])
    return mh


def reference_combine(op, rows, abunds=None, num=0):
    """The reference's loops: `sig merge` as a chain of MinHash.merge into copy_and_clear() of the first sketch,
    `sig intersect` / `sig subtract` as Python sets (sig/__main__.py:459-712)."""
    if not rows:
        return np.zeros(0, np.uint64), None
    mhs = [minhash_of(r, None if abunds is None else abunds[i], num=num) for i, r in enumerate(rows)]
    if op == "union":
        mh = mhs[0].copy_and_clear()
        for m in mhs:
            mh.merge(m)
        got = mh.hashes
        hs = np.array(sorted(got), np.uint64)
        return hs, (np.array([got[int(x)] for x in hs], np.uint64) if abunds is not None else None)
    mins = set(mhs[0].hashes)
    for m in mhs[1:]:
        if op == "all":
            mins.intersection_update(m.hashes)
        else:
            mins -= set(m.hashes)
    return np.array(sorted(mins), np.uint64), None


def assert_same(got, want, tag):
    "(hashes, abunds): equal hashes; equal abundances, where None and an empty array are the same for an empty result"
    assert np.array_equal(got[0], want[0]), (tag, len(got[0]), len(want[0]))
    if len(want[0]) == 0:
        assert got[1] is None or len(got[1]) == 0, tag
        return
    assert (got[1] is None) == (want[1] is None), tag
    if want[1] is not None:
        assert np.array_equal(got[1], want[1]), tag
