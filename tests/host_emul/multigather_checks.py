"""batch.multigather / gather.gather_many end to end with the EMULATED build (emul_lib.py), against a brute force of
the reference's per-query gather loop (CounterGather + GatherDatabases: index/__init__.py:777-909,
search.py:877-949) and against gather_databases for one query at a time.  Run as a script by
tests/test_multigather_emulated.py.

    python tests/host_emul/multigather_checks.py [name ...]
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emulated_boot  # noqa: E402

LIB = emulated_boot.install()

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402
from tests.multigather_cases import NONE, brute_multigather  # noqa: E402
from tests.multigather_cases import assert_same as _assert_same, workload as _workload  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


@check
def multigather_vs_bruteforce():
    rows, queries = _workload()
    db = B.SketchSet.from_rows(rows)
    thresholds = [5, 1, 1, 3, 1, 40]
    min_counts = [1, 1, 1, 8, 1, 30]
    got = B.multigather(queries, db, thresholds, min_counts)
    for i, q in enumerate(queries):
        _assert_same(got[i], brute_multigather(q, rows, thresholds[i], min_counts[i]), i)
    assert len(got[0][0]) >= 4 and 17 not in got[0][0].tolist()
    assert len(got[1][0]) == 0 and (got[1][2] == NONE).all()
    assert (got[2][2] != NONE).all()
    ids, sizes = B.gather(queries[0], db, threshold=5)                 # the single-query device loop agrees
    assert ids.tolist() == got[0][0].tolist() and sizes.tolist() == got[0][1].tolist()
    capped = B.multigather(queries, db, thresholds, min_counts, max_rounds=2)
    for i, q in enumerate(queries):
        _assert_same(capped[i], brute_multigather(q, rows, thresholds[i], min_counts[i], max_rounds=2), ("cap", i))
    assert B.multigather([], db) == []
    empty = B.multigather([np.zeros(0, np.uint64), queries[0]], B.SketchSet.from_rows([]))
    assert [len(r[0]) for r in empty] == [0, 0]


@check
def multigather_grouping_and_fallbacks():
    rows, queries = _workload()
    db = B.SketchSet.from_rows(rows)
    want = B.multigather(queries, db, 3, 2)
    os.environ["SMB_MULTIGATHER_GROUP_BYTES"] = "2000"                 # one or two queries per group
    try:
        small = B.multigather(queries, db, 3, 2)
    finally:
        del os.environ["SMB_MULTIGATHER_GROUP_BYTES"]
    for a, b in zip(want, small):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    for i, q in enumerate(queries):
        _assert_same(want[i], brute_multigather(q, rows, 3, 2), i)
    db.build_index()                                                   # indexed set: the session loop, query by query
    got = B.multigather(queries, db, 3, 2)
    for i, q in enumerate(queries):
        _assert_same(got[i], brute_multigather(q, rows, 3, 2), ("index", i))
    # candidate rows too large for the shared-memory table: that query takes the session loop, the others stay batched
    rng = np.random.Generator(np.random.PCG64(21))
    big = np.unique(rng.integers(1, 2**62, size=34_000, dtype=np.uint64))
    rows2 = rows[:60] + [big]
    db2 = B.SketchSet.from_rows(rows2)
    qs2 = [np.unique(np.concatenate([big[::2], rows[3]])), queries[0]]
    got = B.multigather(qs2, db2, [1, 5])
    _assert_same(got[0], brute_multigather(qs2[0], rows2, 1), "large rows")
    _assert_same(got[1], brute_multigather(qs2[1], rows2, 5), "beside large rows")


@check
def multigather_launches_follow_rounds():
    rows, queries = _workload()
    db = B.SketchSet.from_rows(rows)
    qs = [queries[i % len(queries)] for i in range(32)]
    st_all, st_one = {}, {}
    got = B.multigather(qs, db, stats=st_all)
    slowest = max(range(len(qs)), key=lambda i: len(got[i][0]))
    B.multigather([qs[slowest]], db, stats=st_one)
    assert st_all["round_launches"] > 0
    assert st_all["round_launches"] <= st_one["round_launches"] + 3 * 16, (st_all, st_one)


@check
def multigather_range_major_prefetch():
    "a query too large for the shared-memory table: its first counters come from the range-major pass"
    rows, queries = _workload()
    db = B.SketchSet.from_rows(rows)
    rng = np.random.Generator(np.random.PCG64(31))
    large = np.unique(np.concatenate([rng.integers(1, 2**54, size=40_000, dtype=np.uint64)] + rows[:30]))
    os.environ["SMB_RM_RANGES"] = "7"
    try:
        got = B.multigather([large, queries[0]], db, [2, 5])
    finally:
        del os.environ["SMB_RM_RANGES"]
    _assert_same(got[0], brute_multigather(large, rows, 2), "large query")
    _assert_same(got[1], brute_multigather(queries[0], rows, 5), "small query")


@check
def gather_many_equals_gather_databases():
    import sourmash_b200 as smb
    from sourmash_b200.gather import gather_databases, gather_many
    rng = np.random.Generator(np.random.PCG64(41))
    scaled = 10
    mx = B.max_hash_for_scaled(scaled)
    pool = np.unique(rng.integers(1, mx, size=3000, dtype=np.uint64))
    rows = []
    for i in range(40):
        own = rng.choice(pool, size=int(rng.integers(20, 300)), replace=False)
        extra = np.unique(rng.integers(1, mx, size=int(rng.integers(10, 100)), dtype=np.uint64))
        rows.append(np.unique(np.concatenate([own, extra])))
    rows[7] = rows[3].copy()
    db = B.SketchSet.from_rows(rows)
    names = ["g%d" % i for i in range(len(rows))]
    md5s = ["%032x" % (i * 7919) for i in range(len(rows))]
    mhs = []
    for k, track in enumerate((False, True, True, False)):
        q = rng.choice(pool, size=int(rng.integers(400, 1500)), replace=False)
        mh = smb.MinHash(0, 31, scaled=scaled, track_abundance=track)
        if track:
            mh.set_abundances({int(h): int(a) for h, a in zip(q, rng.integers(1, 30, size=len(q)))})
        else:
            mh.add_many(q)
        mhs.append(mh)
    mhs.append(smb.MinHash(0, 31, scaled=scaled))                       # empty query
    for threshold_bp in (0, 300):
        for ignore_abundance in (False, True):
            kw = dict(threshold_bp=threshold_bp, ignore_abundance=ignore_abundance, names=names, md5s=md5s)
            many = gather_many(mhs, db, query_names=["q%d" % i for i in range(len(mhs))], **kw)
            for i, mh in enumerate(mhs):
                one = gather_databases(mh, db, query_name="q%d" % i, **kw)
                assert many[i] == one, (threshold_bp, ignore_abundance, i)
            assert sum(len(x) for x in many) > 10
    # queries at two scaled values: each compared against its own downsampled copy of the database
    coarse = mhs[1].downsample(scaled=40)
    many = gather_many([mhs[0], coarse, mhs[2]], db, threshold_bp=0, names=names)
    assert many[0] == gather_databases(mhs[0], db, names=names)
    assert many[1] == gather_databases(coarse, db.downsample(B.max_hash_for_scaled(40)), names=names)
    assert many[2] == gather_databases(mhs[2], db, names=names)
    assert len(many[1]) > 0


def main(names):
    names = names or list(CHECKS)
    for name in names:
        t0 = time.time()
        CHECKS[name]()
        print("ok  %-36s %.1f s" % (name, time.time() - t0), flush=True)
    print("multigather checks passed (%s)" % os.path.basename(LIB))


if __name__ == "__main__":
    main(sys.argv[1:])
