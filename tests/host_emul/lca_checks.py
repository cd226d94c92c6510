"""batch.lca_table / batch.lca_counts and the lca module with the EMULATED build (emul_lib.py), against the oracle of
tests/lca_cases.py (the reference's gather_assignments + count_lca_for_assignments restated).  Run as a script by
tests/test_lca_emulated.py; tests/test_gpu_lca.py runs the same checks on the device.

    python tests/host_emul/lca_checks.py [name ...]
"""
import gzip
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    import emulated_boot  # noqa: E402
    emulated_boot.install()

import numpy as np  # noqa: E402

from tests import lca_cases as C  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def _compare(dbs, queries, weights=None, tag=""):
    got, _, _ = C.device_counts(dbs, queries, weights)
    for i, q in enumerate(queries):
        want = C.oracle_counts(q, dbs, None if weights is None else weights[i])
        assert got[i] == want, (tag, i, got[i][:5], want[:5])


@check
def lca_fixtures():
    "the reference's LCA databases, each alone and all together, queried with their own hashes and the TARA sketches"
    from sourmash_b200.signature import load_signatures_from_json
    dbs = C.fixture_dbs()
    queries = []
    for name in sorted(os.listdir(C.FIXTURES)):
        if name.endswith(".sig.gz"):
            with gzip.open(os.path.join(C.FIXTURES, name), "rt") as fh:
                for sig in load_signatures_from_json(fh.read(), ksize=31):
                    queries.append(np.array(sorted(sig.minhash.hashes), dtype=np.uint64))
    for db in dbs:
        queries.append(np.array(sorted(db[0])[:500], dtype=np.uint64))
    for i in range(len(dbs)):
        _compare([dbs[i]], queries, tag="fixture %d" % i)
    _compare(dbs, queries, tag="all fixtures")
    weights = [np.arange(1, len(q) + 1, dtype=np.uint64) % 7 + 1 for q in queries]
    _compare(dbs, queries, weights, tag="weighted")


@check
def lca_random_tries():
    """random tries with empty middle ranks, all-empty lineages and superkingdom disagreements; idx without lid; hashes
    in several databases with equal and different lineages; UINT64_MAX and 0; empty queries; many queries per batch"""
    for seed in range(4):
        rng = np.random.default_rng(seed)
        dbs, pool = C.random_dbs(rng)
        queries = [np.unique(rng.choice(pool, size=int(rng.integers(0, 400)), replace=False)) for _ in range(60)]
        queries[0] = np.zeros(0, np.uint64)
        queries[1] = np.array([0, 1, 2**64 - 1], dtype=np.uint64)
        queries[2] = np.unique(pool)
        _compare(dbs, queries, tag="random %d" % seed)
        weights = [rng.integers(1, 100, size=len(q)).astype(np.uint64) for q in queries]
        _compare(dbs, queries, weights, tag="random weighted %d" % seed)


@check
def lca_same_hash_two_databases():
    "one hash in two databases: equal lineages fold to that lineage, a prefix to the deeper one, a branch to the fork"
    a = ("A", "B", "C", "", "", "", "", "")
    cases = [(a, a, a), (a, ("A", "B", "", "", "", "", "", ""), a),
             (a, ("A", "X", "C", "", "", "", "", ""), ("A",)), (a, ("Z",) + ("",) * 7, ()),
             (a, ("",) * 8, a), (("",) * 8, ("",) * 8, ())]
    for l1, l2, want in cases:
        dbs = [({7: [0]}, {0: l1}), ({7: [3]}, {3: l2})]
        got, _, _ = C.device_counts(dbs, [np.array([7], np.uint64)])
        assert got[0] == C.oracle_counts([7], dbs), (l1, l2, got)
        assert [n for _, n in got[0][0][0]] == [x for x in want if x], (l1, l2, got, want)


@check
def lca_empty_inputs():
    "an empty database gives an empty table and no rows; an empty batch gives no rows; idx without lid: no entry"
    from sourmash_b200 import batch as B
    got, table, _ = C.device_counts([({}, {})], [np.array([1, 2], np.uint64)])
    assert len(table) == 0 and got == [[]]
    got, table, _ = C.device_counts([({5: [1]}, {0: ("A",) + ("",) * 7})], [np.array([5], np.uint64)])
    assert len(table) == 0 and got == [[]]
    _, table, _ = C.device_counts([({5: [0]}, {0: ("A",) + ("",) * 7})], [])
    assert len(table) == 1
    q, n, c, f = B.lca_counts(table, np.zeros(0, np.uint64), np.zeros(1, np.uint64))
    assert len(q) == len(n) == len(c) == len(f) == 0
    before = B.kernel_launches()
    B.lca_counts(table, np.zeros(0, np.uint64), np.zeros(4, np.uint64))
    assert B.kernel_launches() == before


@check
def lca_cut_at_max_hash():
    "hashes above max_hash leave the table, as downsample_scaled removes them"
    from sourmash_b200 import batch as B
    h = np.array([10, 20, 30, 2**64 - 1], dtype=np.uint64)
    t = B.lca_table(h, np.array([1, 1, 1, 1], np.uint32), [0, 0], [0, 1], max_hash=20)
    assert t.to_host()[0].tolist() == [10, 20]
    t = B.lca_table(h, np.array([1, 1, 1, 1], np.uint32), [0, 0], [0, 1])
    assert t.to_host()[0].tolist() == h.tolist()


@check
def lca_argument_errors():
    "node indices, the trie's shape, a trie without nodes and decreasing offsets are refused before any launch"
    from sourmash_b200 import batch as B
    h = np.array([1, 2], dtype=np.uint64)
    bad = [(lambda: B.lca_table(h, [0, 5], [0, 0], [0, 1]), "out of range"),
           (lambda: B.lca_table(h, [0, 1], [], []), "no nodes"),
           (lambda: B.lca_table(h, [0, 1], [0, 1], [0, 1]), "parent below it"),
           (lambda: B.lca_table(h, [0, 1], [0, 0], [0, 2]), "parent below it"),
           (lambda: B.lca_table(h, [0, 1], [0, 0], [1, 2]), "root")]
    t = B.lca_table(h, [1, 1], [0, 0], [0, 1])
    bad.append((lambda: B.lca_counts(t, h, np.array([0, 2, 1, 2], np.uint64)), "decrease"))
    for fn, msg in bad:
        before = B.kernel_launches()
        try:
            fn()
            raise AssertionError("accepted: " + msg)
        except AssertionError:
            raise
        except Exception as exc:                                   # noqa: BLE001
            assert msg in str(exc), (msg, str(exc))
        assert B.kernel_launches() == before, msg


@check
def lca_database_loading():
    "LcaDatabase.load: .lca.json and .lca.json.gz give the same arrays as json; the reference's errors"
    import json
    import tempfile
    from sourmash_b200 import lca as L
    d = C.unpack_fixtures(tempfile.mkdtemp())
    for name in C.DATABASES:
        db = L.LcaDatabase.load(os.path.join(d, name))
        with open(os.path.join(d, name)) as fh:
            pairs = [(int(k), x) for k, v in json.load(fh)["hashval_to_idx"].items() for x in v]
        assert list(zip(db.hashes.tolist(), db.idx.tolist())) == pairs, name
        gz = L.LcaDatabase.load(os.path.join(C.FIXTURES, name + ".gz"))
        assert np.array_equal(gz.hashes, db.hashes) and gz.lid_to_lineage == db.lid_to_lineage, name
    for path, msg in ((d, "is not a file"), (os.path.join(d, "TARA_ASE_MAG_00031.sig"), "is not an LCA database file."),
                      (os.path.join(d, "old-db-format-1.json"), "old-style LCA DB")):
        try:
            L.LcaDatabase.load(path)
            raise AssertionError("loaded " + path)
        except ValueError as exc:
            assert msg in str(exc), (msg, str(exc))


if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        CHECKS[name]()
        print("ok  " + name, flush=True)
    print("lca checks passed")
