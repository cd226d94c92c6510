"""batch.many_vs_many, the multigather first pass built on it, and LinearIndex.search_many / prefetch_many end to end
with the EMULATED build (emul_lib.py), against a brute force with np.intersect1d and against the one-query calls.
Run as a script by tests/test_many_vs_many_emulated.py.

    python tests/host_emul/many_vs_many_checks.py [name ...]
"""
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emulated_boot  # noqa: E402

LIB = emulated_boot.install()
os.environ["SMB_RM_RANGES"] = "5"              # few key ranges: the emulator runs every CTA of the pass on the CPU

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402
from tests.many_vs_many_cases import brute, cases  # noqa: E402
from tests.multigather_cases import brute_multigather  # noqa: E402
from tests.multigather_cases import assert_same as _assert_same, workload as _workload  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def assert_counts(got, queries, rows, what):
    want = brute(queries, rows)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.array_equal(got, want), (what, np.argwhere(got != want)[:5].tolist())
    stacked = np.stack([B.one_vs_many(q, B.SketchSet.from_rows(rows)) for q in queries]) if queries else got
    assert np.array_equal(got, stacked), what


@check
def many_vs_many_equals_stacked_one_vs_many():
    rows, qs = cases()
    db = B.SketchSet.from_rows(rows)
    assert_counts(B.many_vs_many(qs, db), qs, rows, "default")
    assert B.many_vs_many([], db).shape == (0, len(rows))
    assert B.many_vs_many(qs[:3], B.SketchSet.from_rows([])).shape == (3, 0)
    assert_counts(B.many_vs_many([qs[0]], db), [qs[0]], rows, "one query")
    assert_counts(B.many_vs_many([qs[3], qs[3]], db), [qs[3], qs[3]], rows, "empty queries")
    # a database of near-copies of the queries: every element a match, the queues overflow and drain
    near = [np.setdiff1d(qs[i % 3], qs[i % 3][i::17]) for i in range(40)]
    assert_counts(B.many_vs_many(qs[:3] + [qs[4]], B.SketchSet.from_rows(near)), qs[:3] + [qs[4]], near, "near copies")
    # the device form: hashes and counters in (emulated) device memory, offsets on the host
    hashes, offs = B._query_csr(qs)
    out = np.full((len(qs), len(rows)), 7, dtype=np.uint32)
    B.many_vs_many_device(hashes.ctypes.data, offs, db, out.ctypes.data)
    assert_counts(out, qs, rows, "device form")


@check
def many_vs_many_paths_and_grouping():
    rows, qs = cases()
    want = brute(qs, rows)
    n = len(rows)
    for budget in (1, n * 4 * 2 + 12 * 900, n * 4 * 3 + 12 * 2000):           # one query per group, then small groups
        os.environ["SMB_MANY_VS_MANY_GROUP_BYTES"] = str(budget)
        try:
            got = B.many_vs_many(qs, B.SketchSet.from_rows(rows))
        finally:
            del os.environ["SMB_MANY_VS_MANY_GROUP_BYTES"]
        assert np.array_equal(got, want), budget
    os.environ["SMB_SEARCH_LAYOUT"] = "global"
    try:
        assert np.array_equal(B.many_vs_many(qs, B.SketchSet.from_rows(rows)), want), "global layout"
    finally:
        del os.environ["SMB_SEARCH_LAYOUT"]
    db = B.SketchSet.from_rows(rows)
    db.build_index()
    assert np.array_equal(B.many_vs_many(qs, db), want), "indexed set"
    del os.environ["SMB_RM_RANGES"]                                            # the product's number of ranges
    try:
        assert np.array_equal(B.many_vs_many(qs[:5], B.SketchSet.from_rows(rows)), want[:5]), "default ranges"
    finally:
        os.environ["SMB_RM_RANGES"] = "5"


@check
def many_vs_many_launches_do_not_grow_with_queries():
    rows, qs = cases()
    db = B.SketchSet.from_rows(rows)
    B.many_vs_many(qs[:2], db)                                                 # builds the range-major copy

    def launches(queries):
        k0 = B.kernel_launches()
        B.many_vs_many(queries, db)
        return B.kernel_launches() - k0
    few, many = launches(qs[5:7]), launches([qs[(5, 6, 8)[i % 3]] for i in range(48)])   # one group either way
    assert 0 < few == many <= 4, (few, many)


@check
def many_vs_many_rejects_bad_input():
    from sourmash_b200._lowlevel import ffi, lib
    from sourmash_b200.exceptions import SourmashError
    rows, qs = cases()
    db = B.SketchSet.from_rows(rows)

    def raises(msg, fn):
        try:
            fn()
        except SourmashError as e:
            assert msg in str(e), (msg, str(e))
            return
        raise AssertionError("no error: " + msg)
    raises("every query must be sorted and unique", lambda: B.many_vs_many([qs[0], qs[0][::-1].copy()], db))
    raises("every query must be sorted and unique", lambda: B.many_vs_many([np.array([3, 3], np.uint64)], db))
    h = np.concatenate([qs[0], qs[4]])
    out = np.zeros((2, len(rows)), np.uint32)
    for offs, msg in (([1, 5, 9], "query offsets must start at 0"), ([0, 9, 5], "query offsets must not decrease")):
        o = np.array(offs, np.uint64)
        raises(msg, lambda: B.rustcall(lib.smb_many_vs_many, ffi.cast("uint64_t *", h.ctypes.data),
                                       ffi.cast("uint64_t *", o.ctypes.data), 2, db._ptr,
                                       ffi.cast("uint32_t *", out.ctypes.data)))
        raises(msg, lambda: B.many_vs_many_device(h.ctypes.data, o, db, out.ctypes.data))
    bad = np.concatenate([qs[0], qs[4][::-1]])                                 # unsorted, found on the device
    offs = np.array([0, len(qs[0]), len(bad)], np.uint64)
    raises("every query must be sorted and unique", lambda: B.many_vs_many_device(bad.ctypes.data, offs, db, out.ctypes.data))


@check
def multigather_first_pass_is_batched():
    rows, queries = _workload()
    db = B.SketchSet.from_rows(rows)
    thresholds = [5, 1, 1, 3, 1, 40]
    min_counts = [1, 1, 1, 8, 1, 30]
    got = B.multigather(queries, db, thresholds, min_counts)
    for i, q in enumerate(queries):
        _assert_same(got[i], brute_multigather(q, rows, thresholds[i], min_counts[i]), i)
    os.environ["SMB_MANY_VS_MANY_GROUP_BYTES"] = str(len(rows) * 4 * 2 + 12 * 1500)
    try:
        small = B.multigather(queries, db, thresholds, min_counts)
    finally:
        del os.environ["SMB_MANY_VS_MANY_GROUP_BYTES"]
    for i, q in enumerate(queries):
        _assert_same(small[i], brute_multigather(q, rows, thresholds[i], min_counts[i]), ("groups", i))


def _sigs():
    "subjects at scaled 10 (with one duplicate and one empty), queries at finer, equal and coarser scaled"
    import sourmash_b200 as smb
    rng = np.random.Generator(np.random.PCG64(61))
    mx = B.max_hash_for_scaled(5)
    pool = np.unique(rng.integers(1, mx, size=4000, dtype=np.uint64))

    def mh(hashes, scaled, **kw):
        m = smb.MinHash(0, 31, scaled=scaled, **kw)
        m.add_many(hashes)
        return m
    subjects = []
    for i in range(30):
        own = rng.choice(pool, size=int(rng.integers(30, 400)), replace=False)
        subjects.append(smb.SourmashSignature(mh(own, 10), name="s%d" % i))
    subjects[9] = smb.SourmashSignature(subjects[4].minhash.copy(), name="s9")
    subjects[13] = smb.SourmashSignature(mh([], 10), name="s13")
    queries = []
    for i, scaled in enumerate((5, 10, 20, 10, 40, 5)):
        q = rng.choice(pool, size=int(rng.integers(300, 1500)), replace=False)
        queries.append(smb.SourmashSignature(mh(q, scaled), name="q%d" % i))
    queries.append(smb.SourmashSignature(subjects[4].minhash.copy(), name="same"))
    return smb, subjects, queries


def _key(results):
    return [[(r.score, r.signature.md5sum(), r.location) for r in res] for res in results]


def _outcome(fn):
    try:
        return ("ok", _key(fn()))
    except Exception as e:                                                      # noqa: BLE001 -- compared, not hidden
        return ("raised", type(e), str(e))


def _compare_index(idx, queries, what):
    modes = [dict(threshold=0.0), dict(threshold=0.05, do_containment=True), dict(threshold=0.0, do_max_containment=True),
             dict(threshold=0.0, best_only=True), dict(threshold=0.1)]
    outcomes = []
    for kw in modes:
        many = _outcome(lambda: idx.search_many(queries, **kw))
        one = _outcome(lambda: [idx.search(q, **kw) for q in queries])
        assert many == one, (what, kw, many[:2], one[:2])
        outcomes.append(many)
    for bp in (0, 100, 3000):                                    # 3000 bp: unattainable for some queries, raises
        many = _outcome(lambda: idx.prefetch_many(queries, bp))
        one = _outcome(lambda: [list(idx.prefetch(q, bp)) for q in queries])
        assert many == one, (what, bp, many[:2], one[:2])
        outcomes.append(many)
    return outcomes[0]


@check
def search_many_and_prefetch_many_equal_per_query_calls():
    from sourmash_b200.index import LinearIndex, ZipFileLinearIndex
    from sourmash_b200.signature import save_signatures_to_json
    from tests.test_zip_collections import make_zip_deflated
    smb, subjects, queries = _sigs()
    lin = LinearIndex(subjects)
    res = _compare_index(lin, queries, "linear")
    assert res[0] == "ok" and sum(len(r) for r in res[1]) > 20
    with tempfile.TemporaryDirectory() as td:
        members = []
        for i, s in enumerate(subjects):
            p = os.path.join(td, "s%d.sig" % i)
            with open(p, "w") as fp:
                save_signatures_to_json([s], fp)
            members.append(("signatures/s%d.sig" % i, p))
        zidx = ZipFileLinearIndex.load(make_zip_deflated(os.path.join(td, "db.zip"), members))
        _compare_index(zidx, queries, "zip")
    # queries the batched pass leaves to the per-query path: an abundance query, an incompatible ksize (errors at the
    # same query as the per-query calls), num sketches; an empty index
    ab = smb.MinHash(0, 31, scaled=10, track_abundance=True)
    ab.set_abundances({int(h): 2 for h in queries[1].minhash.hashes})
    k21 = smb.MinHash(0, 21, scaled=10)
    k21.add_many(list(queries[1].minhash.hashes)[:50])
    for extra in (smb.SourmashSignature(ab, name="abund"), smb.SourmashSignature(k21, name="k21")):
        out = _compare_index(lin, [queries[0], extra, queries[2]], extra.name)
        assert out[0] == "raised", (extra.name, out)
    nums = []
    rng = np.random.Generator(np.random.PCG64(62))
    for i in range(8):
        m = smb.MinHash(50, 31)
        m.add_many(rng.integers(1, 2**63, size=int(rng.integers(10, 200)), dtype=np.uint64).tolist() + list(range(1, 40)))
        nums.append(smb.SourmashSignature(m, name="n%d" % i))
    out = _compare_index(LinearIndex(nums), nums[:3], "num")
    mixed = _compare_index(LinearIndex(subjects[:5] + nums[:2]), queries[:2] + nums[:1], "mixed")
    assert mixed[0] == "raised"
    empty = LinearIndex([])
    assert _compare_index(empty, queries[:2], "empty") == ("ok", [[], []])
    assert _outcome(lambda: empty.prefetch_many(queries[:2], 0)) == ("raised", ValueError, "no signatures to search")
    assert empty.search_many([], threshold=0.1) == [] and empty.prefetch_many([], 0) == []
    assert lin.search_many(queries[:2], threshold=0.0)[0] == lin.search(queries[0], threshold=0.0)


def main(names):
    names = names or list(CHECKS)
    for name in names:
        t0 = time.time()
        CHECKS[name]()
        print("ok  %-44s %.1f s" % (name, time.time() - t0), flush=True)
    print("many_vs_many checks passed (%s)" % os.path.basename(LIB))


if __name__ == "__main__":
    main(sys.argv[1:])
