"""batch.query_covered (query_cover_kernel) and `b200prefetch --save-matching-hashes / --save-unmatched-hashes` with the
EMULATED build (emul_lib.py), against np.isin over the listed rows and the reference's per-match loop written with this
package's MinHash.  Run as a script by tests/test_query_cover_emulated.py (and on the device by
tests/test_gpu_query_cover.py).

    python tests/host_emul/query_cover_checks.py [--device] [name ...]
"""
import contextlib
import io
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
if "--device" in sys.argv:
    sys.argv.remove("--device")
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
else:
    import emulated_boot  # noqa: E402
    emulated_boot.install()

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402

CHECKS = {}
U64_MAX = np.uint64(2**64 - 1)


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def _want(q, rows, listed):
    held = np.concatenate([rows[i] for i in listed]) if len(listed) else np.zeros(0, np.uint64)
    return np.isin(q, held)


def _same(q, rows, listed, tag):
    got = B.query_covered(q, B.SketchSet.from_rows(rows), listed)
    want = _want(q, rows, listed)
    assert got.dtype == np.bool_ and got.shape == (len(q),), (tag, got.dtype, got.shape)
    bad = np.nonzero(got != want)[0]
    assert not len(bad), (tag, bad[:5].tolist(), q[bad[:5]].tolist())
    return got


@check
def query_cover_edge_cases():
    rng = np.random.default_rng(7)
    pool = np.unique(rng.integers(1, 2**62, size=20_000, dtype=np.uint64))
    q = np.sort(rng.choice(pool, size=3_000, replace=False))
    rows = [np.sort(rng.choice(pool, size=int(n), replace=False)) for n in (1, 31, 33, 64, 100, 127, 129, 1000, 4001)]
    rows += [np.zeros(0, np.uint64), np.zeros(0, np.uint64)]
    every = list(range(len(rows)))
    _same(q, rows, every, "all rows, lengths not multiples of 32, empty rows")
    _same(q, rows, [len(rows) - 1], "only an empty row")
    _same(q, rows, [], "empty row list")
    _same(q, rows, [3, 3, 5, 3], "a row listed twice")
    _same(np.zeros(0, np.uint64), rows, every, "empty query")
    _same(q[:1], rows + [q[:1].copy()], [len(rows), 0], "one-hash query")
    far = [np.arange(2**63, 2**63 + 500, dtype=np.uint64), np.arange(1, 400, dtype=np.uint64)]
    _same(q[q > 1000], far, [0, 1], "rows outside the query's key range")
    qm = np.concatenate([q, [U64_MAX]])
    got = _same(qm, [np.array([U64_MAX], np.uint64), rows[1], np.array([5, U64_MAX], np.uint64)], [0, 1, 2],
                "a query holding UINT64_MAX")
    assert got[-1]
    got = _same(qm, [rows[1]], [0], "UINT64_MAX in the query, padding lanes of a 31-hash row")
    assert not got[-1]
    dense = np.arange(1, 70_000, dtype=np.uint64)
    _same(dense[::3], [dense[::2], dense[5:9000]], [0, 1], "dense small keys")


@check
def query_cover_errors():
    rows = [np.arange(1, 50, dtype=np.uint64), np.arange(10, 90, dtype=np.uint64)]
    sset = B.SketchSet.from_rows(rows)
    q = np.arange(5, 60, dtype=np.uint64)
    for listed in ([2], [0, 1, 7], [2**31]):
        try:
            B.query_covered(q, sset, listed)
            raise AssertionError("accepted row list %r" % (listed,))
        except Exception as exc:                        # noqa: BLE001 -- the message is what is checked
            assert "out of range" in str(exc), str(exc)
    for listed in ([-1], [2**32]):
        try:
            B.query_covered(q, sset, listed)
            raise AssertionError("accepted row list %r" % (listed,))
        except ValueError as exc:
            assert "out of range" in str(exc), str(exc)
    try:
        B.query_covered(q[::-1].copy(), sset, [0])
        raise AssertionError("accepted an unsorted query")
    except Exception as exc:                            # noqa: BLE001
        assert "sorted" in str(exc), str(exc)
    before = B.kernel_launches()
    assert not B.query_covered(q, sset, []).any()
    assert len(B.query_covered(np.zeros(0, np.uint64), sset, [0, 1])) == 0
    assert B.kernel_launches() == before


def _sig_file(d, name, hashes, abunds=None, scaled=10, sig_name=""):
    from sourmash_b200.minhash import MinHash
    from sourmash_b200.signature import SourmashSignature, save_signatures_to_json
    mh = MinHash(0, 31, scaled=scaled, track_abundance=abunds is not None)
    if abunds is None:
        mh.add_many(hashes)
    else:
        mh.set_abundances(dict(zip(hashes.tolist(), abunds.tolist())))
    path = os.path.join(d, name)
    with open(path, "w") as fp:
        save_signatures_to_json([SourmashSignature(mh, name=sig_name)], fp)
    return path


def _reference_split(query_mh, matches, threshold_bp):
    """commands.py:1602-1622 restated: ident_mh += query & match, noident_mh.remove_many(match), match by match, for
    every database sketch whose overlap reaches the threshold; both flat, at the query's scaled (one scaled here)"""
    flat = query_mh.flatten()
    ident, noident = flat.copy_and_clear(), flat.copy_and_clear()
    noident.merge(flat)
    for m in matches:
        common = flat & m.flatten()
        if len(common) * flat.scaled >= threshold_bp and len(common):
            ident.merge(common)
            noident.remove_many(m)
    return ident, noident


@check
def prefetch_saves_the_reference_split():
    from sourmash_b200 import plugin
    from sourmash_b200.signature import load_signatures_from_json
    rng = np.random.default_rng(3)
    max_hash = np.uint64((2**64 - 1) // 10)
    pool = np.unique(rng.integers(1, int(max_hash), size=30_000, dtype=np.uint64))
    q = np.sort(rng.choice(pool, size=5_000, replace=False))
    qa = rng.integers(1, 9, size=len(q)).astype(np.uint64)
    with tempfile.TemporaryDirectory() as d:
        dbs = []
        for i in range(12):
            k = int(rng.integers(0, 900)) if i % 3 else 0
            h = np.unique(np.concatenate([rng.choice(q, size=k, replace=False), rng.choice(pool, size=800)]))
            dbs.append(_sig_file(d, "db%d.sig" % i, h, sig_name="g%d" % i))
        for abund in (False, True):
            qpath = _sig_file(d, "q.sig", q, qa if abund else None, sig_name="meta")
            query = list(load_signatures_from_json(qpath))[0]
            matches = [list(load_signatures_from_json(p))[0].minhash for p in dbs]
            for thr in (3000.0, 0.0, 40000.0):
                out = {k: os.path.join(d, "%s.sig" % k) for k in ("known", "unknown")}
                argv = ["b200prefetch", qpath] + dbs + ["--threshold-bp", str(thr), "-q",
                                                        "--save-matching-hashes", out["known"],
                                                        "--save-unmatched-hashes", out["unknown"] + ".gz"]
                with contextlib.redirect_stderr(io.StringIO()):
                    assert plugin.main(argv) == 0
                ident, noident = _reference_split(query.minhash, matches, max(thr, 1))
                got = {k: list(load_signatures_from_json(p))[0] for k, p in (("known", out["known"]),
                                                                        ("unknown", out["unknown"] + ".gz"))}
                for tag, want in (("known", ident), ("unknown", noident)):
                    g = got[tag]
                    assert g.name == "meta-" + tag, (g.name, tag)
                    assert np.array_equal(g.minhash._mins_array(), want._mins_array()), (abund, thr, tag)
                    assert g.minhash.track_abundance == abund, (abund, tag)
                    if abund:
                        pos = np.searchsorted(q, g.minhash._mins_array())
                        assert np.array_equal(g.minhash._abunds_array(), qa[pos]), (thr, tag)
                assert len(got["known"].minhash) + len(got["unknown"].minhash) == len(q)
                if thr == 40000.0:
                    assert len(got["known"].minhash) == 0


if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        CHECKS[name]()
        print("ok  " + name, flush=True)
    print("query_cover checks passed")
