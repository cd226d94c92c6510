"""batch.search_angular and LinearIndex / ZipFileLinearIndex.search_abund end to end with the EMULATED build
(emul_lib.py), against the numpy restatement and the reference's per-subject loop of tests/search_abund_cases.py.  Run
as a script by tests/test_search_abund_emulated.py (and on the device by tests/test_gpu_search_abund.py).

    python tests/host_emul/search_abund_checks.py [--device] [name ...]
"""
import os
import sys
import tempfile
import zipfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
if "--device" in sys.argv:
    sys.argv.remove("--device")
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
else:
    import emulated_boot  # noqa: E402
    emulated_boot.install()

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402
from tests import search_abund_cases as C  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def _same_bits(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert not len(bad), (what, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())


@check
def search_angular_edge_cases():
    "every set case against the numpy restatement, bit for bit, and the per-pair MinHash path where it applies"
    for tag, qh, qa, rows, abunds, max_hash in C.set_cases(np.random.default_rng(11)):
        h, off, ab = C.csr(rows, abunds)
        sset = B.SketchSet.from_host(h, off, ab)
        got = B.search_angular(qh, qa, sset, max_hash)
        _same_bits(got, C.numpy_angular(qh, qa, h, off, ab, max_hash), tag)
        if max_hash == C.U64_MAX:                        # no cut: MinHash.angular_similarity of scaled=1 sketches
            q = C.minhash_of(qh, qa, scaled=1)
            want = [q.angular_similarity(C.minhash_of(r, a, scaled=1)) for r, a in zip(rows, abunds)]
            _same_bits(got, want, (tag, "MinHash.angular_similarity"))


@check
def search_angular_errors():
    rng = np.random.default_rng(2)
    rows = [np.unique(rng.integers(1, 2**60, size=50, dtype=np.uint64)) for _ in range(3)]
    flat = B.SketchSet.from_rows(rows)
    q = np.unique(rng.integers(1, 2**60, size=20, dtype=np.uint64))
    for qh, sset, want in ((q, flat, "needs abundance"), (q[::-1].copy(), B.SketchSet.from_rows(rows, rows), "sorted"),
                           (np.concatenate([q, q[-1:]]), B.SketchSet.from_rows(rows, rows), "sorted")):
        try:
            B.search_angular(qh, np.ones(len(qh), np.uint64), sset, C.U64_MAX)
            raise AssertionError("accepted: " + want)
        except Exception as exc:                        # noqa: BLE001 -- the message is what is checked
            assert want in str(exc), (str(exc), want)
    assert len(B.search_angular(q, np.ones(len(q), np.uint64), B.SketchSet.from_rows([]), C.U64_MAX)) == 0


def _zip_of(sigs, directory):
    from sourmash_b200.signature import save_signatures_to_json
    path = os.path.join(directory, "db%d.zip" % len(os.listdir(directory)))
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for i, s in enumerate(sigs):
            z.writestr("signatures/%03d.sig" % i, save_signatures_to_json([s]))
    return path


def _indexes(sigs, directory):
    from sourmash_b200.index import LinearIndex, ZipFileLinearIndex
    return [LinearIndex(sigs, filename="lin"), ZipFileLinearIndex.load(_zip_of(sigs, directory))]


def _compare(query, sigs, threshold, directory, tag):
    for idx in _indexes(sigs, directory):
        got = C.outcome(lambda: [(r.score, r.signature, r.location) for r in idx.search_abund(query, threshold=threshold)])
        want = C.outcome(lambda: C.reference_search_abund(query, [(s, idx.location) for s in idx.signatures()],
                                                          threshold))
        assert got == want, (tag, type(idx).__name__, got[:2], want[:2])
    return got


@check
def search_abund_follows_the_reference():
    "every index case, LinearIndex and ZipFileLinearIndex, against the per-subject loop: scores, order, errors"
    with tempfile.TemporaryDirectory() as d:
        for tag, query, sigs, thr in C.index_cases(np.random.default_rng(5)):
            got = _compare(query, sigs, thr, d, tag)
            assert got[0] == "ok", (tag, got)
            if thr == 0.0:
                assert len(got[1]) == len(sigs), tag


class _Subject:
    "a subject that is not a SourmashSignature: only .minhash is read by the search, as by the reference's loop"
    def __init__(self, sig):
        self.minhash, self.name, self.md5sum = sig.minhash, sig.name, sig.md5sum


@check
def search_abund_subjects_that_are_not_signatures():
    from sourmash_b200.index import LinearIndex
    for tag, query, sigs, thr in C.index_cases(np.random.default_rng(5))[:3]:
        subj = [_Subject(s) if i % 2 else s for i, s in enumerate(sigs)]
        idx = LinearIndex(subj, filename="lin")
        got = C.outcome(lambda: [(r.score, r.signature, r.location) for r in idx.search_abund(query, threshold=thr)])
        want = C.outcome(lambda: C.reference_search_abund(query, [(s, "lin") for s in subj], thr))
        assert got == want and got[0] == "ok", (tag, got[:2], want[:2])


@check
def search_abund_errors_at_the_same_subject():
    "each error case raises what the reference's loop raises, at the same subject, and returns nothing"
    with tempfile.TemporaryDirectory() as d:
        for tag, query, sigs, thr in C.error_cases(np.random.default_rng(8)):
            got = _compare(query, sigs, thr, d, tag)
            assert got[0] == "raise", (tag, got)


@check
def search_abund_objects_for_matches_only():
    "a ZipFileLinearIndex builds signature objects for the matches only"
    from sourmash_b200.index import ZipFileLinearIndex
    tag, query, sigs, _ = C.index_cases(np.random.default_rng(5))[1]
    with tempfile.TemporaryDirectory() as d:
        idx = ZipFileLinearIndex.load(_zip_of(sigs, d))
        res = idx.search_abund(query, threshold=0.05)
        assert 0 < len(res) < len(sigs), (tag, len(res))
        assert len(idx._objects) == len(res), (len(idx._objects), len(res))


@check
def search_angular_launches_do_not_grow_with_rows():
    rng = np.random.default_rng(3)
    pool = rng.integers(1, 2**63, size=30_000, dtype=np.uint64)
    for nq in (500, C.SPLIT_MAX + 100):
        q = np.unique(rng.choice(pool, size=nq, replace=False))
        counts = []
        for n in (3, 300):
            rows = [np.unique(rng.choice(pool, size=int(rng.integers(1, 3000)), replace=False)) for _ in range(n)]
            sset = B.SketchSet.from_rows(rows, [np.ones(len(r), np.uint64) for r in rows])
            before = B.kernel_launches()
            B.search_angular(q, np.ones(len(q), np.uint64), sset, C.U64_MAX)
            counts.append(B.kernel_launches() - before)
        assert counts[0] == counts[1] and counts[0] >= 1, (nq, counts)


if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        CHECKS[name]()
        print("ok  " + name, flush=True)
    print("search_abund checks passed")
