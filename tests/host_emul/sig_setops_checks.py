"""batch.combine and the sigsetops functions end to end with the EMULATED build (emul_lib.py), against the numpy
restatement and the reference's loops of tests/sig_setops_cases.py.  Run as a script by
tests/test_sig_setops_emulated.py.

    python tests/host_emul/sig_setops_checks.py [name ...]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emulated_boot  # noqa: E402

LIB = emulated_boot.install()

import numpy as np  # noqa: E402

from sourmash_b200 import batch as B  # noqa: E402
from tests import sig_setops_cases as C  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


@check
def combine_edge_cases():
    "every case of sig_setops_cases, all three ops, flat and with abundances, against numpy and the reference's loops"
    for tag, rows, ab in C.cases(np.random.default_rng(7)):
        sset = B.SketchSet.from_host(*C.csr(rows, ab))
        for op in ("union", "all", "first_only"):
            got = B.combine(sset, op)
            C.assert_same(got, C.numpy_combine(op, rows, ab), (tag, op, "numpy"))
            C.assert_same(got, C.reference_combine(op, rows, ab), (tag, op, "reference loop"))


@check
def combine_num_union():
    "a num union keeps the bottom num of the union, abundances summed, as a chain of merges into a num sketch does"
    rng = np.random.default_rng(9)
    pool = rng.integers(1, 2**63, size=2000, dtype=np.uint64)
    for num in (1, 50, 500):
        rows = [np.sort(rng.choice(pool, size=min(num, int(rng.integers(1, 400))), replace=False)) for _ in range(12)]
        for ab in (None, [rng.integers(1, 50, size=len(r)).astype(np.uint64) for r in rows]):
            got = B.combine(B.SketchSet.from_host(*C.csr(rows, ab)), "union", num=num)
            C.assert_same(got, C.numpy_combine("union", rows, ab, num=num), ("num", num))
            C.assert_same(got, C.reference_combine("union", rows, ab, num=num), ("num loop", num))
            assert len(got[0]) == min(num, len(np.unique(np.concatenate(rows))))


@check
def combine_launches_do_not_grow_with_rows():
    rng = np.random.default_rng(3)
    pool = rng.integers(1, 2**63, size=5000, dtype=np.uint64)
    for op in ("union", "all", "first_only"):
        counts = []
        for n in (3, 300):
            rows = [np.unique(rng.choice(pool, size=200, replace=False)) for _ in range(n)]
            ab = [np.ones(len(r), np.uint64) for r in rows]
            sset = B.SketchSet.from_host(*C.csr(rows, ab))
            before = B.kernel_launches()
            B.combine(sset, op)
            counts.append(B.kernel_launches() - before)
        assert counts[0] == counts[1], (op, counts)


@check
def minhash_functions_follow_the_reference():
    "merge / intersect / subtract_minhashes on MinHash and SourmashSignature lists, and their errors"
    from sourmash_b200.minhash import MinHash
    from sourmash_b200.signature import SourmashSignature
    from sourmash_b200.sigsetops import intersect_minhashes, merge_minhashes, subtract_minhashes
    rng = np.random.default_rng(5)
    pool = rng.integers(1, 2**62, size=600, dtype=np.uint64)
    rows = [np.unique(rng.choice(pool, size=150, replace=False)) for _ in range(5)]
    ab = [rng.integers(1, 9, size=len(r)).astype(np.uint64) for r in rows]
    for abunds in (None, ab):
        mhs = [C.minhash_of(r, None if abunds is None else abunds[i]) for i, r in enumerate(rows)]
        for objs in (mhs, [SourmashSignature(m, name="s%d" % i) for i, m in enumerate(mhs)]):
            want = mhs[0].copy_and_clear()
            for m in mhs:
                want.merge(m)
            got = merge_minhashes(objs)
            assert got == want and got.track_abundance == want.track_abundance
            flat = merge_minhashes(objs, flatten=True)
            assert not flat.track_abundance and set(flat.hashes) == set(want.hashes)
            common = set(mhs[0].hashes)
            for m in mhs[1:]:
                common &= set(m.hashes)
            got = intersect_minhashes(objs)
            assert set(got.hashes) == common and not got.track_abundance
            rest = set(mhs[0].hashes)
            for m in mhs[1:]:
                rest -= set(m.hashes)
            if abunds is None:
                assert set(subtract_minhashes(objs).hashes) == rest
            else:
                try:
                    subtract_minhashes(objs)
                    raise AssertionError("subtract of abundance sketches was accepted")
                except ValueError as exc:
                    assert "abundance tracking" in str(exc)
                assert set(subtract_minhashes(objs, flatten=True).hashes) == rest
    flat = [C.minhash_of(r) for r in rows]
    for other, msg in ((MinHash(0, 21, scaled=1), "different ksizes cannot be compared"),
                       (MinHash(0, 31, scaled=2), "mismatch in scaled; comparison fail"),
                       (MinHash(0, 31, scaled=1, seed=7), "mismatch in seed; comparison fail"),
                       (MinHash(0, 31, scaled=1, is_protein=True), "different ksizes cannot be compared"),
                       (MinHash(0, 31, scaled=1, track_abundance=True), "track_abundance is False in first sig")):
        if "track_abundance" not in msg:                   # MinHash.merge itself raises the same message
            try:
                flat[0].copy_and_clear().merge(other)
                raise AssertionError("MinHash.merge accepted: " + msg)
            except ValueError as exc:
                assert str(exc) == msg, (str(exc), msg)
        for fn, want in ((merge_minhashes, msg),
                         (intersect_minhashes, "incompatible minhashes; specify -k and/or molecule type.")):
            if fn is intersect_minhashes and "track_abundance" in msg:
                continue                                     # intersect does not check abundance tracking
            try:
                fn(flat[:2] + [other])
                raise AssertionError("incompatible sketch accepted: " + msg)
            except ValueError as exc:
                assert want in str(exc), (str(exc), want)

if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        CHECKS[name]()
        print("ok  " + name, flush=True)
    print("sig set-op checks passed")
