"""batch.lca_index with the EMULATED build (emul_lib.py), against the oracle of tests/lca_index_cases.py (the
reference's insert loop restated, serialised with json): the arrays, and the chunked text byte for byte.  Run as a
script by tests/test_lca_index_emulated.py; tests/test_gpu_lca_index.py runs the same checks on the device.

    python tests/host_emul/lca_index_checks.py [name ...]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    import emulated_boot  # noqa: E402
    emulated_boot.install()

import numpy as np  # noqa: E402

from tests import lca_index_cases as C  # noqa: E402

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def _build(rows):
    from sourmash_b200 import batch as B
    h, off = C.csr(rows)
    return B.lca_index(B.SketchSet.from_host(h, off))


def _compare(rows, chunk_sizes=(256 << 20,), tag=""):
    want_h, want_off, want_idx, want_text = C.oracle(rows)
    x = _build(rows)
    assert len(x) == len(want_h) and x.pairs() == len(want_idx), (tag, len(x), len(want_h))
    h, off, idx = x.arrays()
    assert np.array_equal(h, want_h), tag
    assert np.array_equal(off, want_off), tag
    assert np.array_equal(idx, want_idx), tag
    for size in chunk_sizes:
        chunks = list(x.text_chunks(size))
        assert b"".join(chunks) == want_text, (tag, size)
        assert all(len(c) <= size for c in chunks if c.count(b"[") > 1), (tag, size)
    return x


@check
def lca_index_small():
    "one row, two rows sharing hashes, a row of 0 and UINT64_MAX, all-digit-length idx and hashes"
    _compare([np.array([5, 7, 9], np.uint64)], tag="one row")
    _compare([np.array([1, 2, 3], np.uint64), np.array([2, 3, 4], np.uint64)], tag="two rows")
    _compare([np.array([0, C.U64_MAX], np.uint64), np.array([0], np.uint64), np.array([C.U64_MAX], np.uint64)],
             tag="extremes")
    digits = np.array([10**k for k in range(20)] + [10**k - 1 for k in range(1, 20)], dtype=np.uint64)
    _compare([np.unique(digits)], chunk_sizes=(1, 7, 50, 1 << 20), tag="digits")


@check
def lca_index_random():
    """random rows: shared hashes, hashes in no row, empty rows, one row with every hash, idx past 7, several chunk
    sizes including ones below a single key's text"""
    for seed in range(4):
        rng = np.random.default_rng(seed)
        rows = C.random_rows(rng, n_rows=12 + 15 * seed)
        _compare(rows, chunk_sizes=(1, 64, 997, 256 << 20), tag="random %d" % seed)


@check
def lca_index_ranges():
    "every key range the text comes in is the oracle's text of exactly those keys"
    from sourmash_b200._lowlevel import ffi, lib
    rows = C.random_rows(np.random.default_rng(11), n_rows=30)
    x = _build(rows)
    h, off, idx = x.arrays()
    n = len(x)
    size = ffi.new("uintptr_t *")
    for max_bytes in (1, 100, 5000):
        k = 0
        while k < n:
            nxt = int(lib.smb_lca_index_text(x._ptr, k, max_bytes, ffi.NULL, size))
            assert k < nxt <= n
            buf = bytearray(int(size[0]))
            size[0] = len(buf)
            lib.smb_lca_index_text(x._ptr, k, max_bytes, ffi.from_buffer(buf), size)
            assert bytes(buf) == C.text_of_keys(h, off, idx, k, nxt, n), (max_bytes, k, nxt)
            assert nxt == k + 1 or len(buf) <= max_bytes
            k = nxt


@check
def lca_index_empty():
    "no rows, only empty rows: no keys, the text {}, and no launch"
    from sourmash_b200 import batch as B
    for rows in ([], [np.zeros(0, np.uint64)] * 3):
        before = B.kernel_launches()
        x = _compare(rows, chunk_sizes=(1, 1 << 20), tag="empty %d" % len(rows))
        assert len(x) == 0 and B.kernel_launches() == before
        h, off, idx = x.arrays()
        assert len(h) == 0 and off.tolist() == [0] and len(idx) == 0


@check
def lca_index_budget():
    """the byte budget counts the braces: a budget of the whole text gives one range, one byte less gives two, and no
    range of more than one key is longer than its budget"""
    rows = C.random_rows(np.random.default_rng(5), n_rows=20)
    want = C.oracle(rows)[3]
    x = _build(rows)
    assert [len(c) for c in x.text_chunks(len(want))] == [len(want)]
    parts = list(x.text_chunks(len(want) - 1))
    assert len(parts) == 2 and b"".join(parts) == want and all(len(c) <= len(want) - 1 for c in parts)
    for size in range(2, 200, 7):
        for c in x.text_chunks(size):
            assert len(c) <= size or c.count(b"[") == 1, (size, c[:80])


@check
def lca_index_capacity():
    """one call per range: the text is written when it fits the caller's buffer; a buffer too small gets nothing and
    learns the range's size"""
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import ffi, lib
    rows = C.random_rows(np.random.default_rng(6), n_rows=10)
    h, off, idx, want = C.oracle(rows)
    x = _build(rows)
    size = ffi.new("uintptr_t *")
    buf = bytearray(b"#" * (len(want) + 10))
    size[0] = len(buf)
    before = B.kernel_launches()
    nxt = lib.smb_lca_index_text(x._ptr, 0, len(want), ffi.from_buffer(buf), size)
    assert B.kernel_launches() - before == 2                        # the plan and the text, nothing more
    assert nxt == len(x) and size[0] == len(want) and bytes(buf[:len(want)]) == want
    small = bytearray(b"#" * 8)
    size[0] = len(small)
    nxt = lib.smb_lca_index_text(x._ptr, 0, 1 << 20, ffi.from_buffer(small), size)
    assert nxt == len(x) and size[0] == len(want) and bytes(small) == b"#" * 8


@check
def lca_index_argument_errors():
    "a first key out of range is refused before any launch"
    from sourmash_b200 import batch as B
    from sourmash_b200._ffi import rustcall
    from sourmash_b200._lowlevel import ffi, lib
    x = _build([np.array([1, 2, 3], np.uint64)])
    empty = _build([])
    size = ffi.new("uintptr_t *")
    bad = [(lambda: rustcall(lib.smb_lca_index_text, x._ptr, 3, 100, ffi.NULL, size), "out of range"),
           (lambda: rustcall(lib.smb_lca_index_text, empty._ptr, 1, 100, ffi.NULL, size), "out of range")]
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
def lca_index_numpy_oracle():
    "the numpy oracle of the GPU test agrees with the dict oracle on random rows"
    for seed in range(3):
        rows = C.random_rows(np.random.default_rng(100 + seed), n_rows=25)
        want = C.oracle(rows)[:3]
        got = C.np_oracle_arrays(*C.csr(rows))
        for a, b in zip(got, want):
            assert np.array_equal(a, b), seed
    h, off = C.skewed_rows(1, 200, 20000)
    x = _compare_arrays(h, off)
    assert len(x) > 0


def _compare_arrays(h, off):
    from sourmash_b200 import batch as B
    x = B.lca_index(B.SketchSet.from_host(h, off))
    for a, b in zip(x.arrays(), C.np_oracle_arrays(h, off)):
        assert np.array_equal(a, b)
    return x


if __name__ == "__main__":
    names = sys.argv[1:] or list(CHECKS)
    for name in names:
        CHECKS[name]()
        print("ok  " + name, flush=True)
    print("lca index checks passed")
