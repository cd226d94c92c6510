"""The many-query range-major pass (csrc/range_kernels.cuh: one_vs_many_range_major_kernel with a query-id array) on
the CPU through the SIMT emulator (tests/host_emul/simt_many_emul.cu), against a brute force with np.intersect1d for
every (query, row), and its null-id one-query form against the single-query harness (tests/host_emul/simt_emul.cu)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
BIG = np.uint64(2**64 - 1)


def _compile(src, name):
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_mvm_"), name)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++", src, "-o", exe])
    return exe


def _csr(arrays):
    off = np.zeros(len(arrays) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(a) for a in arrays])
    h = np.concatenate([np.asarray(a, np.uint64) for a in arrays]) if arrays else np.zeros(0, np.uint64)
    return h.astype(np.uint64), off


@pytest.fixture(scope="module")
def many():
    exe = _compile(os.path.join(HERE, "host_emul", "simt_many_emul.cu"), "simt_many_emul")

    def run(queries, rows, P, bm_log2, threads, ids=1):
        with tempfile.TemporaryDirectory() as td:
            paths = [os.path.join(td, x) for x in ("q", "qo", "h", "o", "c")]
            for arr, p in zip(_csr(queries) + _csr(rows), paths):
                arr.tofile(p)
            subprocess.check_call([exe, str(P), str(bm_log2), str(threads), str(ids)] + paths)
            return np.fromfile(paths[-1], dtype=np.uint32).reshape(len(queries), len(rows))
    return run


@pytest.fixture(scope="module")
def single():
    exe = _compile(os.path.join(HERE, "host_emul", "simt_emul.cu"), "simt_emul")

    def run(query, rows, P, bm_log2, threads):
        with tempfile.TemporaryDirectory() as td:
            fq, fh, fo, fc = (os.path.join(td, x) for x in ("q", "h", "o", "c"))
            np.asarray(query, np.uint64).tofile(fq)
            h, off = _csr(rows)
            h.tofile(fh); off.tofile(fo)
            subprocess.check_call([exe, "ranges", str(P), str(bm_log2), str(threads), fq, fh, fo, fc])
            return np.fromfile(fc, dtype=np.uint32)
    return run


def brute(queries, rows):
    return np.array([[len(np.intersect1d(q, r)) for r in rows] for q in queries], dtype=np.uint32).reshape(
        len(queries), len(rows))


def _cases():
    from sourmash_b200.synth import synth_sketches
    rng = np.random.default_rng(19)
    mx = np.uint64(2**64 // 1000)
    h, off = synth_sketches(70, mean=250, sd=60, lo=0, hi=600, n_families=3, pool=400, seed=23)
    fam = [h[int(off[i]):int(off[i + 1])] for i in range(70)]
    fam[5] = np.zeros(0, np.uint64)                                                    # empty rows
    fam[40] = np.array([0, 1, 2, BIG - 1, BIG], np.uint64)
    fam[41] = np.zeros(0, np.uint64)
    a = np.unique(np.concatenate([fam[3], fam[17][:100], rng.integers(1, mx, size=800, dtype=np.uint64),
                                  np.array([0, mx + 5, 2**63, BIG], dtype=np.uint64)]))
    b = np.unique(np.concatenate([fam[3][::2], fam[20], fam[40]]))
    low = np.unique(rng.integers(0, 1000, size=120, dtype=np.uint64))                  # every key in the first range
    fam_q = [a, a.copy(), a[::3].copy(), np.zeros(0, np.uint64), b, fam[20].copy(), np.array([0, BIG], np.uint64),
             low, a[::2].copy()]                                                        # identical, nested, empty, edge keys
    # near-copies of the queries: every element a match, the warps' queues overflow and drain mid-loop
    near = [np.setdiff1d(a, a[i::13]) for i in range(30)] + [b, np.zeros(0, np.uint64)]
    near_q = [a, a[::2].copy(), a, b]
    return [(fam, fam_q), (near, near_q), ([fam[5]], fam_q[:3]), (fam[:3], [low, low])]


@pytest.mark.parametrize("P,bm_log2,threads", [(5, 16, 64), (2, 6, 96), (9, 12, 32), (3, 8, 64), (4, 10, 64)])
def test_simt_many_query_pass_matches_bruteforce(many, P, bm_log2, threads):
    """bitmaps of 2^6 .. 2^16 bits (false positives common), few ranges (small SMB_RM_RANGES; with 9 ranges some hold
    no query key), keys held by many queries, keys 0 and 2^64 - 1, empty rows and queries, overflowing queues"""
    for rows, queries in _cases():
        got = many(queries, rows, P, bm_log2, threads)
        assert np.array_equal(got, brute(queries, rows)), (len(rows), P, bm_log2, threads)


@pytest.mark.parametrize("P,bm_log2,threads", [(5, 16, 64), (2, 6, 96), (3, 8, 64)])
def test_simt_null_id_form_equals_single_query_pass(many, single, P, bm_log2, threads):
    "one query with a null id array: the counts of the single-query harness for the same inputs"
    for rows, queries in _cases():
        for q in queries[:3]:
            if not len(q):
                continue
            got = many([q], rows, P, bm_log2, threads, ids=0)[0]
            assert np.array_equal(got, single(q, rows, P, bm_log2, threads)), (len(rows), P, bm_log2)
            assert np.array_equal(got, brute([q], rows)[0])
