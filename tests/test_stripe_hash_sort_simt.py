"""The stripe join's stream built from the sorted hashes themselves (csrc/join_stripe.cuh: stripe_iota_kernel or
stripe_gather_slice_kernel, stripe_hash_tag_kernel, the position pass, stripe_hash_fix_kernel), on the CPU through the
SIMT emulator (tests/host_emul/simt_hash_sort_emul.cu), kernel by kernel as join_stripe_create_shard launches it.

Sort windows of 8, 16, 24 and 32 bits: the narrow ones make most runs of equal window bits mix hashes.  Sets: families
drawn from a shared pool with empty rows, hashes that agree in their top 32 bits, a hash held by every row, hashes with
bit 63 set, one run holding the whole set, and hashes no wider than the window (no run can mix hashes).  Whole rows and
the slices of key-range shards (sorted as hash - lo), both tag widths, the swizzle on (n >= 32) and off (n < 32), one
window of pos[] or hundreds of sub-windows.  Tags, positions and successor bits must be those of the stream in (hash,
element) order; the matrix counted from them must be the oracle's."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as orc
from tests.test_stripe_succ_bits_simt import _sets, expected, in_shard, want_counts

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hash_sort_emul():
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_stripe_hash_sort_"), "simt_hash_sort_emul")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++",
                           os.path.join(HERE, "host_emul", "simt_hash_sort_emul.cu"), "-o", exe])

    def run(rows, tag_bits, sort_bits, shards, shard, window, sub, R=3):
        hashes, offsets = orc.to_csr(rows)
        n = len(rows)
        env = {k: v for k, v in os.environ.items() if k not in ("SMB_STRIPE_POS_WINDOW", "SMB_STRIPE_POS_SUBWINDOW")}
        if window:
            env["SMB_STRIPE_POS_WINDOW"] = str(window)
            env["SMB_STRIPE_POS_SUBWINDOW"] = str(sub)
        with tempfile.TemporaryDirectory() as td:
            fh, fo, fc = (os.path.join(td, x) for x in ("h", "o", "c"))
            hashes.tofile(fh)
            offsets.tofile(fo)
            r = subprocess.run([exe, str(tag_bits), str(sort_bits), str(shards), str(shard), str(R), fh, fo, fc], env=env,
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            info = {line.split(":")[0]: int(line.split(":")[1]) for line in r.stderr.splitlines() if ":" in line}
            got = {x: np.fromfile(fc + "." + x, dtype=np.uint32) for x in ("tags", "pos", "succ")}
            got["mat"] = np.fromfile(fc + ".mat", dtype=np.uint32 if shards > 1 else np.float64).reshape(n, n)
            return got, info
    return run


def _more_sets():
    rng = np.random.default_rng(41)
    pool = rng.integers(2**63, 2**64 - 1, size=300, dtype=np.uint64, endpoint=True)
    high = [np.unique(np.concatenate([rng.choice(pool, size=int(rng.integers(0, 120))),
                                      rng.integers(2**63, 2**64 - 1, size=int(rng.integers(0, 60)), dtype=np.uint64, endpoint=True)]))
            for _ in range(40)]
    high[3] = np.zeros(0, np.uint64)
    high[7] = np.array([2**64 - 1], np.uint64)
    # every hash in [2^40, 2^40 + 2^12): with an 8-bit window all of them share their window bits -- one run
    one = [np.unique(rng.integers(2**40, 2**40 + 2**12, size=int(rng.integers(0, 90)), dtype=np.uint64)) for _ in range(20)]
    # hashes below 2^12: narrower than the 32-bit window, so no run can mix hashes
    narrow = [np.unique(rng.integers(1, 2**12, size=int(rng.integers(0, 200)), dtype=np.uint64)) for _ in range(36)]
    return {"bit63": high, "one_run": one, "narrow": narrow}


def _check(hash_sort_emul, rows, tag_bits, sort_bits, shards, shard, window, sub, want_mat):
    got, info = hash_sort_emul(rows, tag_bits, sort_bits, shards, shard, window, sub)
    tags, pos, succ = expected(rows, tag_bits, shards, shard)
    case = (tag_bits, sort_bits, shards, shard, window)
    assert np.array_equal(got["tags"], tags), case
    assert np.array_equal(got["pos"], pos), case
    assert np.array_equal(got["succ"], succ), case
    if shards == 1:
        assert np.array_equal(got["mat"], want_mat), case
    else:
        assert np.array_equal(got["mat"], want_counts(in_shard(rows, shards, shard))), case
    return info


@pytest.mark.parametrize("window,sub", [(256, 32), (None, None)])
@pytest.mark.parametrize("name", ["families", "mixed", "every_row"])
def test_hash_sorted_stream(hash_sort_emul, name, window, sub):
    rows = _sets()[name]
    want_mat = orc.compare_all_pairs(*orc.to_csr(rows), nthreads=2)
    for tag_bits, sort_bits, shards, shard in ((16, 32, 1, 0), (32, 8, 1, 0), (16, 16, 1, 0), (32, 24, 1, 0), (16, 8, 3, 1),
                                               (32, 32, 3, 2), (16, 8, 3, 0), (32, 24, 3, 2)):
        info = _check(hash_sort_emul, rows, tag_bits, sort_bits, shards, shard, window, sub, want_mat)
        if sort_bits == 8 and shards == 1:
            assert info["sort window bits"] == 8 and info["mixed runs repaired"] > 0
        if name == "mixed" and shards == 1:            # hashes that agree in their top 32 bits
            assert info["mixed runs repaired"] > 0


@pytest.mark.parametrize("name", ["bit63", "one_run", "narrow"])
def test_hash_sorted_stream_edges(hash_sort_emul, name):
    rows = _more_sets()[name]
    want_mat = orc.compare_all_pairs(*orc.to_csr(rows), nthreads=2)
    for tag_bits, sort_bits, shards, shard, window, sub in ((16, 32, 1, 0, None, None), (32, 8, 1, 0, 64, 32), (16, 8, 2, 1, None, None),
                                                            (32, 16, 2, 0, 128, 32), (16, 32, 3, 2, 64, 32)):
        info = _check(hash_sort_emul, rows, tag_bits, sort_bits, shards, shard, window, sub, want_mat)
        if name == "one_run" and sort_bits == 8 and shards == 1:
            assert info["mixed runs repaired"] == 1
        if name == "narrow" and sort_bits == 32:
            assert info["sort window bits"] < 32 and info["mixed runs repaired"] == 0
