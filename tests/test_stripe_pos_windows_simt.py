"""The sorted stream of the stripe join (csrc/join_stripe.cuh) built through windows of pos[] far smaller than the product's,
on the CPU through the SIMT emulator (tests/host_emul/simt_stream_emul.cu): window offsets, tags + position buckets, the
window pass and the repair of runs that mix hashes, as join_stripe_create_shard launches them.

SMB_STRIPE_POS_WINDOW = 16, 32, 64 elements splits the sets into hundreds of windows; without it the sets are one window
and the tag kernel stores the positions itself.  The sets have empty rows (first,
last, and in the middle), rows longer than a window and element counts that are not a multiple of it; the streams are
whole rows or the slices of one key range out of three; sort keys cut to 8 bits and hashes that agree in their top 32
bits make runs that mix hashes, whose positions come from the fix kernel.  Both tag widths.  The tags and positions
must be exactly those of the stream defined by the sort: elements in (hash, element) order."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
PAD = 128                                   # STRIPE_TAG_PAD


@pytest.fixture(scope="module")
def stream():
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_stripe_windows_"), "simt_stream_emul")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++",
                           os.path.join(HERE, "host_emul", "simt_stream_emul.cu"), "-o", exe])

    def run(rows, tag_bits, sort_bits, shards, shard, window):
        hashes, offsets = orc.to_csr(rows)
        env = {k: v for k, v in os.environ.items() if k != "SMB_STRIPE_POS_WINDOW"}
        env["SMB_EMUL_REPORT"] = "1"
        if window:
            env["SMB_STRIPE_POS_WINDOW"] = str(window)
        with tempfile.TemporaryDirectory() as td:
            fh, fo, fc = (os.path.join(td, x) for x in ("h", "o", "c"))
            hashes.tofile(fh)
            offsets.tofile(fo)
            r = subprocess.run([exe, str(tag_bits), str(sort_bits), str(shards), str(shard), fh, fo, fc], env=env,
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            windows = int(r.stderr.split("windows:")[1].split()[0])
            return np.fromfile(fc, dtype=np.uint32), windows
    return run


def expected(rows, tag_bits, shards, shard):
    "tags (with the head flags behind the stream) and pos of the stream of key range `shard` of `shards`"
    h, off = orc.to_csr(rows)
    n = len(rows)
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(off).astype(np.int64))
    step = int(h.max()) // shards + 1 if len(h) else 1
    lo, hi = shard * step, (shard + 1) * step
    hv = h.astype(object)
    keep = np.array([lo <= x and (shard + 1 == shards or x < hi) for x in hv], dtype=bool)
    e = np.nonzero(keep)[0]
    e = e[np.lexsort((e, h[e]))]                         # hash order, elements ascending inside a group
    head_flag = 0x8000 if tag_bits == 16 else 0x80000000
    swz = n & ~31
    col = np.where(row[e] < swz, row[e] ^ ((row[e] >> 5) & 31), row[e]).astype(np.uint64)
    head = np.ones(len(e), dtype=bool)
    head[1:] = h[e][1:] != h[e][:-1]
    tags = np.concatenate([(col | np.where(head, head_flag, 0).astype(np.uint64)).astype(np.uint32),
                           np.full(PAD, head_flag, np.uint32)])
    pos = np.full(len(h), 0xFFFFFFFF, np.uint32)
    pos[e] = np.arange(len(e), dtype=np.uint32)
    return np.concatenate([tags, pos])


def _sets():
    rng = np.random.default_rng(5)
    # rows of 0 .. 150 hashes (several 16- to 64-element windows long), families sharing hashes, empty rows at both ends
    pool = rng.integers(1, 2**62, size=400, dtype=np.uint64)
    fam = []
    for i in range(41):
        m = 0 if i in (0, 17, 18, 40) else int(rng.integers(1, 150))
        fam.append(np.unique(np.concatenate([rng.choice(pool, size=m // 2), rng.integers(1, 2**62, size=m - m // 2, dtype=np.uint64)])))
    # hashes that agree in their top 32 bits and differ below, interleaved over rows: mixed runs with the full 32-bit keys
    top = [np.uint64(v) << np.uint64(32) for v in (9, 3, 7)]
    lows = [np.uint64(0x1234abcd), np.uint64(1), np.uint64(0xffffffff)]
    mixed = []
    for i in range(37):
        mine = [t | lo for ti, t in enumerate(top) for li, lo in enumerate(lows) if (i + ti + 2 * li) % 3 != 0]
        mixed.append(np.unique(np.array(mine + rng.integers(1, 2**63, size=int(rng.integers(0, 70)), dtype=np.uint64).tolist(),
                                        dtype=np.uint64)))
    mixed[5] = np.zeros(0, np.uint64)
    one = [np.arange(1, 1001, dtype=np.uint64) * np.uint64(7919)]          # a single row of 1000 elements
    return {"families": fam, "mixed": mixed, "one_long_row": one}


@pytest.mark.parametrize("window", [16, 32, 64, None])
@pytest.mark.parametrize("name", ["families", "mixed", "one_long_row"])
def test_stream_through_small_pos_windows(stream, name, window):
    rows = _sets()[name]
    total = sum(len(r) for r in rows)
    if window:
        assert total % window != 0 and total > 10 * window
    for tag_bits in (16, 32):
        for sort_bits in (32, 8):
            for shards, shard in ((1, 0), (3, 0), (3, 1), (3, 2)):
                got, windows = stream(rows, tag_bits, sort_bits, shards, shard, window)
                assert windows == (-(-total // window) if window else 1)
                want = expected(rows, tag_bits, shards, shard)
                assert np.array_equal(got, want), (name, window, tag_bits, sort_bits, shards, shard)
