"""The successor bits of the stripe join (csrc/join_stripe.cuh) and the positions written with them through shared-memory
sub-windows, on the CPU through the SIMT emulator (tests/host_emul/simt_succ_emul.cu): window offsets, tags + position
buckets, the partition into sub-window buckets, the sub-window pass, the repair of runs that mix hashes and the count
kernel reading the bits, as join_stripe_create_shard and join_stripe_rows launch them.

SMB_STRIPE_POS_WINDOW / SMB_STRIPE_POS_SUBWINDOW of 64 to 512 / 32 or 64 elements split the sets into tens of windows
and hundreds of sub-windows; without them a set is one window and the tag kernel stores positions and bits itself.
The sets have empty rows (first, last, and in the middle), rows longer than a window, element counts that are not a
multiple of either size and a hash held by every row; the streams are whole rows or the slices of one key range out of
three; hashes that agree in their top 32 bits make runs that mix hashes, whose positions and bits come from the fix
kernel (sort keys cut to 8 bits as well).  Both tag widths.  Tags and positions must be those of the stream defined by the
sort, elements in (hash, element) order; succ[e] must say whether the next stream element holds the same hash; the
matrix counted with the bits must be the oracle's."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
PAD = 128                                   # STRIPE_TAG_PAD


@pytest.fixture(scope="module")
def succ_emul():
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_stripe_succ_"), "simt_succ_emul")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++",
                           os.path.join(HERE, "host_emul", "simt_succ_emul.cu"), "-o", exe])

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


def in_shard(rows, shards, shard):
    "the part of every row that lies in key range `shard` of `shards` (join_shard_range)"
    if shards == 1:
        return [np.asarray(r, np.uint64) for r in rows]
    step = int(max(int(r.max()) for r in rows if len(r))) // shards + 1
    lo, hi = shard * step, (shard + 1) * step
    return [np.array([x for x in r if lo <= int(x) and (shard + 1 == shards or int(x) < hi)], dtype=np.uint64) for r in rows]


def expected(rows, tag_bits, shards, shard):
    "tags (with the head flags behind the stream), pos and succ words of the stream of key range `shard` of `shards`"
    h, off = orc.to_csr(rows)
    n = len(rows)
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(off).astype(np.int64))
    step = int(h.max()) // shards + 1
    lo, hi = shard * step, (shard + 1) * step
    keep = np.array([lo <= x and (shard + 1 == shards or x < hi) for x in h.astype(object)], dtype=bool)
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
    bit = np.zeros(-(-len(h) // 32) * 32, dtype=bool)
    bit[e[:-1]] = h[e][1:] == h[e][:-1]                  # the next stream element holds the same hash
    succ = np.packbits(bit, bitorder="little").view("<u4").astype(np.uint32)
    return tags, pos, succ


def want_counts(rows):
    "a shard's partial counts: |A_i ∩ A_j| off the diagonal; the diagonal counter is never bumped"
    n = len(rows)
    c = np.zeros((n, n), dtype=np.uint32)
    for i in range(n):
        for j in range(n):
            if i != j:
                c[i, j] = len(np.intersect1d(rows[i], rows[j]))
    return c


def _sets():
    rng = np.random.default_rng(23)
    # 60 rows of 0 .. 300 hashes drawn half from a shared pool, empty rows first, last and in the middle, one row of 1100
    pool = rng.integers(1, 2**62, size=500, dtype=np.uint64)
    fam = []
    for i in range(60):
        m = 0 if i in (0, 17, 18, 59) else (1100 if i == 30 else int(rng.integers(1, 300)))
        fam.append(np.unique(np.concatenate([rng.choice(pool, size=m // 2), rng.integers(1, 2**62, size=m - m // 2, dtype=np.uint64)])))
    # hashes that agree in their top 32 bits and differ below, interleaved over rows: mixed runs with the full 32-bit keys
    top = [np.uint64(v) << np.uint64(32) for v in (9, 3, 7)]
    lows = [np.uint64(0x1234abcd), np.uint64(1), np.uint64(0xffffffff)]
    mixed = []
    for i in range(37):
        mine = [t | lo for ti, t in enumerate(top) for li, lo in enumerate(lows) if (i + ti + 2 * li) % 3 != 0]
        mixed.append(np.unique(np.array(mine + rng.integers(1, 2**63, size=int(rng.integers(0, 150)), dtype=np.uint64).tolist(),
                                        dtype=np.uint64)))
    mixed[5] = np.zeros(0, np.uint64)
    # one hash held by every row (the largest of the set: the last group of the stream), each row's other hashes its own
    every = [np.unique(np.concatenate([np.array([2**62 + 5], np.uint64), rng.integers(1, 2**62, size=int(rng.integers(0, 120)), dtype=np.uint64)]))
             for _ in range(45)]
    return {"families": fam, "mixed": mixed, "every_row": every}


@pytest.mark.parametrize("window,sub", [(256, 32), (64, 32), (512, 64), (None, None)])
@pytest.mark.parametrize("name", ["families", "mixed", "every_row"])
def test_succ_bits_through_sub_windows(succ_emul, name, window, sub):
    rows = _sets()[name]
    total = sum(len(r) for r in rows)
    want_mat = orc.compare_all_pairs(*orc.to_csr(rows), nthreads=2)
    if window:
        assert total % window != 0 and total % sub != 0 and total > 40 * sub
    for tag_bits, sort_bits, shards, shard in ((16, 32, 1, 0), (32, 8, 1, 0), (16, 8, 3, 1), (32, 32, 3, 2), (16, 8, 3, 0)):
        got, info = succ_emul(rows, tag_bits, sort_bits, shards, shard, window, sub)
        assert info["windows"] == (-(-total // window) if window else 1)
        if window:
            assert info["sub-windows"] == -(-total // sub)
        tags, pos, succ = expected(rows, tag_bits, shards, shard)
        case = (name, window, tag_bits, sort_bits, shards, shard)
        assert np.array_equal(got["tags"], tags), case
        assert np.array_equal(got["pos"], pos), case
        assert np.array_equal(got["succ"], succ), case
        if name == "mixed" and shard == 0:              # (the mixed hashes are small: key range 0)
            assert info["mixed runs repaired"] > 0, case
        if shards == 1:
            assert np.array_equal(got["mat"], want_mat), case
        else:
            assert np.array_equal(got["mat"], want_counts(in_shard(rows, shards, shard))), case
