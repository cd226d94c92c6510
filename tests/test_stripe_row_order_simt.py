"""The row order of the stripe join's count kernel (csrc/join_stripe.cuh: stripe_label_kernel, stripe_select_rows_kernel)
on the CPU through the SIMT emulator (tests/host_emul/simt_order_emul.cu): the labels are compared with
a restatement of the rule, and the matrix counted in that order -- two ranges of rows, each in the order's order --
with the oracle bit for bit.

The rule: label[r] = min(r, the lowest row of the group of each of r's first 8 stream elements that are not singletons,
among its first 256 elements).
The sets have rows that share no hash (their label is their own row), a hash held by every row (every label 0, except
for a row that holds it behind its first 256 elements),
families at a stride with groups of more than 64 rows (walks back over several 32-tag windows), and a group at stream
position 0.  Both tag widths, swizzle on and off, the whole set and the slices of one key range out of three."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
GROUPS = 8                                  # STRIPE_LABEL_GROUPS
SCAN = 256                                  # STRIPE_LABEL_SCAN


@pytest.fixture(scope="module")
def order():
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_stripe_order_"), "simt_order_emul")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++",
                           os.path.join(HERE, "host_emul", "simt_order_emul.cu"), "-o", exe])

    def run(rows, tag_bits, swizzle, shards, shard, R):
        hashes, offsets = orc.to_csr(rows)
        n = len(rows)
        with tempfile.TemporaryDirectory() as td:
            fh, fo, fc = (os.path.join(td, x) for x in ("h", "o", "c"))
            hashes.tofile(fh)
            offsets.tofile(fo)
            subprocess.check_call([exe, str(tag_bits), str(swizzle), str(shards), str(shard), str(R), fh, fo, fc])
            lab = np.fromfile(fc + ".lab", dtype=np.uint32)
            mat = np.fromfile(fc + ".mat", dtype=np.uint32 if shards > 1 else np.float64).reshape(n, n)
            return lab, mat
    return run


def in_shard(rows, shards, shard):
    "the part of every row that lies in key range `shard` of `shards` (join_shard_range)"
    if shards == 1:
        return [np.asarray(r, np.uint64) for r in rows]
    step = int(max(int(r.max()) for r in rows if len(r))) // shards + 1
    lo, hi = shard * step, (shard + 1) * step
    return [np.array([x for x in r if lo <= int(x) and (shard + 1 == shards or int(x) < hi)], dtype=np.uint64) for r in rows]


def want_labels(rows):
    "the labelling rule, restated on the rows' hashes (rows ascend inside a group: its lowest row is its first holder)"
    first, held = {}, {}
    for r, row in enumerate(rows):
        for x in row.tolist():
            first.setdefault(x, r)
            held[x] = held.get(x, 0) + 1
    lab = []
    for r, row in enumerate(rows):
        shared = [x for x in row.tolist()[:SCAN] if held[x] > 1][:GROUPS]
        lab.append(min([r] + [first[x] for x in shared]))
    return np.array(lab, dtype=np.uint32)


def want_counts(rows):
    "a shard's partial counts: |A_i ∩ A_j| off the diagonal; the diagonal counter is never bumped (finalize writes 1)"
    n = len(rows)
    c = np.zeros((n, n), dtype=np.uint32)
    for i in range(n):
        for j in range(n):
            if i != j:
                c[i, j] = len(np.intersect1d(rows[i], rows[j]))
    return c


def _sets():
    rng = np.random.default_rng(11)
    n = 150
    # families at a stride: odd rows draw from pool 1 (with the even rows r % 5 == 1: groups of about 80 rows), even rows
    # from pool r % 5; every 13th row shares nothing
    pools = [rng.choice(np.arange(10, 2**40, 7919, dtype=np.uint64)[:4000], size=60, replace=False) for _ in range(5)]
    fam = []
    for r in range(n):
        own = rng.integers(2**41, 2**62, size=int(rng.integers(5, 40)), dtype=np.uint64)
        if r % 13 == 5:
            fam.append(np.unique(own))
            continue
        f = 1 if r % 2 else r % 5
        take = pools[f][rng.random(60) < 0.9]
        fam.append(np.unique(np.concatenate([own, take])))
    for r in (3, 40, 77):                                # hash 1: the smallest, a group at stream position 0
        fam[r] = np.unique(np.concatenate([fam[r], np.array([1], np.uint64)]))
    # one hash held by every row, each row's other hashes its own
    every = [np.unique(np.concatenate([np.array([2**50], np.uint64),
                                       rng.integers(1, 2**62, size=int(rng.integers(0, 30)), dtype=np.uint64)]))
             for _ in range(70)]
    every[1] = np.unique(np.concatenate([every[1], np.arange(2, 2 + 300, dtype=np.uint64)]))   # 2^50 is its 301st hash or later
    return {"families": fam, "every_row": every}


@pytest.mark.parametrize("name", ["families", "every_row"])
def test_row_order_labels_and_matrix(order, name):
    rows = _sets()[name]
    n = len(rows)
    want_mat = orc.compare_all_pairs(*orc.to_csr(rows), nthreads=2)
    for tag_bits, swizzle, R in ((16, 1, 3), (32, 0, 2), (16, 0, 5), (32, 1, 1)):
        for shards, shard in ((1, 0), (3, 1)):
            lab, mat = order(rows, tag_bits, swizzle, shards, shard, R)
            part = in_shard(rows, shards, shard)
            want = want_labels(part)
            assert np.array_equal(lab, want), (name, tag_bits, swizzle, shards, shard)
            if shards == 1:
                assert np.array_equal(mat, want_mat), (name, tag_bits, swizzle, R)
            else:
                assert np.array_equal(mat, want_counts(part)), (name, tag_bits, swizzle, shard, R)
    # what the sets are there for
    lab = want_labels(rows)
    if name == "every_row":
        assert lab[1] == 1 and not lab[0] and not lab[2:].any()
    else:
        loners = [r for r in range(n) if r % 13 == 5]
        assert all(lab[r] == r for r in loners)
        assert len(set(lab.tolist())) < n // 4
        assert max(sum(1 for r in rows if x in set(r.tolist())) for x in rows[1].tolist()) > 64
