"""Row sets at the read boundaries of the stripe count kernel (csrc/join_stripe.cuh: join_stripe_kernel), shared by the
emulated test (tests/test_stripe_group_edges_simt.py) and the GPU test (tests/test_gpu_stripe_group_edges.py).

For an element with members behind it, the kernel reads the 64 tags that follow it, then 32 more per round until it meets
the next group head.  The sets put single hashes into k rows for k around those sizes (k - 1 members behind the group's
head: 1, 7, 8, 56, 57, 63, 64, 65, 120, 128), give every row 0-7 private hashes that land between the groups in the
sorted stream (so that groups and elements start at many positions modulo 8, i.e. modulo 16 bytes of u16 tags), and end
the stream with one of the groups (its reads run into the head flags behind the stream)."""
import numpy as np

SHARED = (2, 8, 9, 57, 58, 64, 65, 66, 121, 129)
LAST = (129, 65, 2)                      # the group at the end of the stream, one row set each


def edge_rows(last, seed=0):
    """max(SHARED) + 3 rows.  Group j (hash (j + 1) << 24) holds the k = order[j] rows i with (i + 7 j) mod n < k, where
    `order` is SHARED with `last` moved to the end: its hash is the largest of the set.  Row i also holds i mod 8
    private odd hashes below that largest one."""
    rng = np.random.Generator(np.random.PCG64(seed))
    order = [k for k in SHARED if k != last] + [last]
    n = max(SHARED) + 3
    rows = []
    for i in range(n):
        shared = [(j + 1) << 24 for j, k in enumerate(order) if (i + 7 * j) % n < k]
        private = (rng.integers(1, len(order) << 23, size=i % 8, dtype=np.uint64) << np.uint64(1)) | np.uint64(1)
        rows.append(np.unique(np.concatenate([np.array(shared, dtype=np.uint64), private])))
    return rows
