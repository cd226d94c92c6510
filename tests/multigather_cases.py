"""Cases of the multigather tests shared by the emulated checks (tests/host_emul/multigather_checks.py) and the GPU
tests (tests/test_gpu_multigather.py): a brute force of the reference's gather loop for one query with Python sets
(CounterGather + GatherDatabases: index/__init__.py:777-909, search.py:877-949) and a small workload with a tie, a
query without candidates, a query that is consumed completely and queries of very different lengths."""
import numpy as np

from sourmash_b200.synth import rows_of, synth_sketches

NONE = 0xffffffff


def brute_multigather(query, rows, threshold=1, min_count=1, max_rounds=None):
    """The reference loop for one query with Python sets: counters of the rows sharing at least min_count hashes (in
    row order, the first one wins ties), pick while the best counter is >= threshold (and > 0).  Returns rows, sizes
    and, per query hash, the round that took it."""
    q = [int(x) for x in query]
    sets = [set(int(x) for x in r) for r in rows]
    counters = {}
    for i, r in enumerate(sets):
        c = len(r.intersection(q))
        if c and c >= max(min_count, 1):
            counters[i] = c
    remaining = set(q)
    taken = {}
    picks, sizes = [], []
    while remaining and counters and (max_rounds is None or len(picks) < max_rounds):
        best = max(counters.values())
        if best == 0 or best < max(threshold, 1):
            break
        i = next(k for k, v in counters.items() if v == best)
        isect = remaining & sets[i]
        for h in isect:
            taken[h] = len(picks)
        picks.append(i)
        sizes.append(len(isect))
        for k in counters:
            counters[k] -= len(isect & sets[k])
        remaining -= isect
    return picks, sizes, [taken.get(h, NONE) for h in q]


def assert_same(got, want, what):
    rows, sizes, consumed = got
    assert rows.tolist() == want[0], (what, rows.tolist()[:10], want[0][:10])
    assert sizes.tolist() == want[1], (what, sizes.tolist()[:10], want[1][:10])
    assert consumed.tolist() == want[2], what


def workload():
    h, off = synth_sketches(240, mean=220, sd=50, lo=0, hi=420, n_families=4, pool=300, seed=11)
    rows = rows_of(h, off)
    rows[17] = rows[4].copy()                                          # exact tie: the first row must win
    rng = np.random.Generator(np.random.PCG64(12))
    queries = [
        np.unique(np.concatenate([rows[4], rows[9][:150], rows[25][50:200], rows[41][::2]])),
        np.unique(rng.integers(1, 2**54, size=300, dtype=np.uint64)),                       # no candidates
        np.unique(rows[8].copy()),                                                          # consumed completely
        np.unique(np.concatenate([rows[i][::3] for i in range(0, 200, 5)])),                # long
        rows[33][:5].copy(),                                                                # short
        np.unique(np.concatenate([rows[2], rows[6][:60], rows[10][::4]])),
    ]
    return rows, queries
