"""batch.multigather and gather.gather_many on the H100: the brute-force cases of the emulated checks on the device,
and 32 configs[4]-style metagenome queries against one 50 000-row resident database, every query compared with the
single-query paths (batch.gather for the picks, gather_databases for the report).  The configs[4] queries hold
~1.4e5 hashes, more than the shared-memory table takes: their first counters come from the range-major pass."""
import numpy as np
import pytest

from tests.multigather_cases import NONE, assert_same, brute_multigather, workload

pytestmark = pytest.mark.gpu

N_DB = 50_000
N_QUERIES = 32
BLOCK = 6250


def test_multigather_vs_bruteforce_on_device():
    from sourmash_b200 import batch as B
    rows, queries = workload()
    db = B.SketchSet.from_rows(rows)
    thresholds, min_counts = [5, 1, 1, 3, 1, 40], [1, 1, 1, 8, 1, 30]
    got = B.multigather(queries, db, thresholds, min_counts)
    for i, q in enumerate(queries):
        assert_same(got[i], brute_multigather(q, rows, thresholds[i], min_counts[i]), i)
    assert len(got[1][0]) == 0 and (got[2][2] != NONE).all() and 17 not in got[0][0].tolist()
    capped = B.multigather(queries, db, thresholds, min_counts, max_rounds=2)
    for i, q in enumerate(queries):
        assert_same(capped[i], brute_multigather(q, rows, thresholds[i], min_counts[i], max_rounds=2), ("cap", i))
    db.build_index()
    for i, r in enumerate(B.multigather(queries, db, thresholds, min_counts)):
        assert_same(r, brute_multigather(queries[i], rows, thresholds[i], min_counts[i]), ("index", i))


@pytest.fixture(scope="module")
def configs4():
    import torch

    from sourmash_b200 import batch as B
    from sourmash_b200.synth import database_block, multigather_workload
    queries, sizes, frac, overrides = multigather_workload(N_DB, N_QUERIES)
    dev = torch.device("cuda")
    h_off = np.zeros(N_DB + 1, dtype=np.uint64)
    h_off[1:] = np.cumsum(sizes)
    d_h = torch.empty(int(h_off[-1]), dtype=torch.int64, device=dev)
    for b in range(0, N_DB, BLOCK):
        e = min(b + BLOCK, N_DB)
        d_h[int(h_off[b]):int(h_off[e])] = database_block(sizes, frac, np.zeros(1, np.uint64), b, e, 5002,
                                                          overrides=overrides, torch=torch, device=dev)
    d_off = torch.from_numpy(h_off.view(np.int64)).to(dev)
    db = B.SketchSet.from_device(d_h.data_ptr(), d_off.data_ptr(), h_off, keepalive=(d_h, d_off))
    return queries, db


def test_multigather_configs4_picks_equal_gather(configs4):
    from sourmash_b200 import batch as B
    queries, db = configs4
    stats = {}
    got = B.multigather(queries, db, thresholds=50, stats=stats)
    total = 0
    for i, q in enumerate(queries):
        ids, sizes = B.gather(q, db, threshold=50)
        assert got[i][0].tolist() == ids.tolist() and got[i][1].tolist() == sizes.tolist(), i
        assert int((got[i][2] != NONE).sum()) == int(sizes.sum())
        total += len(ids)
    assert total > 20 * N_QUERIES
    one = {}
    slowest = max(range(len(queries)), key=lambda i: len(got[i][0]))
    B.multigather([queries[slowest]], db, thresholds=50, stats=one)
    assert stats["round_launches"] <= one["round_launches"] + 3 * 16, (stats, one)


def test_gather_many_configs4_equals_gather_databases(configs4):
    import sourmash_b200 as smb
    from sourmash_b200.gather import gather_databases, gather_many
    queries, db = configs4
    mhs = []
    for q in queries:
        mh = smb.MinHash(0, 31, scaled=1000)
        mh.add_many(q)
        mhs.append(mh)
    names = ["row%d" % r for r in range(N_DB)]
    many = gather_many(mhs, db, threshold_bp=50_000, names=names, query_names=["q%d" % i for i in range(len(mhs))])
    for i, mh in enumerate(mhs):
        assert many[i] == gather_databases(mh, db, threshold_bp=50_000, names=names, query_name="q%d" % i), i
    assert all(len(x) > 20 for x in many)
