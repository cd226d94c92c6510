"""batch.many_vs_many, multigather's batched first pass and LinearIndex.search_many on the H100: the brute-force cases
of the emulated checks on the device, and 32 configs[4] metagenome queries against one 50 000-row resident database
(the batched range-major pass) compared bit for bit with a loop of one_vs_many."""
import numpy as np
import pytest

from tests.many_vs_many_cases import brute, cases
from tests.test_gpu_multigather import configs4  # noqa: F401 -- the 50 000-row database fixture

pytestmark = pytest.mark.gpu


def test_many_vs_many_vs_bruteforce_on_device():
    from sourmash_b200 import batch as B
    rows, qs = cases()
    want = brute(qs, rows)
    db = B.SketchSet.from_rows(rows)
    got = B.many_vs_many(qs, db)
    assert np.array_equal(got, want)
    assert np.array_equal(got, np.stack([B.one_vs_many(q, db) for q in qs]))
    near = [np.setdiff1d(qs[i % 3], qs[i % 3][i::17]) for i in range(40)]          # queues overflow and drain
    assert np.array_equal(B.many_vs_many(qs[:5], B.SketchSet.from_rows(near)), brute(qs[:5], near))
    import torch
    hashes, offs = B._query_csr(qs)
    d_h = torch.from_numpy(hashes.view(np.int64)).cuda()
    d_c = torch.full((len(qs), len(rows)), 7, dtype=torch.int32, device="cuda")
    B.many_vs_many_device(d_h.data_ptr(), offs, db, d_c.data_ptr())
    assert np.array_equal(d_c.cpu().numpy().view(np.uint32), want)
    db.build_index()
    assert np.array_equal(B.many_vs_many(qs, db), want)


def test_many_vs_many_configs4_equals_one_vs_many(configs4):  # noqa: F811
    from sourmash_b200 import batch as B
    queries, db = configs4
    got = B.many_vs_many(queries, db)
    want = np.stack([B.one_vs_many(q, db) for q in queries])
    assert got.shape == (len(queries), len(db)) and np.array_equal(got, want)
    assert int(got.sum()) > 0
    picks = B.multigather(queries, db, thresholds=50)
    for i, q in enumerate(queries):
        ids, sizes = B.gather(q, db, threshold=50)
        assert picks[i][0].tolist() == ids.tolist() and picks[i][1].tolist() == sizes.tolist(), i


def test_search_many_equals_search_on_device():
    import sourmash_b200 as smb
    from sourmash_b200.index import LinearIndex
    rows, qs = cases()
    subjects = []
    for i, r in enumerate(rows[:100]):
        mh = smb.MinHash(0, 31, scaled=1)
        mh.add_many(r)
        subjects.append(smb.SourmashSignature(mh, name="s%d" % i))
    idx = LinearIndex(subjects)
    queries = []
    for i, q in enumerate([qs[0], qs[2], qs[4], qs[6], qs[7], qs[8], qs[0], qs[4]]):
        mh = smb.MinHash(0, 31, scaled=1)
        mh.add_many(q)
        queries.append(smb.SourmashSignature(mh.downsample(scaled=1 + 3 * (i % 3)), name="q%d" % i))

    def key(res):
        return [(r.score, r.signature.md5sum()) for r in res]
    for kw in (dict(threshold=0.0), dict(threshold=0.01, do_containment=True), dict(threshold=0.0, best_only=True)):
        many = idx.search_many(queries, **kw)
        assert [key(m) for m in many] == [key(idx.search(q, **kw)) for q in queries], kw
    assert sum(len(m) for m in idx.search_many(queries, threshold=0.0)) > 20
    assert [key(m) for m in idx.prefetch_many(queries, 0)] == [key(idx.prefetch(q, 0)) for q in queries]
