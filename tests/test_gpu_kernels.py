"""Parity of the CUDA kernels (through the C ABI) against the CPU oracle.  Needs an H100."""
import numpy as np
import pytest

import oracle as orc
from sourmash_b200.synth import MAX_HASH_1000, rows_of, synth_genome, synth_sketches

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def B():
    from sourmash_b200 import batch
    assert batch.device_count() > 0, "GPU tests need a CUDA device"
    return batch


def _csr(rows):
    return orc.to_csr(rows)


# ---------------------------------------------------------------- sketch path
@pytest.mark.parametrize("k", [21, 31, 51])
def test_ecoli_golden_bit_exact(B, golden, ecoli_seq, k):
    info = golden["meta"]["ecoli"][str(k)]
    seq = np.frombuffer(ecoli_seq, dtype=np.uint8)
    sset, nk = B.sketch_sequences(seq, [0, len(seq)], [k], scaled=1000, seed=info["seed"])
    (row,) = sset.rows()
    assert nk == len(seq) - k + 1
    assert np.array_equal(row, golden["arrays"][f"ecoli_k{k}"])
    assert orc.md5sum(k, row) == info["md5sum"]


def test_ecoli_three_k_one_call(B, golden, ecoli_seq):
    seq = np.frombuffer(ecoli_seq, dtype=np.uint8)
    sset, nk = B.sketch_sequences(seq, [0, len(seq)], [21, 31, 51], scaled=1000)
    rows = sset.rows()
    for r, k in zip(rows, (21, 31, 51)):
        assert np.array_equal(r, golden["arrays"][f"ecoli_k{k}"])


@pytest.mark.parametrize("k", [4, 15, 21, 31, 32, 33, 51, 64, 70])
def test_sketch_vs_oracle_with_bad_bases(B, k):
    # N every 89 bases, lowercase stretch, odd lengths, several records incl. shorter-than-k
    g = synth_genome(200_003, seed=77, n_every=89)
    g[5000:9000] = np.frombuffer(bytes(g[5000:9000]).lower(), dtype=np.uint8)
    recs = [g[:100_001], g[100_001:100_001 + 17], g[100_018:150_000], g[150_000:]]
    seqs = np.concatenate(recs)
    offs = np.cumsum([0] + [len(r) for r in recs]).astype(np.uint64)
    scaled = 50
    mx = orc.max_hash_for_scaled(scaled)
    sset, nk = B.sketch_sequences(seqs, offs, [k], scaled=scaled)
    rows = sset.rows()
    assert len(rows) == len(recs)
    for r, rec in zip(rows, recs):
        assert np.array_equal(r, orc.sketch_scaled(rec, k, mx))
    assert nk == sum(max(len(r) - k + 1, 0) for r in recs)


def test_sketch_records_into_one_sketch_num_mode(B, golden, s10_records):
    seqs = np.concatenate([np.frombuffer(s, dtype=np.uint8) for _, s in s10_records])
    offs = np.cumsum([0] + [len(s) for _, s in s10_records]).astype(np.uint64)
    for k in (21, 30):
        sset, _ = B.sketch_sequences(seqs, offs, [k], num=500,
                                     seq_to_sketch=np.zeros(len(s10_records), dtype=np.uint32), n_sketches=1)
        (row,) = sset.rows()
        assert np.array_equal(row, golden["arrays"][f"s10_k{k}"])


def test_sketch_abundance(B):
    g = synth_genome(50_000, seed=5)
    seq = np.concatenate([g, g[:20_000], g[:10_000]])          # repeated content -> abundances > 1
    k, scaled = 21, 20
    sset, _ = B.sketch_sequences(seq, [0, len(seq)], [k], scaled=scaled, track_abundance=True)
    h, off, ab = sset.to_host(with_abunds=True)
    mh = orc.OracleMinHash(scaled=scaled, ksize=k, track_abundance=True)
    mh.add_sequence(bytes(seq), force=True)
    assert np.array_equal(h, mh.mins())
    assert np.array_equal(ab, mh.abunds())


def test_sketch_scaled_1_keeps_everything(B):
    g = synth_genome(30_000, seed=9)
    sset, _ = B.sketch_sequences(g, [0, len(g)], [31], scaled=1)
    (row,) = sset.rows()
    assert np.array_equal(row, orc.sketch_scaled(g, 31, 2**64 - 1))


def test_sketch_empty_and_short(B):
    g = synth_genome(100, seed=1)
    sset, nk = B.sketch_sequences(g, [0, 0, 10, 100], [31], scaled=10)
    rows = sset.rows()
    assert [len(r) for r in rows[:2]] == [0, 0] and nk == 90 - 31 + 1
    assert np.array_equal(rows[2], orc.sketch_scaled(g[10:], 31, orc.max_hash_for_scaled(10)))


# ---------------------------------------------------------------- intersection path
def test_47_63_counts(B, golden):
    a, b = golden["arrays"]["s47"], golden["arrays"]["s63"]
    sset = B.SketchSet.from_rows([a, b])
    c = B.pairwise_common(sset)
    assert c.tolist() == [[5177, 2529], [2529, 5238]]
    m = B.compare_jaccard(sset)
    assert m[0, 1] == m[1, 0] == 2529 / 7886 and m[0, 0] == m[1, 1] == 1.0
    assert B.one_vs_many(a, sset).tolist() == [5177, 2529]


def test_demo_matrix_num500(B, golden):
    rows = [golden["arrays"][f"demo{i}"] for i in range(7)]
    m = B.compare_jaccard(B.SketchSet.from_rows(rows), num=500)
    assert np.array_equal(m, np.array(golden["meta"]["demo_matrix"]))


def test_scaled100_downsample(B, golden):
    a, b = golden["arrays"]["scaled100_ecoli"], golden["arrays"]["scaled100_salmonella"]
    sset = B.SketchSet.from_rows([a, b])
    assert B.pairwise_common(sset)[0, 1] == 1522
    for scaled, want in ((1000, (175, 9339)), (10000, (9, 900)), (100000, (1, 100))):
        ds = sset.downsample(orc.max_hash_for_scaled(scaled))
        c = int(B.pairwise_common(ds)[0, 1])
        sz = ds.sizes()
        assert (c, int(sz[0] + sz[1] - c)) == want


@pytest.mark.parametrize("n,mean", [(64, 5000), (257, 300), (33, 12000)])
def test_pairwise_vs_oracle_synthetic(B, n, mean):
    h, off = synth_sketches(n, mean=mean, sd=mean // 10, lo=mean // 2, hi=mean * 2, n_families=8,
                            pool=int(mean * 1.2), seed=n)
    sset = B.SketchSet.from_host(h, off)
    got = B.pairwise_common(sset)
    want = orc.pairwise_common(h, off, nthreads=8)
    assert np.array_equal(got, want)
    m = B.compare_jaccard(sset)
    assert np.array_equal(m, orc.compare_all_pairs(h, off, nthreads=8))     # bit-identical f64


def test_pairwise_ragged_and_edge_values(B):
    rng = np.random.Generator(np.random.PCG64(42))
    rows = [np.zeros(0, np.uint64),
            np.array([0], np.uint64),
            np.array([0, 1, 2, 3, 2**64 - 1], np.uint64),
            np.array([2**64 - 1], np.uint64),
            np.array([2**64 - 2, 2**64 - 1], np.uint64),
            np.arange(1, 3000, dtype=np.uint64),                    # dense small values: one bucket
            np.unique(rng.integers(0, 2**63, size=7000, dtype=np.uint64)),
            np.unique(rng.integers(0, 1000, size=400, dtype=np.uint64)),
            np.zeros(0, np.uint64)]
    h, off = _csr(rows)
    sset = B.SketchSet.from_host(h, off)
    assert np.array_equal(B.pairwise_common(sset), orc.pairwise_common(h, off))
    assert np.array_equal(B.compare_jaccard(sset), orc.compare_all_pairs(h, off))
    # rectangular, A != B
    other = B.SketchSet.from_rows(rows[2:7])
    got = B.pairwise_common(sset, other)
    for i, a in enumerate(rows):
        for j, b in enumerate(rows[2:7]):
            assert got[i, j] == orc.count_common(a, b)


def test_pairwise_large_rows_generic_kernel(B):
    rng = np.random.Generator(np.random.PCG64(7))
    base = np.unique(rng.integers(1, 2**60, size=120_000, dtype=np.uint64))
    rows = [base[::2], base[::3], base[:40_000], np.unique(rng.integers(1, 2**60, size=50_000, dtype=np.uint64))]
    h, off = _csr(rows)
    sset = B.SketchSet.from_host(h, off)
    assert np.array_equal(B.pairwise_common(sset), orc.pairwise_common(h, off))


def test_num_pairwise_vs_oracle(B):
    rng = np.random.Generator(np.random.PCG64(11))
    pool = np.unique(rng.integers(1, 2**64 - 1, size=4000, dtype=np.uint64))
    rows = []
    for i in range(12):
        pick = np.sort(rng.choice(pool, size=rng.integers(100, 900), replace=False))
        rows.append(pick[:500])
    h, off = _csr(rows)
    m = B.compare_jaccard(B.SketchSet.from_host(h, off), num=500)
    assert np.array_equal(m, orc.compare_all_pairs(h, off, num=500))


def test_one_vs_many_small_and_large_query(B):
    h, off = synth_sketches(300, mean=2000, sd=200, lo=1000, hi=3000, n_families=5, pool=2500, seed=3)
    rows = rows_of(h, off)
    db = B.SketchSet.from_host(h, off)
    q_small = rows[7]
    assert np.array_equal(B.one_vs_many(q_small, db), orc.one_vs_many(q_small, h, off).astype(np.uint32))
    rng = np.random.Generator(np.random.PCG64(4000))
    q_large = np.unique(np.concatenate([rng.integers(1, MAX_HASH_1000, size=400_000, dtype=np.uint64)] + rows[:40]))
    assert np.array_equal(B.one_vs_many(q_large, db), orc.one_vs_many(q_large, h, off).astype(np.uint32))


def test_one_vs_many_large_query_holding_uint64_max(B):
    """A query too large for shared memory that holds UINT64_MAX (scaled = 1): the padding lanes of the global pass
    carry that key too and must not count (found by the emulated build, tests/test_emulated_library.py)."""
    h, off = synth_sketches(300, mean=300, sd=60, lo=0, hi=600, n_families=4, pool=400, seed=5)
    rows = rows_of(h, off)
    rng = np.random.Generator(np.random.PCG64(6))
    q = np.unique(np.concatenate([rng.integers(1, 2**54, size=60_000, dtype=np.uint64)] + rows[:30] +
                                 [np.array([2**63, 2**64 - 1], dtype=np.uint64)]))
    db = B.SketchSet.from_host(h, off)
    assert np.array_equal(B.one_vs_many(q, db), orc.one_vs_many(q, h, off).astype(np.uint32))
    rows[5] = np.unique(np.concatenate([rows[5], np.array([2**64 - 1], dtype=np.uint64)]))     # and a row that holds it
    h2, off2 = orc.to_csr(rows)
    assert np.array_equal(B.one_vs_many(q, B.SketchSet.from_host(h2, off2)), orc.one_vs_many(q, h2, off2).astype(np.uint32))


def _gather_oracle(query, rows, threshold=1):
    """CounterGather semantics (index/__init__.py:777-909) with the oracle's count_common."""
    q = np.array(query, dtype=np.uint64)
    counts = {j: orc.count_common(q, r) for j, r in enumerate(rows)}
    counts = {j: c for j, c in counts.items() if c > 0}
    out = []
    while counts:
        best = max(counts.values())
        j = min(jj for jj, c in counts.items() if c == best)      # first inserted wins ties
        if best < threshold:
            break
        isect = np.intersect1d(q, rows[j])
        out.append((j, len(isect)))
        for jj in list(counts):
            counts[jj] -= orc.count_common(isect, rows[jj])
            if counts[jj] <= 0:
                del counts[jj]
        q = np.setdiff1d(q, rows[j])
    return out


def test_gather_vs_oracle(B):
    h, off = synth_sketches(120, mean=800, sd=100, lo=400, hi=1200, n_families=6, pool=1000, seed=21)
    rows = rows_of(h, off)
    query = np.unique(np.concatenate([rows[3], rows[10][:500], rows[47][100:700], rows[90][::2], rows[5][:50]]))
    db = B.SketchSet.from_host(h, off)
    ids, sizes = B.gather(query, db, threshold=3)
    want = _gather_oracle(query, rows, threshold=3)
    assert list(zip(ids.tolist(), sizes.tolist())) == want


def test_gather_session_steps_equal_library_loop(B):
    h, off = synth_sketches(80, mean=700, sd=90, lo=300, hi=1000, n_families=5, pool=900, seed=44)
    rows = rows_of(h, off)
    query = np.unique(np.concatenate([rows[2], rows[11][:400], rows[40][100:600], rows[77][::3]]))
    db = B.SketchSet.from_host(h, off)
    ids, sizes = B.gather(query, db, threshold=4)
    sess = B.GatherSession(query, db)
    got = []
    while True:
        cnt, row = sess.peek()
        if cnt < 4:
            break
        isect = sess.intersect(row)
        assert len(isect) == cnt and np.array_equal(isect, np.intersect1d(isect, rows[row]))
        got.append((row, len(isect)))
        if sess.apply(isect) == 0:
            break
    assert got == list(zip(ids.tolist(), sizes.tolist())) == _gather_oracle(query, rows, threshold=4)


def test_one_vs_many_medium_query_and_big_row_gather(B):
    rng = np.random.Generator(np.random.PCG64(91))
    # query of 20 000 hashes: single shared-memory table without occupancy flags
    h, off = synth_sketches(150, mean=3000, sd=400, lo=1500, hi=5000, n_families=4, pool=3600, seed=17)
    rows = rows_of(h, off)
    db = B.SketchSet.from_host(h, off)
    q = np.unique(np.concatenate([rng.integers(1, MAX_HASH_1000, size=20_000, dtype=np.uint64), rows[3], rows[77]]))
    assert 16_380 < len(q) < 28_000
    assert np.array_equal(B.one_vs_many(q, db), orc.one_vs_many(q, h, off).astype(np.uint32))
    # gather over a database whose rows do not fit shared memory (synchronous round path)
    pool = np.unique(rng.integers(1, 2**62, size=200_000, dtype=np.uint64))
    big_rows = [np.sort(rng.choice(pool, size=40_000, replace=False)) for _ in range(6)]
    bdb = B.SketchSet.from_rows(big_rows)
    query = np.unique(np.concatenate([big_rows[2][:30_000], big_rows[4][5_000:25_000], big_rows[0][::7]]))
    ids, sizes = B.gather(query, bdb, threshold=10)
    assert list(zip(ids.tolist(), sizes.tolist())) == _gather_oracle(query, big_rows, threshold=10)


# ---------------------------------------------------------------------------------------------
# inverted join (sort by hash + co-occurrence counts) vs tile kernel vs oracle
# ---------------------------------------------------------------------------------------------
def _with_algo(algo, fn):
    import os
    old = os.environ.get("SMB_COMPARE_ALGO")
    os.environ["SMB_COMPARE_ALGO"] = algo
    try:
        return fn()
    finally:
        if old is None:
            del os.environ["SMB_COMPARE_ALGO"]
        else:
            os.environ["SMB_COMPARE_ALGO"] = old


@pytest.mark.parametrize("seed,n,mean", [(1, 300, 400), (2, 1100, 120), (3, 70, 3000)])
def test_join_and_tile_agree_with_oracle(seed, n, mean):
    from sourmash_b200 import batch as B
    from sourmash_b200.synth import synth_sketches
    h, off = synth_sketches(n, mean=mean, sd=mean // 5, lo=mean // 3, hi=mean * 2, n_families=max(n // 25, 2),
                            pool=int(mean * 1.3), seed=seed)
    want_c = orc.pairwise_common(h, off, nthreads=8)
    want_j = orc.compare_all_pairs(h, off, nthreads=8)
    sset = B.SketchSet.from_host(h, off)
    iu = np.triu_indices(n, 1)
    for algo in ("join", "tile"):
        c = _with_algo(algo, lambda: B.pairwise_common(sset))
        assert np.array_equal(c[iu], want_c[iu]), algo
        assert np.array_equal(_with_algo(algo, lambda: B.compare_jaccard(sset)), want_j), algo


def test_join_edge_cases():
    from sourmash_b200 import batch as B
    rng = np.random.default_rng(0)
    big = np.uint64(2**64 - 1)
    shared = np.unique(rng.integers(0, 2**63, size=50, dtype=np.uint64))
    rows = []
    for i in range(130):
        own = np.unique(rng.integers(0, 2**64 - 1, size=int(rng.integers(0, 40)), dtype=np.uint64))
        parts = [own]
        if i % 3 == 0:
            parts.append(shared)                      # one hash group spanning 44 rows
        if i % 7 == 0:
            parts.append(np.array([0, 1, 2, big], dtype=np.uint64))
        rows.append(np.unique(np.concatenate(parts)) if i != 5 else np.zeros(0, np.uint64))   # row 5 empty
    rows[10] = rows[9].copy()                         # identical rows
    dense = [np.arange(i % 5, 40, dtype=np.uint64) for i in range(70)]   # tiny dense keys: every hash in ~all rows
    # two hashes shared by thousands of rows: groups far longer than the kernel's staged window
    wide = [np.unique(np.concatenate([rng.integers(1, 2**60, size=3, dtype=np.uint64),
                                      np.array([7] if i % 4 else [7, 2**61], dtype=np.uint64)])) for i in range(3300)]
    for rr in (rows, dense, wide):
        h, off = orc.to_csr(rr)
        n = len(rr)
        want = orc.pairwise_common(h, off)
        sset = B.SketchSet.from_host(h, off)
        iu = np.triu_indices(n, 1)
        for algo in ("join", "tile"):
            assert np.array_equal(_with_algo(algo, lambda: B.pairwise_common(sset))[iu], want[iu]), algo
            assert np.array_equal(_with_algo(algo, lambda: B.compare_jaccard(sset)), orc.compare_all_pairs(h, off)), algo


def test_join_key_range_shards_sum_to_full():
    import torch
    from sourmash_b200 import batch as B
    from sourmash_b200.synth import synth_sketches
    n = 400
    h, off = synth_sketches(n, mean=300, sd=60, lo=100, hi=600, n_families=8, pool=400, seed=4)
    sset = B.SketchSet.from_host(h, off)
    want = orc.pairwise_common(h, off, nthreads=8)
    iu = np.triu_indices(n, 1)
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    for algo in ("join", "tile"):
        for shards in (1, 3, 8):
            total = torch.zeros((n, n), dtype=torch.int32, device="cuda")
            for r in range(shards):
                part = torch.zeros((n, n), dtype=torch.int32, device="cuda")
                _with_algo(algo, lambda: B.pairwise_counts_shard_device(sset, r, shards, part.data_ptr()))
                total += part
            torch.cuda.synchronize()
            assert np.array_equal(total.cpu().numpy().astype(np.uint32)[iu], want[iu]), (algo, shards)
    B.set_stream(0)
