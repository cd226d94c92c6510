"""Parity of the Python object model (MinHash / SourmashSignature / compare / index), whose
compute goes through the reference-compatible C ABI to the GPU, against the oracle and the
reference's golden vectors.  Written to read like the reference's own tests
(tests/test_minhash.py, test_compare.py, test_index_protocol.py)."""
import numpy as np
import pytest

import oracle as orc
from sourmash_b200.synth import rows_of, synth_genome, synth_sketches

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def smb():
    import sourmash_b200
    assert sourmash_b200.batch.device_count() > 0
    return sourmash_b200


def _mh(smb, hashes, ksize=31, scaled=1000, **kw):
    mh = smb.MinHash(0, ksize, scaled=scaled, **kw)
    mh.add_many(hashes)
    return mh


def _sig(smb, hashes, name, **kw):
    return smb.SourmashSignature(_mh(smb, hashes, **kw), name=name)


# ---------------------------------------------------------------- hashing through kmerminhash_*
def test_hash_murmur_kat(smb, golden):
    assert smb.hash_murmur("ACG", 42) == golden["meta"]["kat"]["hash_murmur_ACG_42"]     # test_minhash.py:1239
    assert smb.hash_murmur(b"ACG") == smb.hash_murmur("ACG")
    for s in ("", "A", "ACGTACGTACGTACGTACGTA", "x" * 16, "y" * 33):
        assert smb.hash_murmur(s, 7) == orc.hash_murmur(s, 7)


def test_basic_dna(smb, golden):
    mh = smb.MinHash(1, 4)
    mh.add_sequence("ATGC")
    assert list(mh.hashes) == golden["meta"]["kat"]["n1_k4_ATGC"]                        # test_minhash.py:98-112
    mh.add_sequence("GCAT")                                                                # revcomp -> same hash
    assert len(mh) == 1


def test_add_sequence_ecoli_golden_all_k(smb, golden, ecoli_seq):
    for k in (21, 31, 51):
        info = golden["meta"]["ecoli"][str(k)]
        mh = smb.MinHash(0, k, scaled=1000)
        mh.add_sequence(ecoli_seq, force=True)
        assert mh._mins_array().tolist() == golden["arrays"][f"ecoli_k{k}"].tolist()
        assert mh.md5sum() == info["md5sum"]


def test_signature_add_sequence_three_ksizes(smb, golden, ecoli_seq):
    sig = smb.SourmashSignature.from_params(smb.ComputeParameters(ksizes=[21, 31, 51], scaled=1000))
    sig.add_sequence(ecoli_seq[:1_000_000], force=True)
    for mh in sig.sketches():
        want = orc.sketch_scaled(ecoli_seq[:1_000_000], mh.ksize, mh._max_hash)
        assert np.array_equal(mh._mins_array(), want)


def test_merge_kat_through_add_sequence(smb, golden):
    kat = golden["meta"]["kat"]["merge_k10_num20"]                                        # src/core/tests/minhash.rs:29-54
    a, b = smb.MinHash(20, 10), smb.MinHash(20, 10)
    for s in kat["a"]:
        a.add_sequence(s)
    for s in kat["b"]:
        b.add_sequence(s)
    a.merge(b)
    assert list(a.hashes) == kat["merged"]


def test_invalid_dna_semantics(smb):
    mh = smb.MinHash(20, 3)
    mh.add_sequence("AAANNCCCTN", force=True)                                              # tests/minhash.rs:56-66
    assert len(mh) == 3
    mh2 = smb.MinHash(20, 3)
    mh2.add_sequence("NAAA", True)
    assert len(mh2) == 1
    e = smb.MinHash(1, 4)
    with pytest.raises(ValueError, match="invalid DNA character in input k-mer: ATGR"):    # test_minhash.py:719
        e.add_sequence("ATGR")
    assert len(e) == 0
    p = smb.MinHash(50, 3)
    with pytest.raises(ValueError, match="invalid DNA character in input k-mer: AAN"):
        p.add_sequence("aaanncc")                                                          # upper-cased in the message
    assert len(p) == 1                                                                      # "AAA" went in before the error
    q = smb.MinHash(0, 21, scaled=1)
    q.add_sequence("N" * 100, force=True)                                                  # test_minhash.py:197-203
    assert len(q) == 0
    s = smb.MinHash(10, 21)
    s.add_sequence("ACGT")                                                                 # shorter than k: no hashes, no error
    assert len(s) == 0
    lo, up = smb.MinHash(0, 5, scaled=1), smb.MinHash(0, 5, scaled=1)
    lo.add_sequence("acgtacgtggcca"); up.add_sequence("ACGTACGTGGCCA")                    # test_minhash.py:755-765
    assert lo == up and len(lo) > 0


def test_seq_to_hashes(smb):
    mh = smb.MinHash(0, 21, scaled=1)
    seq = bytes(synth_genome(3000, seed=3, n_every=97))
    want0, _ = orc.seq_to_hashes(seq, 21, force=True, keep_zeros=True)
    want, _ = orc.seq_to_hashes(seq, 21, force=True)
    assert mh.seq_to_hashes(seq, force=True, bad_kmers_as_zeroes=True) == want0.tolist()  # test_minhash.py:265-281
    assert len(want0) == len(seq) - 21 + 1
    assert mh.seq_to_hashes(seq, force=True) == want.tolist()
    with pytest.raises(ValueError, match="invalid DNA character"):
        mh.seq_to_hashes(seq)
    with pytest.raises(ValueError):
        mh.seq_to_hashes(seq, bad_kmers_as_zeroes=True)
    clean = bytes(synth_genome(500, seed=4))
    assert mh.seq_to_hashes(clean) == orc.seq_to_hashes(clean, 21)[0].tolist()
    assert len(mh) == 0
    kh = list(mh.kmers_and_hashes(clean[:40].decode()))
    assert [h for _, h in kh] == orc.seq_to_hashes(clean[:40], 21)[0].tolist() and kh[0][0] == clean[:21].decode()
    g = smb.MinHash(0, 7, scaled=1)                                                         # generic-k kernel
    assert g.seq_to_hashes(clean) == orc.seq_to_hashes(clean, 7)[0].tolist()


def test_num_and_abundance_add_sequence(smb, golden, s10_records):
    for k in (21, 30):
        mh = smb.MinHash(500, k)
        for _, seq in s10_records:
            mh.add_sequence(seq, force=True)
        assert mh.md5sum() == golden["meta"]["genome_s10"][str(k)]["md5sum"]
    g = bytes(synth_genome(30_000, seed=8))
    seq = g + g[:9000]
    for num, scaled in ((0, 10), (300, 0)):
        mh = smb.MinHash(num, 21, scaled=scaled, track_abundance=True)
        om = orc.OracleMinHash(scaled=scaled, ksize=21, num=num, track_abundance=True)
        for chunk in (seq[:20_000], seq[20_000:]):                 # two calls: second merges into existing
            mh.add_sequence(chunk, force=True)
            om.add_sequence(chunk, force=True)
        assert mh._mins_array().tolist() == om.mins().tolist()
        assert mh._abunds_array().tolist() == om.abunds().tolist()


# ---------------------------------------------------------------- pair operations
def test_pair_operations_47_63(smb, golden):
    a, b = _mh(smb, golden["arrays"]["s47"]), _mh(smb, golden["arrays"]["s63"])
    assert a.count_common(b) == 2529 and b.count_common(a) == 2529                         # test_prefetch.py:272
    assert a.intersection_and_union_size(b) == (2529, 7886)
    assert a.jaccard(b) == 2529 / 7886 == a.similarity(b)
    assert round(a.similarity(b), 2) == 0.32 and round(b.contained_by(a), 2) == 0.48       # test_index_protocol.py:217-269
    assert a.contained_by(b) == pytest.approx(2529 / 5177, rel=1e-3)
    i = a & b
    assert len(i) == 2529 and i._mins_array().tolist() == np.intersect1d(a._mins_array(), b._mins_array()).tolist()
    assert a.max_containment(b) == a.contained_by(b) and a.avg_containment(b) == (a.contained_by(b) + b.contained_by(a)) / 2
    u = a + b
    assert len(u) == 7886
    empty = smb.MinHash(0, 31, scaled=1000)
    assert a.jaccard(empty) == 0.0 and empty.jaccard(empty) == 0.0 and empty.contained_by(a) == 0.0


def test_jaccard_small_exact(smb):
    a, b = smb.MinHash(0, 20, scaled=1), smb.MinHash(0, 20, scaled=1)                      # test_jaccard.py:16-56
    a.add_many([1, 3, 5, 8]); b.add_many([1, 3, 5, 6, 8, 10])
    assert a.jaccard(b) == 4.0 / 6.0 == b.jaccard(a) and a.similarity(a) == 1.0
    n1, n2 = smb.MinHash(5, 20), smb.MinHash(5, 20)
    n1.add_many([1, 2, 3, 4, 5]); n2.add_many([1, 2, 3, 4, 6])
    assert n1.jaccard(n2) == 4.0 / 5.0                                                      # bottom-5 of the union
    with pytest.raises(ValueError, match="different ksizes"):
        a.jaccard(smb.MinHash(0, 21, scaled=1))
    with pytest.raises(ValueError, match="mismatch in scaled"):
        a.count_common(smb.MinHash(0, 20, scaled=2))


def test_scaled_downsample_on_real_data(smb, golden):
    a = _mh(smb, golden["arrays"]["scaled100_ecoli"], ksize=21, scaled=100)
    b = _mh(smb, golden["arrays"]["scaled100_salmonella"], ksize=21, scaled=100)
    assert round(a.similarity(b), 5) == 0.01644                                            # test_jaccard.py:205-264
    a1, b1 = a.downsample(scaled=1000), b.downsample(scaled=1000)
    assert round(a1.similarity(b1), 5) == 0.01874
    assert round(a.similarity(b1, downsample=True), 5) == 0.01874                          # on-the-fly downsample
    assert a.count_common(b1, downsample=True) == 175
    with pytest.raises(ValueError, match="mismatch in scaled"):
        a.similarity(b1)
    a2, b2 = a1.downsample(scaled=10000), b1.downsample(scaled=10000)
    assert a2.similarity(b2) == 0.01


def test_num_on_real_data(smb, golden):
    a = smb.MinHash(10000, 21); a.add_many(golden["arrays"]["n10000_ecoli"])
    b = smb.MinHash(10000, 21); b.add_many(golden["arrays"]["n10000_salmonella"])
    assert a.similarity(b) == 0.0183 == b.similarity(a)                                    # test_jaccard.py:175-202
    a, b = a.downsample(num=1000), b.downsample(num=1000)
    assert a.similarity(b) == 0.011
    a, b = a.downsample(num=100), b.downsample(num=100)
    assert a.similarity(b) == 0.01
    assert a.intersection_and_union_size(b) == (1, 100)


def test_angular_similarity(smb):
    rng = np.random.Generator(np.random.PCG64(5))
    ha = np.unique(rng.integers(1, 10**9, size=400, dtype=np.uint64))
    hb = np.unique(np.concatenate([ha[::2], rng.integers(1, 10**9, size=200, dtype=np.uint64)]))
    aa, bb = rng.integers(1, 20, size=len(ha)), rng.integers(1, 20, size=len(hb))
    a = smb.MinHash(0, 21, scaled=1, track_abundance=True); a.set_abundances(dict(zip(ha.tolist(), aa.tolist())))
    b = smb.MinHash(0, 21, scaled=1, track_abundance=True); b.set_abundances(dict(zip(hb.tolist(), bb.tolist())))
    want = orc.angular_similarity(ha, aa, hb, bb)
    assert abs(a.angular_similarity(b) - want) < 1e-12 and abs(a.similarity(b) - want) < 1e-12
    assert a.similarity(b, ignore_abundance=True) == orc.jaccard(ha, hb)
    assert abs(a.angular_similarity(a) - 1.0) < 1e-7
    with pytest.raises(TypeError):
        a.angular_similarity(a.flatten())


# ---------------------------------------------------------------- compare
def test_compare_serial_demo_matrix(smb, golden):
    from sourmash_b200.compare import compare_all_pairs, compare_serial
    sigs = []
    for i in range(7):
        mh = smb.MinHash(500, 31); mh.add_many(golden["arrays"][f"demo{i}"])
        sigs.append(smb.SourmashSignature(mh, name=f"demo{i}"))
    want = np.array(golden["meta"]["demo_matrix"])
    assert np.array_equal(compare_serial(sigs, True), want)                                # test_compare.py:49-61
    assert np.array_equal(compare_all_pairs(sigs, True, n_jobs=2), want)


def test_compare_matrices_vs_per_pair_calls(smb):
    from sourmash_b200 import compare as C
    h, off = synth_sketches(24, mean=1500, sd=300, lo=200, hi=2500, n_families=4, pool=1800, seed=9)
    rows = rows_of(h, off) + [np.zeros(0, np.uint64)]
    sigs = [_sig(smb, r, f"s{i}") for i, r in enumerate(rows)]
    n = len(sigs)
    sim = C.compare_all_pairs(sigs, ignore_abundance=True)
    cont = C.compare_serial_containment(sigs)
    mx = C.compare_serial_max_containment(sigs)
    avg = C.compare_serial_avg_containment(sigs)
    for i in range(n):
        for j in range(n):
            a, b = sigs[i].minhash, sigs[j].minhash
            if i == j:
                assert sim[i, j] == cont[i, j] == mx[i, j] == avg[i, j] == 1.0
                continue
            assert sim[i, j] == orc.jaccard(rows[i], rows[j])                              # bit-exact f64
            assert cont[i, j] == b.contained_by(a)                                         # compare.py:97 orientation
            assert mx[i, j] == a.max_containment(b)
            assert avg[i, j] == a.avg_containment(b)
    with pytest.raises(ValueError, match="different ksizes"):
        C.compare_all_pairs(sigs[:2] + [_sig(smb, rows[0], "k21", ksize=21)], True)


def test_compare_abundance_angular_matrix(smb):
    from sourmash_b200 import compare as C
    rng = np.random.Generator(np.random.PCG64(77))
    pool = np.unique(rng.integers(1, 10**12, size=3000, dtype=np.uint64))
    sigs = []
    for i in range(9):
        pick = np.sort(rng.choice(pool, size=int(rng.integers(200, 1500)), replace=False))
        mh = smb.MinHash(0, 21, scaled=1, track_abundance=(i != 4))
        if i != 4:
            mh.set_abundances(dict(zip(pick.tolist(), rng.integers(1, 50, size=len(pick)).tolist())))
        else:
            mh.add_many(pick)
        sigs.append(smb.SourmashSignature(mh, name=f"a{i}"))
    m = C.compare_all_pairs(sigs, ignore_abundance=False)
    mi = C.compare_all_pairs(sigs, ignore_abundance=True)
    for i in range(9):
        for j in range(9):
            if i == j:
                assert m[i, j] == 1.0
                continue
            a, b = sigs[i].minhash, sigs[j].minhash
            assert abs(m[i, j] - a.similarity(b)) < 1e-12                     # angular, or jaccard if one is flat
            assert mi[i, j] == a.similarity(b, ignore_abundance=True)
            if i != 4 and j != 4:
                ha, hb = a.hashes, b.hashes
                want = orc.angular_similarity(list(ha), list(ha.values()), list(hb), list(hb.values()))
                assert abs(m[i, j] - want) < 1e-12


def test_compare_downsample_mixed_scaled(smb):
    from sourmash_b200 import compare as C
    h, off = synth_sketches(6, mean=3000, sd=300, lo=2000, hi=4000, n_families=2, pool=3500, seed=2)
    rows = rows_of(h, off)
    sigs = [_sig(smb, r, f"s{i}", scaled=1000 if i % 2 else 2000) for i, r in enumerate(rows)]
    with pytest.raises(ValueError, match="mismatch in scaled"):
        C.compare_all_pairs(sigs, True)
    # the reference downsamples per pair to max(scaled_i, scaled_j) (similarity(other, downsample=True),
    # minhash.rs:682-702): two scaled=1000 sketches are compared at 1000 although the list holds 2000s
    m = C.compare_all_pairs(sigs, True, downsample=True)
    ds = {sc: [orc.downsample(r, orc.max_hash_for_scaled(sc)) for r in rows] for sc in (1000, 2000)}
    for i in range(6):
        for j in range(i + 1, 6):
            sc = 1000 if (i % 2 and j % 2) else 2000
            assert m[i, j] == m[j, i] == orc.jaccard(ds[sc][i], ds[sc][j])
            assert m[i, j] == sigs[i].minhash.similarity(sigs[j].minhash, ignore_abundance=True, downsample=True)
    cm = C.compare_serial_containment(sigs, downsample=True)
    for i in range(6):
        for j in range(6):
            if i != j:                                      # compare.py:97-99
                assert cm[i, j] == sigs[j].minhash.contained_by(sigs[i].minhash, downsample=True)


# ---------------------------------------------------------------- search / prefetch / gather
def test_index_search_prefetch(smb, golden):
    from sourmash_b200.index import LinearIndex
    s47, s63 = _sig(smb, golden["arrays"]["s47"], "47"), _sig(smb, golden["arrays"]["s63"], "63")
    other = _sig(smb, np.arange(1, 4000, dtype=np.uint64) * 1000003, "other")
    idx = LinearIndex([s47, s63, other], filename="mem")
    sr = idx.search(s47, threshold=0.1)                                                    # test_index_protocol.py:217-269
    assert [r.signature.name for r in sr] == ["47", "63"] and sr[0].score == 1.0
    assert round(sr[1].score, 2) == 0.32 and sr[1].location == "mem"
    sr = idx.search(s47, threshold=0.1, do_containment=True)
    assert sr[1].score == 2529 / 5177
    sr = idx.search(s47, threshold=0.1, do_max_containment=True)
    assert sr[1].score == 2529 / 5177
    assert [r.signature.name for r in idx.search(s47, threshold=0.9)] == ["47"]
    pf = list(idx.prefetch(s47, threshold_bp=0))
    assert [r.signature.name for r in pf] == ["47", "63"]
    assert [r.signature.name for r in idx.prefetch(s47, threshold_bp=3_000_000)] == ["47"]
    with pytest.raises(ValueError):
        list(idx.prefetch(s47, threshold_bp=10**10))
    with pytest.raises(TypeError):
        idx.search(s47)
    # mixed scaled: subject finer than the query and vice versa (index/__init__.py:133-141)
    fine = _sig(smb, golden["arrays"]["scaled100_ecoli"], "ecoli100", ksize=21, scaled=100)
    coarse_q = smb.SourmashSignature(fine.minhash.downsample(scaled=1000), name="q1000")
    idx2 = LinearIndex([fine])
    (r,) = idx2.search(coarse_q, threshold=0.5)
    assert r.score == 1.0
    (r,) = LinearIndex([coarse_q]).search(fine, threshold=0.5, do_containment=True)
    assert r.score == 1.0


def _gather_reference_loop(smb, query_sig, sigs, threshold_bp):
    """The reference algorithm with per-pair calls (search.py:877-949 + CounterGather)."""
    scaled = query_sig.minhash.scaled
    cur = query_sig.minhash.to_mutable()
    remaining = list(sigs)
    out = []
    while remaining and len(cur):
        best, best_c = None, 0
        for s in remaining:
            c = cur.count_common(s.minhash)
            if c > best_c:
                best, best_c = s, c
        if best is None or best_c * scaled < threshold_bp or best_c == 0:
            break
        out.append((best.name, best_c))
        cur.remove_many(best.minhash)
        remaining = [s for s in remaining if s is not best]
    return out


def test_gather_matches_reference_loop(smb):
    from sourmash_b200.index import CounterGather, LinearIndex, gather
    h, off = synth_sketches(40, mean=600, sd=80, lo=300, hi=900, n_families=4, pool=800, seed=33)
    rows = rows_of(h, off)
    sigs = [_sig(smb, r, f"g{i}") for i, r in enumerate(rows)]
    q = np.unique(np.concatenate([rows[3], rows[8][:300], rows[21][100:500], rows[30][::2], rows[5][:20]]))
    query = _sig(smb, q, "query")
    idx = LinearIndex(sigs)
    for tbp in (0, 50_000):
        got = [(r.match.name, r.intersect_size) for r in gather(query, idx, threshold_bp=tbp)]
        assert got == _gather_reference_loop(smb, query, sigs, tbp)
        assert len(got) >= 3
    # batched C-ABI gather gives the same picks
    ids, sizes = smb.batch.gather(q, smb.batch.SketchSet.from_rows(rows), threshold=1)
    want = _gather_reference_loop(smb, query, sigs, 0)
    assert [(f"g{i}", s) for i, s in zip(ids.tolist(), sizes.tolist())] == want
    # CounterGather protocol details (test_index_protocol.py:766-1312)
    cg = CounterGather(query)
    with pytest.raises(ValueError, match="no overlap"):
        cg.add(_sig(smb, np.array([7, 11], dtype=np.uint64), "none"))
    cg.add(sigs[3]); cg.add(sigs[8])
    assert {s.name for s in cg.signatures()} == {"g3", "g8"}
    res, isect = cg.peek(query.minhash)
    assert res.signature.name == "g3" and len(isect) == len(rows[3])
    with pytest.raises(ValueError, match="cannot add more"):
        cg.add(sigs[5])
    cg.consume(isect)
    res2, isect2 = cg.peek(query.minhash.to_mutable().__isub__(isect) if False else _minus(smb, query.minhash, isect))
    assert res2.signature.name == "g8"
    assert len(cg.union_found) == len(np.union1d(np.intersect1d(q, rows[3]), np.intersect1d(q, rows[8])))
    with pytest.raises(ValueError, match="requires scaled"):
        CounterGather(smb.SourmashSignature(smb.MinHash(10, 31), name="num"))


def _minus(smb, mh, remove):
    m = mh.to_mutable()
    m.remove_many(remove)
    return m


def test_sketch_fasta_files_matches_golden_signatures(smb, golden):
    """`sourmash sketch dna` on the two reference genomes -> the reference's own .sig contents."""
    import os
    from sourmash_b200.sketch import read_sequences, sketch_fasta_files
    from tests.conftest import GOLDEN, ecoli_k12_path
    ecoli, s10 = ecoli_k12_path(), os.path.join(GOLDEN, "genome-s10.fa.gz")
    sigs = sketch_fasta_files([ecoli, s10], ksizes=[21, 31, 51], scaled=1000, name_from_first=True)
    assert len(sigs) == 2 and len(sigs[0]) == 3 and sigs[0].filename == ecoli
    assert sigs[0].name.startswith("NC_000913.3 Escherichia coli")
    for mh in sigs[0].sketches():
        assert mh.md5sum() == golden["meta"]["ecoli"][str(mh.ksize)]["md5sum"]
    # num=500 sketches of the multi-record file equal the reference's golden sig
    nsig, = sketch_fasta_files([s10], ksizes=[21, 30], scaled=0, num=500)
    assert [m.md5sum() for m in nsig.sketches()] == [golden["meta"]["genome_s10"][k]["md5sum"] for k in ("21", "30")]
    # singleton: one signature per record; abundance tracking
    recs = read_sequences(s10)
    single = sketch_fasta_files([s10], ksizes=[21], scaled=100, singleton=True, track_abundance=True)
    assert len(single) == len(recs) and single[0].name == recs[0][0]
    om = orc.OracleMinHash(scaled=100, ksize=21, track_abundance=True)
    om.add_sequence(recs[0][1], force=True)
    assert single[0].minhash._mins_array().tolist() == om.mins().tolist()
    assert single[0].minhash._abunds_array().tolist() == om.abunds().tolist()
    # --merge: all records of all files in one signature (command_sketch.py:791-824)
    merged, = sketch_fasta_files([ecoli, s10], ksizes=[31], scaled=1000, merge="both")
    k31 = [next(m for m in s.sketches() if m.ksize == 31) for s in sigs]
    assert merged.name == "both" and merged.filename == s10
    assert merged.minhash._mins_array().tolist() == sorted(set(k31[0].hashes) | set(k31[1].hashes))
    # --check-sequence semantics
    import tempfile
    with tempfile.NamedTemporaryFile("w", suffix=".fa", delete=False) as fh:
        fh.write(">bad\nACGTACGTNACGTACGTACGTAGCATGCATGCA\n")
    with pytest.raises(ValueError, match="invalid DNA character"):
        sketch_fasta_files([fh.name], ksizes=[5], scaled=1, check_sequence=True)
    ok, = sketch_fasta_files([fh.name], ksizes=[5], scaled=1)
    assert len(ok.minhash) > 0
    os.unlink(fh.name)


def test_compare_of_num_sketches_of_different_sizes_follows_the_reference_pair_by_pair(smb):
    """The reference does not refuse num sketches of different num: cells (i, j) and (j, i) are siglist[i].similarity(siglist[j])
    for i < j, and that value depends on which sketch is self (compare.py:36-54, minhash.rs:596-617).  A scaled sketch against
    a num sketch is 'mismatch in scaled', as there."""
    from sourmash_b200 import compare as CMP
    a, b, c = smb.MinHash(10, 21), smb.MinHash(20, 21), smb.MinHash(10, 21)
    for i in range(40):
        a.add_hash(i * 3 + 1); b.add_hash(i * 2 + 1); c.add_hash(i * 5 + 1)
    sigs = [smb.SourmashSignature(m, name=n) for m, n in ((a, "a"), (b, "b"), (c, "c"))]
    m = CMP.compare_all_pairs(sigs, True)
    assert m[0][1] == m[1][0] == a.similarity(b) == 0.3 and m[1][2] == m[2][1] == b.similarity(c) and m[0][2] == a.similarity(c)
    assert b.similarity(a) == 0.25                                  # why this cannot be one symmetric batched matrix
    with pytest.raises(TypeError, match="incompatible num values"):
        CMP._collect(sigs, downsample=False)
    scaled = smb.SourmashSignature(_mh(smb, range(1, 100, 3), ksize=21, scaled=1), name="s")
    for order in ([scaled, sigs[1]], [sigs[1], scaled]):
        with pytest.raises(ValueError, match="mismatch in scaled; comparison fail"):
            CMP.compare_all_pairs(order, True)
