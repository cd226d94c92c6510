"""GPU parity of the stripe join's stream sorted from the hashes themselves (csrc/join_stripe.cuh: stripe_hash_tag_kernel,
stripe_hash_fix_kernel) at the benchmark's shape: the 10 000 x 10 000 matrices of synth_sketches(10 000), of the same size
with a pool per row (n_families = 10 000), and of a set whose hashes all lie below 2^34 (synth_sketches(10 000,
max_hash=2^34): the sort window then holds the top 32 of 34 bits, and runs of equal window bits that mix hashes are
common), compared bit for bit with the global-reduction join (SMB_JOIN_LAYOUT=plain), which builds no stream.  Small
sets, narrow windows and key-range shards are covered on the CPU by tests/test_stripe_hash_sort_simt.py."""
import numpy as np
import pytest

from sourmash_b200.synth import synth_sketches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kw", [{}, {"n_families": 10_000}, {"max_hash": 2**34}])
def test_stripe_hash_sort_matrix_matches_plain_join(monkeypatch, kw):
    from sourmash_b200 import batch as B
    h, off = synth_sketches(10_000, **kw)
    monkeypatch.setenv("SMB_COMPARE_ALGO", "join")
    monkeypatch.delenv("SMB_JOIN_LAYOUT", raising=False)
    got = B.compare_jaccard(B.SketchSet.from_host(h, off))
    monkeypatch.setenv("SMB_JOIN_LAYOUT", "plain")
    want = B.compare_jaccard(B.SketchSet.from_host(h, off))
    assert got.shape == (10_000, 10_000)
    assert np.array_equal(got, want)
