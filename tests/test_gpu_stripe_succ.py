"""GPU parity of the stripe join's count kernel reading the successor bits (csrc/join_stripe.cuh: StripeArgs::succ, built
with the positions through shared-memory sub-windows) at the benchmark's shape: the 10 000 x 10 000 matrix of
synth_sketches(10 000) -- 5e7 elements, twelve windows of pos[] and 3 000 sub-windows -- and of the same size with a pool
per row (n_families = 10 000), compared bit for bit with the global-reduction join (SMB_JOIN_LAYOUT=plain), which
builds no stream.  Small sets, single windows and key-range shards are covered on the CPU by
tests/test_stripe_succ_bits_simt.py."""
import numpy as np
import pytest

from sourmash_b200.synth import synth_sketches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_families", [100, 10_000])
def test_stripe_succ_matrix_matches_plain_join(monkeypatch, n_families):
    from sourmash_b200 import batch as B
    h, off = synth_sketches(10_000, n_families=n_families)
    monkeypatch.setenv("SMB_COMPARE_ALGO", "join")
    monkeypatch.delenv("SMB_JOIN_LAYOUT", raising=False)
    got = B.compare_jaccard(B.SketchSet.from_host(h, off))
    monkeypatch.setenv("SMB_JOIN_LAYOUT", "plain")
    want = B.compare_jaccard(B.SketchSet.from_host(h, off))
    assert got.shape == (10_000, 10_000)
    assert np.array_equal(got, want)
