"""The stripe count kernel (csrc/join_stripe.cuh) on the device, on the row sets of tests/stripe_group_edge_cases.py
(the same sets run through the SIMT emulator in tests/test_stripe_group_edges_simt.py): the host, resident and
block-of-rows entry points with both tag widths and both count modes, and key-range shards whose partial counters add
up to the oracle's.  Bit for bit."""
import numpy as np
import pytest

import oracle as orc
from tests.stripe_group_edge_cases import LAST, edge_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def B():
    from sourmash_b200 import batch
    return batch


@pytest.mark.parametrize("layout,tags", [(None, None), (None, "u32"), ("stripe_full", None), ("stripe_full", "u32")])
@pytest.mark.parametrize("last", LAST)
def test_stripe_group_edges_match_oracle(B, monkeypatch, last, layout, tags):
    import torch
    monkeypatch.setenv("SMB_COMPARE_ALGO", "join")
    if layout:
        monkeypatch.setenv("SMB_JOIN_LAYOUT", layout)
    if tags:
        monkeypatch.setenv("SMB_STRIPE_TAGS", tags)
    h, off = orc.to_csr(edge_rows(last, seed=last))
    n = len(off) - 1
    want = orc.compare_all_pairs(h, off, nthreads=8)
    sset = B.SketchSet.from_host(h, off)
    assert np.array_equal(B.compare_jaccard(sset), want)
    d_out = torch.full((n, n), -1.0, dtype=torch.float64, device="cuda")
    B.compare_jaccard_device(sset, d_out.data_ptr())
    assert np.array_equal(d_out.cpu().numpy(), want)
    lo, hi = 50, 90
    d_rows = torch.full((hi - lo, n), -1.0, dtype=torch.float64, device="cuda")
    B.compare_jaccard_rows_device(sset, lo, hi, d_rows.data_ptr())
    assert np.array_equal(d_rows.cpu().numpy(), want[lo:hi])


@pytest.mark.parametrize("last", LAST)
def test_stripe_group_edges_key_range_shards(B, monkeypatch, last):
    "every shard's stream ends with a group: its reads run into the head flags behind that shard's stream"
    import torch
    monkeypatch.setenv("SMB_COMPARE_ALGO", "join")
    h, off = orc.to_csr(edge_rows(last, seed=last))
    n = len(off) - 1
    want = orc.pairwise_common(h, off, nthreads=8)
    sset = B.SketchSet.from_host(h, off)
    off_diag = ~np.eye(n, dtype=bool)
    for shards in (1, 3, 8):
        total = torch.zeros((n, n), dtype=torch.int32, device="cuda")
        for r in range(shards):
            part = torch.full((n, n), -1, dtype=torch.int32, device="cuda")
            B.compare_counts_shard_device(sset, r, shards, part.data_ptr(), bits=32)
            total += part
        got = total.cpu().numpy().view(np.uint32)
        assert np.array_equal(got[off_diag], want[off_diag].astype(np.uint32)), (last, shards)
