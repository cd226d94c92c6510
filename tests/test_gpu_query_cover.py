"""batch.query_covered on the GPU: every check of tests/host_emul/query_cover_checks.py with the real library, and the
configs[4] shape (a 10^7-hash query, rows of ~5 000 hashes, 1 % planted at 20-80 % of the query) cut to 30 000 rows,
against np.isin over the rows that pass 50 kbp."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_gpu_query_cover_checks():
    "edge cases, errors, and b200prefetch's two hash outputs against the reference's per-match loop"
    r = subprocess.run([sys.executable, os.path.join(HERE, "host_emul", "query_cover_checks.py"), "--device"],
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "query_cover checks passed" in r.stdout


def test_gpu_query_cover_configs4_shape():
    from sourmash_b200 import batch as B
    from sourmash_b200.synth import database_block, database_plan, search_query
    n_rows = 30_000
    query = search_query(10_000_000)
    sizes, frac = database_plan(n_rows, 4001, planted_frac=0.01)
    h = database_block(sizes, frac, query, 0, n_rows, 4002)
    off = np.zeros(n_rows + 1, dtype=np.uint64)
    off[1:] = np.cumsum(sizes)
    db = B.SketchSet.from_host(h, off)
    counts = B.one_vs_many(query, db)
    rows = np.nonzero(counts.astype(np.int64) * 1000 >= 50_000)[0]
    assert 100 < len(rows) < 600, len(rows)
    got = B.query_covered(query, db, rows)
    held = np.concatenate([h[int(off[r]):int(off[r + 1])] for r in rows])
    want = np.isin(query, held)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:5]
    assert int(got.sum()) > 0
