"""batch.search_angular and search_abund on the GPU: every emulated check of tests/host_emul/search_abund_checks.py on
the device, and the benchmark's workload 1 at full size (50 000 subjects of ~5 000 hashes) against the numpy
restatement, bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import search_abund_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_gpu_search_abund_checks():
    "the cases, errors, objects-for-matches and launch-count checks, with the real library"
    r = subprocess.run([sys.executable, os.path.join(HERE, "host_emul", "search_abund_checks.py"), "--device"],
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "search_abund checks passed" in r.stdout


def test_gpu_search_angular_workload_1():
    from sourmash_b200 import batch as B
    q, qa, h, off, ab = C.bench_workload(1)
    got = B.search_angular(q, qa, B.SketchSet.from_host(h, off, ab), C.U64_MAX)
    want = C.numpy_angular(q, qa, h, off, ab, C.U64_MAX)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert not len(bad), (bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
    assert (got > 0).sum() > len(got) // 2
