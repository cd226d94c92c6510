"""batch.query_covered and prefetch's matched / unmatched hash outputs without a GPU: tests/host_emul/query_cover_checks.py
drives the EMULATED build of the library (tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT
emulator as the device) in a subprocess and compares every result with np.isin over the listed rows and with the
reference's per-match loop."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "query_cover_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "query_cover checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_query_cover_edge_cases():
    "empty rows and row list, a row listed twice, rows outside the key range, one-hash query, UINT64_MAX, odd lengths"
    assert "ok  " in _run("query_cover_edge_cases")


@pytest.mark.timeout(1800)
def test_emulated_query_cover_errors():
    "an out-of-range row index is the library's error; empty inputs launch nothing"
    assert "ok  " in _run("query_cover_errors")


@pytest.mark.timeout(1800)
def test_emulated_prefetch_saves_the_reference_split():
    "b200prefetch --save-matching-hashes / --save-unmatched-hashes against the reference's per-match loop"
    assert "ok  " in _run("prefetch_saves_the_reference_split")
