"""batch.multigather and gather.gather_many without a GPU: tests/host_emul/multigather_checks.py drives the EMULATED
build of the library (tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the
device) in a subprocess and compares every query's picks, intersection sizes and consumed rounds with a brute force of
the reference's gather loop, and gather_many with gather_databases."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "multigather_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "multigather checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_multigather_rounds():
    "ties, no candidates, full consumption, per-query thresholds / min_counts, max_rounds, grouping, both fallbacks"
    out = _run("multigather_vs_bruteforce", "multigather_grouping_and_fallbacks", "multigather_range_major_prefetch")
    assert out.count("ok  ") == 3


@pytest.mark.timeout(1800)
def test_emulated_multigather_launches_do_not_grow_with_queries():
    "32 queries issue no more round launches than the slowest of them alone, plus one batch of rounds"
    assert "ok  " in _run("multigather_launches_follow_rounds")


@pytest.mark.timeout(1800)
def test_emulated_gather_many_equals_gather_databases():
    "flat and abundance queries, threshold_bp 0 and > 0, an empty query, queries at two scaled values"
    assert "ok  " in _run("gather_many_equals_gather_databases")
