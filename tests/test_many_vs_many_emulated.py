"""batch.many_vs_many, multigather's batched first pass and LinearIndex.search_many / prefetch_many without a GPU:
tests/host_emul/many_vs_many_checks.py drives the EMULATED build of the library (tests/host_emul/emul_lib.py: the
product's kernels and host glue, the SIMT emulator as the device) in a subprocess and compares the counts with a brute
force and with the one-query calls."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "many_vs_many_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "many_vs_many checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_many_vs_many_counts():
    """shared / identical / nested / empty queries, keys 0 and 2^64 - 1, empty rows, near-copies (queue overflow), the
    device form; forced one-query and many-query groups, SMB_SEARCH_LAYOUT=global, an indexed set"""
    out = _run("many_vs_many_equals_stacked_one_vs_many", "many_vs_many_paths_and_grouping")
    assert out.count("ok  ") == 2


@pytest.mark.timeout(1800)
def test_emulated_many_vs_many_launches_do_not_grow_with_queries():
    assert "ok  " in _run("many_vs_many_launches_do_not_grow_with_queries")


@pytest.mark.timeout(1800)
def test_emulated_many_vs_many_rejects_bad_input():
    "offsets that do not start at 0 or decrease, unsorted queries (host and device forms)"
    assert "ok  " in _run("many_vs_many_rejects_bad_input")


@pytest.mark.timeout(1800)
def test_emulated_multigather_with_batched_first_pass():
    "batch.multigather still equals the brute force of the reference loop, in one group and in several"
    assert "ok  " in _run("multigather_first_pass_is_batched")


@pytest.mark.timeout(1800)
def test_emulated_search_many_prefetch_many_equal_per_query_calls():
    """finer, equal and coarser query scaled; Jaccard, containment, max-containment, best_only; abundance and
    incompatible-ksize queries, num sketches, an empty index; LinearIndex and ZipFileLinearIndex"""
    assert "ok  " in _run("search_many_and_prefetch_many_equal_per_query_calls")
