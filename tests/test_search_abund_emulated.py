"""batch.search_angular and search_abund without a GPU: tests/host_emul/search_abund_checks.py drives the EMULATED build
of the library (tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the device) in a
subprocess and compares every result with a numpy restatement and with the reference's per-subject loop written with
this package's MinHash (tests/search_abund_cases.py)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "search_abund_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "search_abund checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_search_angular_edge_cases():
    "empty set / query / rows, rows and query cut by max_hash, UINT64_MAX, the clamp, wrapping terms, both layouts"
    assert "ok  " in _run("search_angular_edge_cases")


@pytest.mark.timeout(1800)
def test_emulated_search_angular_errors():
    "a set without abundances, a query that is not sorted and unique; an empty set gives nothing"
    assert "ok  " in _run("search_angular_errors")


@pytest.mark.timeout(1800)
def test_emulated_search_abund_follows_the_reference():
    "LinearIndex and ZipFileLinearIndex against the per-subject loop: query and subject cuts, num groups, ties"
    assert "ok  " in _run("search_abund_follows_the_reference")


@pytest.mark.timeout(1800)
def test_emulated_search_abund_subjects_that_are_not_signatures():
    "a LinearIndex of objects that only carry .minhash, mixed with signatures"
    assert "ok  " in _run("search_abund_subjects_that_are_not_signatures")


@pytest.mark.timeout(1800)
def test_emulated_search_abund_errors_at_the_same_subject():
    assert "ok  " in _run("search_abund_errors_at_the_same_subject")


@pytest.mark.timeout(1800)
def test_emulated_search_abund_objects_for_matches_only():
    assert "ok  " in _run("search_abund_objects_for_matches_only")


@pytest.mark.timeout(1800)
def test_emulated_search_angular_launches_do_not_grow_with_rows():
    assert "ok  " in _run("search_angular_launches_do_not_grow_with_rows")
