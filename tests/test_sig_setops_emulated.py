"""batch.combine and sigsetops without a GPU: tests/host_emul/sig_setops_checks.py drives the EMULATED build of the
library (tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the device) in a
subprocess and compares every result with a numpy restatement and with the reference's loops (a chain of MinHash.merge,
Python sets) written with this package's MinHash (tests/sig_setops_cases.py)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "sig_setops_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "sig set-op checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_combine_edge_cases():
    "empty set, one row, empty rows (row 0 too), a sketch twice, UINT64_MAX and dense small keys, long runs; +abund"
    assert "ok  " in _run("combine_edge_cases")


@pytest.mark.timeout(1800)
def test_emulated_combine_num_union():
    "the bottom num of the union with summed abundances, as a chain of merges into a num sketch keeps"
    assert "ok  " in _run("combine_num_union")


@pytest.mark.timeout(1800)
def test_emulated_combine_launches_do_not_grow_with_rows():
    assert "ok  " in _run("combine_launches_do_not_grow_with_rows")


@pytest.mark.timeout(1800)
def test_emulated_minhash_functions_follow_the_reference():
    "merge / intersect / subtract_minhashes on MinHash and SourmashSignature lists, and the reference's errors"
    assert "ok  " in _run("minhash_functions_follow_the_reference")
