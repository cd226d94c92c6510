"""kmers.match_records without a GPU: tests/host_emul/sig_kmers_checks.py drives the EMULATED build of the library
(tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the device) in a subprocess and
compares every match, the per-record flags and the found hashes with the reference's per-record loop written with this
package's MinHash (tests/sig_kmers_cases.py)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "sig_kmers_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "sig kmers checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_match_equals_per_record_loop():
    "k = 21/31/51/17, scaled = 2 and 1, num (with a record whose hits fail the record test), protein / dayhoff / hp"
    assert "ok  " in _run("match_vs_per_record_loop")


@pytest.mark.timeout(1800)
def test_emulated_match_large_query_and_staging_overflow():
    "a query above the shared-memory table (global directory) and every window a match"
    assert "ok  " in _run("match_large_query_and_overflow")


@pytest.mark.timeout(1800)
def test_emulated_match_launches_and_errors():
    "launches do not depend on the number of records (scaled and num); protein input into a DNA sketch; an empty query"
    out = _run("match_launches_do_not_grow_with_records", "match_num_launches_do_not_grow_with_records",
               "match_input_errors")
    assert out.count("ok  ") == 3


@pytest.mark.timeout(1800)
def test_emulated_match_buffer_rerun_and_skipped_records():
    "a match buffer overflow rerun at the exact size; records with invalid DNA left out of found (scaled and num)"
    assert "ok  " in _run("match_overflow_rerun_and_skipped_records")


@pytest.mark.timeout(1800)
def test_emulated_command_writes_what_the_reference_loop_writes():
    "b200sigkmers --save-kmers / --save-sequences without a moltype flag: DNA scaled and num, translate, protein"
    assert "ok  " in _run("command_writes_what_the_loop_writes")
