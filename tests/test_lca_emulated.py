"""batch.lca_table / batch.lca_counts without a GPU: tests/host_emul/lca_checks.py drives the EMULATED build of the
library (tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the device) in a
subprocess and compares every result with the reference's per-hash loop restated in tests/lca_cases.py."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "lca_checks.py")
NAMES = ["lca_fixtures", "lca_random_tries", "lca_same_hash_two_databases", "lca_empty_inputs", "lca_cut_at_max_hash",
         "lca_argument_errors", "lca_database_loading"]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", NAMES)
def test_emulated_lca(name):
    r = subprocess.run([sys.executable, SCRIPT, name], capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ok  " + name in r.stdout and "lca checks passed" in r.stdout
