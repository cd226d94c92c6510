"""batch.lca_index without a GPU: tests/host_emul/lca_index_checks.py drives the EMULATED build of the library
(tests/host_emul/emul_lib.py: the product's kernels and host glue, the SIMT emulator as the device) in a subprocess and
compares the arrays and the chunked text with the reference's insert loop restated in tests/lca_index_cases.py."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "lca_index_checks.py")
NAMES = ["lca_index_small", "lca_index_random", "lca_index_ranges", "lca_index_empty", "lca_index_budget",
         "lca_index_capacity", "lca_index_argument_errors", "lca_index_numpy_oracle"]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", NAMES)
def test_emulated_lca_index(name):
    r = subprocess.run([sys.executable, SCRIPT, name], capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ok  " + name in r.stdout and "lca index checks passed" in r.stdout
