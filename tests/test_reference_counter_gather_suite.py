"""The reference's CounterGather conformance suite -- sourmash/tests/test_index_protocol.py:712-1312, the 22
`test_counter_*` functions, read from the reference at test time and run UNMODIFIED -- against this package's
CounterGather / MinHash / SourmashSignature.

The functions run in a subprocess whose library is the emulated
build (tests/host_emul/emul_lib.py: the product's capi.cu and kernels, the device played by the CPU), like
tests/test_reference_python_over_abi.py.  The GPU counterparts with their own data are tests/test_gpu_counter_gather_port.py.
What is supplied here: the names the reference module imports at its top (`sourmash.MinHash`, `sourmash.load_one_signature`,
`SourmashSignature`, `utils.get_test_data`, `glob`) bound to this package's classes / the reference's test-data directory,
and the `counter_gather_constructor` fixture bound to this package's CounterGather."""
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import reference as _reference  # noqa: E402

REF_TESTS = os.path.join(_reference.root(), "tests", "test_index_protocol.py")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.skipif(not os.path.exists(REF_TESTS), reason="needs the reference copy that build() makes from its checkout (oracle/reference.py)")

HEADER = '''
import os, sys
sys.path.insert(0, {host_emul!r})
import emulated_boot
emulated_boot.install()                      # sourmash_b200._lowlevel -> the emulated build of libsourmash_b200
sys.path.insert(0, {root!r})
import glob, types
import pytest
import sourmash_b200
from sourmash_b200 import SourmashSignature
from sourmash_b200.index import CounterGather
from sourmash_b200.signature import load_one_signature_from_json
sourmash = types.SimpleNamespace(MinHash=sourmash_b200.MinHash, load_one_signature=load_one_signature_from_json)
utils = types.SimpleNamespace(get_test_data=lambda name: os.path.join({test_data!r}, name))   # sourmash_tst_utils.get_test_data


@pytest.fixture
def counter_gather_constructor():
    return CounterGather

'''


@pytest.mark.timeout(1200)
def test_reference_counter_gather_functions_pass_unmodified(tmp_path):
    with open(REF_TESTS) as fh:
        lines = fh.read().splitlines(keepends=True)
    start = next(i for i, line in enumerate(lines) if line.startswith("def test_counter_get_signatures"))
    body = "".join(lines[start:])
    n_tests = body.count("\ndef test_counter_") + 1
    assert n_tests == 22
    path = tmp_path / "test_ref_counter_gather.py"
    path.write_text(HEADER.format(host_emul=os.path.join(HERE, "host_emul"), root=ROOT,
                                  test_data=os.path.join(os.path.dirname(REF_TESTS), "test-data")) + body)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "--noconftest", "-p", "no:cacheprovider", "--no-header",
                        "--rootdir", str(tmp_path), str(path)], capture_output=True, text=True, cwd=str(tmp_path), timeout=1100)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ""
    assert r.returncode == 0 and ("%d passed" % n_tests) in tail, r.stdout[-6000:] + r.stderr[-2000:]
