"""The stripe count kernel (csrc/join_stripe.cuh) on the CPU through the SIMT emulator (tests/host_emul/simt_emul.cu),
on the row sets of tests/stripe_group_edge_cases.py: groups of 2 to 129 rows around the kernel's read sizes, groups and
elements at many stream alignments, a group at the end of the stream; both tag widths, both count modes, full and
shortened sort keys.  Compared with the oracle bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as orc
from tests.stripe_group_edge_cases import LAST, edge_rows

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def stripe():
    exe = os.path.join(tempfile.mkdtemp(prefix="smb_stripe_edges_"), "simt_emul")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-x", "c++",
                           os.path.join(HERE, "host_emul", "simt_emul.cu"), "-o", exe])

    def run(rows, *args):
        hashes, offsets = orc.to_csr(rows)
        with tempfile.TemporaryDirectory() as td:
            fh, fo, fc = (os.path.join(td, x) for x in ("h", "o", "c"))
            hashes.tofile(fh)
            offsets.tofile(fo)
            subprocess.check_call([exe, "stripe"] + [str(a) for a in args] + [fh, fo, fc])
            return np.fromfile(fc, dtype=np.float64).reshape(len(rows), len(rows))
    return run


@pytest.mark.parametrize("last", LAST)
def test_simt_stripe_group_edges_match_oracle(stripe, last):
    rows = edge_rows(last, seed=last)
    want = orc.compare_all_pairs(*orc.to_csr(rows), nthreads=2)
    # (rows per CTA, upper only, threads, tag bits, sort-key bits)
    for cfg in ((5, 0, 64, 16, 32), (3, 1, 96, 32, 32), (32, 0, 32, 16, 8), (7, 1, 128, 16, 3), (4, 1, 64, 32, 8)):
        assert np.array_equal(stripe(rows, *cfg), want), (last, cfg)
