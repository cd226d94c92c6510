"""batch.lca_index and `b200lcaindex` on the GPU: the emulated checks of tests/host_emul/lca_index_checks.py on the
device, a GTDB-sized synthetic build (30 000 genomes, 3*10^7 pairs, hashes shared with a skewed distribution) checked
against the numpy oracle of tests/lca_index_cases.py on the arrays and on sampled key ranges of the text, and the
command end to end on the reference's fixtures, its database then loaded and used for classification."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "host_emul"))
import lca_index_checks  # noqa: E402

from tests import lca_cases  # noqa: E402
from tests import lca_index_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(lca_index_checks.CHECKS))
def test_gpu_lca_index_checks(name):
    lca_index_checks.CHECKS[name]()


def test_gpu_lca_index_gtdb_sized():
    from sourmash_b200 import batch as B
    from sourmash_b200._lowlevel import ffi, lib
    h, off = C.skewed_rows(seed=7, n_rows=30_000, n_pairs=30_000_000)
    x = B.lca_index(B.SketchSet.from_host(h, off))
    got = x.arrays()
    want = C.np_oracle_arrays(h, off)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    hashes, offsets, idx = got
    sizes = np.diff(offsets.astype(np.int64))
    assert sizes.max() > 1000 and (sizes == 1).mean() > 0.5          # skewed: some keys in thousands of rows
    n = len(x)
    size = ffi.new("uintptr_t *")
    rng = np.random.default_rng(0)
    starts = [0, n - 1, int(np.argmax(sizes))] + rng.integers(0, n, size=20).tolist()
    for k in starts:
        nxt = int(lib.smb_lca_index_text(x._ptr, k, 1 << 16, ffi.NULL, size))
        buf = bytearray(int(size[0]))
        size[0] = len(buf)
        lib.smb_lca_index_text(x._ptr, k, 1 << 16, ffi.from_buffer(buf), size)
        assert bytes(buf) == C.text_of_keys(hashes, offsets, idx, k, nxt, n), k
    total = sum(len(c) for c in x.text_chunks(64 << 20))
    parts = [len(c) for c in x.text_chunks(64 << 20)]
    assert len(parts) > 1 and total == sum(parts)


def test_gpu_lca_index_command(tmp_path):
    from sourmash_b200 import lca as L
    work = C.unpack_fixtures(str(tmp_path))
    lca_cases.unpack_fixtures(os.path.join(work, "lca"))
    out = os.path.join(work, "db.lca.json")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.lca", "index", "tara-delmont-SuppTable3.csv", out,
                        "dir1", "dir2", "-C", "3", "--split-identifiers", "-f"], capture_output=True, text=True,
                       cwd=work, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "... loaded 2 signatures." in r.stderr and "identifiers used out of" in r.stderr
    db = L.LcaDatabase.load(out)
    with open(out) as fh:
        d = json.load(fh)
    assert list(d) == ["version", "type", "license", "ksize", "scaled", "moltype", "lid_to_lineage",
                       "hashval_to_idx", "ident_to_name", "ident_to_idx", "idx_to_lid"]
    assert len(d["ident_to_idx"]) == 20 and len(db.hashes) == sum(len(v) for v in d["hashval_to_idx"].values())
    csv_out = os.path.join(work, "cl.csv")
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.lca", "classify", "--db", out, "--query",
                        "dir1/TARA_ANE_MAG_00044.fa.gz.sig", "-o", csv_out], capture_output=True, text=True, cwd=work,
                       env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    with open(csv_out) as fh:
        assert fh.read().splitlines()[1].startswith(("TARA_ANE_MAG_00044,found,", "TARA_ANE_MAG_00044,disagree,"))
