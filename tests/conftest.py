import gzip
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _ensure_built():
    """Compile libsourmash_b200.so if it is missing or stale (needs nvcc; without it a library that is
    already there is used).  Loaded by path so the package is not imported first."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_smb_build", os.path.join(ROOT, "sourmash_b200", "_build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    try:
        if mod.needs_build():
            mod.build()
    except Exception as exc:                      # no nvcc on this machine: use what is there
        if not os.path.exists(mod.LIB):
            raise RuntimeError(f"cannot build {mod.LIB}: {exc}")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    _ensure_built()


_ECOLI = []


def ecoli_k12_path():
    """The E. coli K-12 genome as one .fna.gz: stored as two gzip members (files under 1 MB each), whose concatenation is
    a valid gzip file; written once per session into a temporary directory that is removed when the session ends."""
    if not _ECOLI:
        import atexit
        import shutil
        import tempfile
        tmp = tempfile.mkdtemp(prefix="smb_golden_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "ecoli_k12.fna.gz")
        with open(path, "wb") as out:
            for part in ("ecoli_k12.part1.fna.gz", "ecoli_k12.part2.fna.gz"):
                with open(os.path.join(GOLDEN, part), "rb") as fh:
                    out.write(fh.read())
        _ECOLI.append(path)
    return _ECOLI[0]


def read_fasta(path):
    """Minimal FASTA reader -> list of (name, bytes)."""
    opener = gzip.open if path.endswith(".gz") else open
    recs, name, chunks = [], None, []
    with opener(path, "rb") as fh:
        for line in fh:
            line = line.rstrip(b"\r\n")
            if line.startswith(b">"):
                if name is not None:
                    recs.append((name, b"".join(chunks)))
                name, chunks = line[1:].decode(), []
            elif line:
                chunks.append(line)
    if name is not None:
        recs.append((name, b"".join(chunks)))
    return recs


@pytest.fixture(scope="session")
def golden():
    arrays = {}
    for part in ("golden_arrays_1.npz", "golden_arrays_2.npz"):     # two archives: each file stays under 1 MB
        with np.load(os.path.join(GOLDEN, part)) as z:
            arrays.update({k: z[k] for k in z.files})
    with open(os.path.join(GOLDEN, "golden_meta.json")) as fh:
        meta = json.load(fh)
    return {"arrays": arrays, "meta": meta}


@pytest.fixture(scope="session")
def ecoli_seq():
    recs = read_fasta(ecoli_k12_path())
    assert len(recs) == 1
    return recs[0][1]


@pytest.fixture(scope="session")
def s10_records():
    return read_fasta(os.path.join(GOLDEN, "genome-s10.fa.gz"))


@pytest.fixture(scope="session")
def golden_dir():
    import pathlib
    return pathlib.Path(GOLDEN)
