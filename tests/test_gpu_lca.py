"""batch.lca_table / batch.lca_counts and the lca commands on the GPU: the emulated checks of
tests/host_emul/lca_checks.py on the device, a GTDB-sized synthetic setting (10^5 lineages, 10^7 database pairs,
1 000 queries of about 5 000 hashes) checked against the oracle of tests/lca_cases.py, and one command end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "host_emul"))
import lca_checks  # noqa: E402

from tests import lca_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(lca_checks.CHECKS))
def test_gpu_lca_checks(name):
    lca_checks.CHECKS[name]()


def test_gpu_lca_synthetic_user_scale():
    from sourmash_b200 import batch as B
    from sourmash_b200 import lca as L
    dbs, queries = C.synth_lca(seed=3)
    tax = L.Taxonomy(dbs)
    table = L.build_table(dbs, tax)
    assert 0 < len(table) <= sum(len(db.hashes) for db in dbs)
    off = np.concatenate([[0], np.cumsum([len(q) for q in queries])]).astype(np.uint64)
    sset = B.SketchSet.from_host(np.concatenate(queries), off)
    ranked = L.ranked_counts(table, sset, len(queries), False)
    assert sum(len(r) for r in ranked) > len(queries)
    picked = np.random.default_rng(0).choice(len(queries), size=8, replace=False).tolist()
    for i, want in zip(picked, C.synth_oracle(dbs, [queries[i] for i in picked])):
        assert [(tuple(tax.lineage(n)), c) for n, c in ranked[i]] == want, i


def test_gpu_lca_classify_command(tmp_path):
    d = C.FIXTURES
    out = str(tmp_path / "out.csv")
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.lca", "classify", "--db", os.path.join(d, "both.lca.json.gz"),
                        "--query", os.path.join(d, "TARA_ASE_MAG_00031.sig.gz"), "-o", out],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    with open(out) as fh:
        lines = fh.read().splitlines()
    assert lines[0].startswith("ID,status,superkingdom")
    assert lines[1].startswith("TARA_ASE_MAG_00031,found,Bacteria,Proteobacteria,Gammaproteobacteria")
