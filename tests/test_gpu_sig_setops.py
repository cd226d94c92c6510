"""batch.combine and the sigsetops commands on the GPU: the emulated cases of tests/sig_setops_cases.py on the device,
the benchmark's 10 000 synthetic sketches against the numpy restatement (flat and with abundances), and one command run
end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sig_setops_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gpu_combine_cases():
    from sourmash_b200 import batch as B
    for tag, rows, ab in C.cases(np.random.default_rng(7)):
        sset = B.SketchSet.from_host(*C.csr(rows, ab))
        for op in ("union", "all", "first_only"):
            got = B.combine(sset, op)
            C.assert_same(got, C.numpy_combine(op, rows, ab), (tag, op, "numpy"))
            C.assert_same(got, C.reference_combine(op, rows, ab), (tag, op, "reference loop"))
    rng = np.random.default_rng(9)
    pool = rng.integers(1, 2**63, size=2000, dtype=np.uint64)
    rows = [np.sort(rng.choice(pool, size=int(rng.integers(1, 300)), replace=False)) for _ in range(12)]
    ab = [rng.integers(1, 50, size=len(r)).astype(np.uint64) for r in rows]
    got = B.combine(B.SketchSet.from_host(*C.csr(rows, ab)), "union", num=300)
    C.assert_same(got, C.reference_combine("union", rows, ab, num=300), "num union")


def test_gpu_combine_synthetic_10000():
    "the benchmark's set: 10 000 sketches, about 5 x 10^7 hashes, all three ops, flat and with abundances"
    from sourmash_b200 import batch as B
    from sourmash_b200.synth import synth_sketches
    h, off = synth_sketches(10_000)
    ab = np.random.default_rng(1).integers(1, 100, size=len(h)).astype(np.uint64)
    rows = [h[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]
    ab_rows = [ab[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]
    for abund, arows in ((None, None), (ab, ab_rows)):
        sset = B.SketchSet.from_host(h, off, abund)
        for op in ("union", "all", "first_only"):
            C.assert_same(B.combine(sset, op), C.numpy_combine(op, rows, arows), op)


def test_gpu_merge_command(tmp_path):
    "python -m sourmash_b200.sigsetops merge on 200 sketches in two .sig files: the union, abundances summed"
    from sourmash_b200.signature import SourmashSignature, load_signatures_from_json, save_signatures_to_json
    from sourmash_b200.synth import synth_sketches
    h, off = synth_sketches(200, seed=3)
    rng = np.random.default_rng(2)
    rows = [h[int(off[i]):int(off[i + 1])] for i in range(200)]
    ab = [rng.integers(1, 9, size=len(r)).astype(np.uint64) for r in rows]
    sigs = [SourmashSignature(C.minhash_of(r, a, scaled=1000), name="s%d" % i) for i, (r, a) in enumerate(zip(rows, ab))]
    paths = [str(tmp_path / "a.sig"), str(tmp_path / "b.sig")]
    for path, part in zip(paths, (sigs[:70], sigs[70:])):
        with open(path, "wb") as fh:
            save_signatures_to_json(part, fh)
    out = str(tmp_path / "m.sig")
    r = subprocess.run([sys.executable, "-m", "sourmash_b200.sigsetops", "merge"] + paths + ["-o", out, "--name", "m"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "loaded and merged 200 signatures" in r.stderr
    (merged,) = load_signatures_from_json(out)
    want_h, want_a = C.numpy_combine("union", rows, ab)
    assert merged.name == "m"
    assert merged.minhash.hashes == dict(zip(want_h.tolist(), want_a.tolist()))
