"""The library end to end without a GPU: tests/host_emul/emul_lib.py builds an EMULATED copy of it (the product's
sources, kernel launches redirected to the SIMT emulator of tests/host_emul/simt.h, host stand-ins for the CUDA
runtime and cub) and tests/host_emul/emulated_checks.py drives it through the C ABI and the Python layer against
the oracle -- default paths and, above all, the paths behind switches that have not run on a GPU yet (their host
glue is reached by no other CPU test).  The emulated library lives in the temp directory and is loaded in a
subprocess only; the package itself never sees it."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "host_emul", "emulated_checks.py")


def _run(*names):
    r = subprocess.run([sys.executable, SCRIPT] + list(names), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "emulated checks passed" in r.stdout
    return r.stdout


@pytest.mark.timeout(1800)
def test_emulated_compare_paths():
    out = _run("compare_default_and_join", "compare_stripe_layouts_resident", "compare_host_path_row_chunks",
               "compare_shards_sum_to_full")
    assert out.count("ok  ") == 4


@pytest.mark.timeout(1800)
def test_emulated_search_gather_sketch_paths():
    out = _run("search_layouts_and_index", "gather_default_and_index", "sketch_default_and_fused")
    assert out.count("ok  ") == 3


def test_package_does_not_know_the_emulated_library():
    "the product only ever loads libsourmash_b200.so next to the package (no CPU fallback, DESIGN.md section 2)"
    import sourmash_b200._lowlevel as ll
    assert os.path.basename(ll.LIB_PATH) == "libsourmash_b200.so" and os.path.dirname(ll.LIB_PATH) == os.path.dirname(ll.__file__)
    pkg = os.path.dirname(ll.__file__)
    for base, _dirs, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                with open(os.path.join(base, f)) as fh:
                    text = fh.read()
                assert "emul_lib" not in text and "libsourmash_b200_emul" not in text, f


@pytest.mark.timeout(900)
def test_emulated_sharded_search_and_gather_world2():
    """distributed.ShardedDatabase with the real batch module on two gloo ranks (one of them probing the inverted
    index): all-gathered counts and the gather rounds' exchanges give the single-process result on both ranks."""
    script = os.path.join(HERE, "host_emul", "emulated_sharded.py")
    r = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "passed on 2 ranks" in r.stdout


def test_emulated_smoke_hook():
    "__graft_entry__.smoke() -- the end-to-end GPU smoke run -- against the emulated library"
    code = ("import sys; sys.path.insert(0, %r); import emulated_boot; emulated_boot.install(); sys.path.insert(0, %r); "
            "import __graft_entry__ as g; g.smoke()") % (os.path.join(HERE, "host_emul"), os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "smoke ok" in r.stdout, r.stdout[-1000:] + r.stderr[-2000:]


@pytest.mark.timeout(900)
def test_bench_b200_arm_dry_run():
    """bench.py's GPU arm against the emulated library with tiny workloads and a stand-in for its torch.cuda calls:
    not a measurement, a proof that every workload / switch assembles its JSON line (roofline, dram, issue, e2e,
    launches, clocks) and its --dump-outputs arrays without raising -- a benchmark run must not die on a KeyError."""
    script = os.path.join(HERE, "host_emul", "bench_dryrun.py")
    r = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=800)
    assert r.returncode == 0 and "bench dry run ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
