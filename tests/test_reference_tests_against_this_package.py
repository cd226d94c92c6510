"""The reference's own tests against THIS package's Python layer (sourmash_b200 imported as `sourmash`).

tests/test_reference_python_over_abi.py runs the reference's Python over this library's C ABI; this file is the other
half of the host-side claim (DESIGN.md section 2: minhash.py / signature.py / compare.py / index.py "mirror the reference
modules' names, arguments and error behaviour"): the reference's test modules, unmodified and read in place, import a
package `sourmash` that IS sourmash_b200 -- so test_compare.py checks this package's batched compare_serial* / compare_parallel
/ compare_all_pairs (one device pass instead of the reference's per-pair loops), test_index_protocol.py its LinearIndex and
CounterGather, test_minhash.py / test_signature.py its object model.  The library is the emulated build (no GPU where the
reference checkout is).

Names the reference's modules import for classes this package does not have (storage containers, report dataclasses,
out-of-scope engines) are placeholders; the tests that use them are deselected by name below."""
import os
import subprocess
import sys
import textwrap

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_reference_python_over_abi as over_abi  # noqa: E402  (the stand-ins for absent third-party packages, _counts, _workers)

REF = over_abi.REF
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "sourmash")),
                                reason="needs the reference copy that build() makes from its checkout (oracle/reference.py)")

ALIAS_INIT = textwrap.dedent('''
    """`sourmash` = sourmash_b200 on the emulated library"""
    import importlib, sys, types
    sys.path.insert(0, {host_emul!r}); sys.path.insert(0, {root!r})
    import emulated_boot
    emulated_boot.install()
    import sourmash_b200 as _pkg
    for _name in ("minhash", "signature", "compare", "search", "index", "distance_utils", "exceptions", "manifest", "sbt_storage"):
        _m = importlib.import_module("sourmash_b200." + _name)
        sys.modules["sourmash." + _name] = _m
        globals()[_name] = _m
    globals().update({{k: getattr(_pkg, k) for k in dir(_pkg) if not k.startswith("__")}})

    def _placeholder(modname, *names):
        m = sys.modules.get(modname) or types.ModuleType(modname)
        for n in names:
            if not hasattr(m, n):
                setattr(m, n, type(n, (), {{}}))
        sys.modules[modname] = m
        return m
    _placeholder("sourmash.index", "LazyLinearIndex", "MultiIndex", "StandaloneManifestIndex")      # storage containers
    _placeholder("sourmash.index.sqlite_index", "SqliteIndex")
    _placeholder("sourmash.index.revindex", "RevIndex")
    _placeholder("sourmash.sbt", "SBT", "GraphFactory")
    _placeholder("sourmash.lca")
    _placeholder("sourmash.lca.lca_db", "LCA_Database", "load_single_database")
    _placeholder("sourmash.manifest", "BaseCollectionManifest")
    _placeholder("sourmash.search", "SearchResult", "PrefetchResult", "GatherResult")               # report dataclasses
    _placeholder("sourmash.picklist", "SignaturePicklist", "PickStyle")
    sourmash_args = _placeholder("sourmash.sourmash_args")
    sourmash_args.load_file_as_signatures = _pkg.load_file_as_signatures
    sourmash_args.load_file_as_index = _pkg.load_file_as_index
    ''')

MODULES = ("test_minhash.py", "test_jaccard.py", "test__minhash_hypothesis.py", "test_signature.py", "test_compare.py",
           "test_index_protocol.py", "test_index.py")


def _run(tmp_path, modules, extra=()):
    tmp = str(tmp_path)
    site = os.path.join(tmp, "site")
    os.makedirs(os.path.join(site, "sourmash"))
    with open(os.path.join(site, "sourmash", "__init__.py"), "w") as fh:
        fh.write(ALIAS_INIT.format(host_emul=os.path.join(HERE, "host_emul"), root=ROOT))
    for rel, text in over_abi.STUBS.items():                      # deprecation, screed, matplotlib stand-ins
        path = os.path.join(site, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as fh:
            fh.write(text)
    tests = os.path.join(tmp, "reftests")
    os.makedirs(tests)
    for name in ("conftest.py", "sourmash_tst_utils.py", "test-data") + MODULES:
        os.symlink(os.path.join(REF, "tests", name), os.path.join(tests, name))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, tests]), PYTHONDONTWRITEBYTECODE="1")
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "--rootdir", tests, "--no-header", "-rN"] + \
        over_abi._workers() + list(extra) + [os.path.join(tests, m) for m in modules]
    return subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=tmp, timeout=3000)


def _check(r, at_least):
    counts, tail = over_abi._counts(r.stdout)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert counts["failed"] == 0 and counts["error"] + counts["errors"] == 0 and counts["passed"] >= at_least, tail


@pytest.mark.timeout(1800)
def test_reference_object_model_tests_pass_against_this_package(tmp_path):
    "test_minhash.py (311 cases), test_jaccard.py, test__minhash_hypothesis.py, test_signature.py against sourmash_b200's classes"
    _check(_run(tmp_path, ["test_minhash.py", "test_jaccard.py", "test__minhash_hypothesis.py", "test_signature.py"]), 415)


@pytest.mark.timeout(1800)
def test_reference_compare_tests_pass_against_this_package(tmp_path):
    """test_compare.py: compare_serial, compare_serial_containment / max_containment / avg_containment, compare_parallel,
    compare_all_pairs, and their ANI forms -- against sourmash_b200.compare, which computes each matrix in one batched pass."""
    _check(_run(tmp_path, ["test_compare.py"]), 15)


# not run in the two index modules: everything built on classes this package does not have, by name; picklists; the CLI
NOT_HERE = ("not sbt and not SBT and not lca and not LCA and not sql and not revindex and not RevIndex and not lazy and not Lazy "
            "and not multi and not Multi and not standalone and not simple_index and not command and not picklist "
            "and not fsstorage and not zipfile_does_not_exist")


@pytest.mark.timeout(1800)
def test_reference_index_tests_pass_against_this_package(tmp_path):
    """test_index_protocol.py for this package's LinearIndex and CounterGather (the conformance suite's `build_linear_index`
    and `CounterGather` parametrisations) and test_index.py's LinearIndex / ZipFileLinearIndex / CounterGather tests."""
    r = _run(tmp_path, ["test_index_protocol.py"], ["-k", "build_linear_index or (counter_gather and CounterGather and not CounterGather_)"])
    _check(r, 39)


@pytest.mark.timeout(1800)
def test_reference_index_class_tests_pass_against_this_package(tmp_path):
    _check(_run(tmp_path, ["test_index.py"], ["-k", NOT_HERE]), 46)
