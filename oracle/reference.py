"""The reference's Python package, C header, test modules and test data as the CPU tests use them.  TEST INFRASTRUCTURE ONLY.

The reference (sourmash-bio/sourmash) is Rust underneath; its Python layer, its header and its own test suite run over this
project's library instead (tests/test_reference_*.py, tests/test_plugin_through_reference_cli.py, ...).  build() copies
those parts of the checkout recorded in BASELINE.json ("reference_path"; SMB_REFERENCE overrides it) into oracle/_ref/sourmash
(git-ignored), so that the tests read a build product inside the tree, not a path outside it.  Without a checkout nothing
is copied and a copy made earlier is kept; the tests that need it skip when there is none.
"""
import json
import os
import shutil
import stat

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
COPY = os.path.join(_HERE, "_ref", "sourmash")
PARTS = ("src/sourmash", "include", "tests", "data")


def checkout():
    "the reference checkout build() copies from (it may not exist on this machine)"
    if os.environ.get("SMB_REFERENCE"):
        return os.environ["SMB_REFERENCE"]
    with open(os.path.join(ROOT, "BASELINE.json")) as fh:
        return json.load(fh)["reference_path"]


def root():
    "the reference tree the tests use: SMB_REFERENCE if set, else the copy build() made (may be missing)"
    return os.environ.get("SMB_REFERENCE") or COPY


def build():
    """Copy PARTS of the checkout into oracle/_ref/sourmash (replacing an older copy).  Returns the copy, or None when
    there is no readable checkout."""
    src = checkout()
    if not all(os.path.isdir(os.path.join(src, p)) and os.access(os.path.join(src, p), os.R_OK | os.X_OK) for p in PARTS):
        return None
    tmp = COPY + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    for part in PARTS:
        shutil.copytree(os.path.join(src, part), os.path.join(tmp, part), symlinks=True,
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc", ".pytest_cache"))
    # the checkout may be read-only; its tests copy test data to temporary directories and write there, and a later
    # build() must be able to replace this copy: the owner may write every file and directory of it
    for top, dirs, files in os.walk(tmp):
        for name in dirs + files:
            path = os.path.join(top, name)
            if not os.path.islink(path):
                os.chmod(path, os.stat(path).st_mode | stat.S_IWUSR)
    os.chmod(tmp, os.stat(tmp).st_mode | stat.S_IWUSR)
    shutil.rmtree(COPY, ignore_errors=True)
    os.replace(tmp, COPY)
    return COPY
