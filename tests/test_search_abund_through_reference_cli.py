"""`sourmash scripts b200search` next to the reference's `sourmash search` with abundance queries, through the
reference's command line: the angular-similarity route (Index.search_abund) of both, database by database, with md5
de-duplication across databases.

The setting of tests/test_sig_setops_through_reference_cli.py: the reference's package runs over the emulated library
and finds this package's commands in a dist-info written next to it; both commands run on the same inputs, and the CSV
files they write, their exit codes and the ERROR lines of their reports must be equal.  The rest of the reports is not
compared: b200search prints its own report (no loading progress, its own results table), the same for abundance and
flat queries.

Inputs: the track_abund 47/63 sketches as .sig.gz files, as a .zip collection and as a directory; several databases
sharing sketches; abundance sketches at scaled 10 and 100 made with `b200sketch -p ...,abund` (the query's scaled, a
coarser and a finer one in the same search).  A directory database is an expected failure: the reference loads it as a
MultiIndex whose location column holds each file's path, `load_file_as_index` as one LinearIndex whose location is the
directory, so the CSVs differ in that column.  Options --threshold 0, --best-only and -n; the error paths of a flat
subject in a database and of --containment without --ignore-abundance.  The reference's side is stored in
tests/golden/search_abund_cli_reference.json.gz (SHA-256 of every file it wrote, its ERROR lines and its exit
code); without the reference copy that build() makes, `python -m sourmash_b200.plugin b200search` is checked
against the stored side, with it the live reference must do exactly what is stored (SMB_PLUGIN_CLI_RECORD=1 rewrites
the stored side)."""
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys
import zipfile

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_plugin_through_reference_cli as base  # noqa: E402
from test_sig_setops_through_reference_cli import report_lines  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "search_abund_cli_reference.json.gz")
STDERR, RC = "<report>", "<rc>"


def error_lines(text):
    "the ERROR lines of a report (stdout and stderr together); the rest of b200search's report is its own"
    return [line for line in report_lines(text) if line.startswith("ERROR")]


def _digest(b):
    return hashlib.sha256(b).hexdigest()


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refsearchabund"))
    site = os.path.join(tmp, "site")
    data = base.DATA
    stored, recorded = {}, {}
    if LIVE:
        over_abi._stub_package(tmp, emul_lib.build())
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + "".join("%s = sourmash_b200.plugin:Command_%s\n" % (c.lower(), c)
                                                        for c in base.COMMANDS))
        if os.path.exists(STORED) and not os.environ.get("SMB_PLUGIN_CLI_RECORD"):
            with gzip.open(STORED, "rt") as fh:
                stored = json.load(fh)
    else:
        emul_lib.build()
        os.makedirs(site)
        data = os.path.join(tmp, "test-data")
        base._stored_inputs(data)
        with gzip.open(STORED, "rt") as fh:
            recorded = json.load(fh)
    with open(os.path.join(site, "sitecustomize.py"), "w") as fh:
        fh.write("import sys\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport emulated_boot\nemulated_boot.install()\n"
                 % (os.path.join(HERE, "host_emul"), ROOT))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, os.path.join(tmp, "reftests")]), PYTHONDONTWRITEBYTECODE="1")
    work = os.path.join(tmp, "work")
    os.makedirs(os.path.join(work, "abdir", "sub"))
    # the track_abund sketches as .sig.gz, in a directory (one below a subdirectory) and as a .zip collection
    for name in ("47", "63"):
        with open(os.path.join(data, "track_abund", name + ".fa.sig"), "rb") as src:
            raw = src.read()
        with gzip.GzipFile(os.path.join(work, "ab%s.sig.gz" % name), "wb", mtime=0) as fh:
            fh.write(raw)
        shutil.copy(os.path.join(work, "ab%s.sig.gz" % name),
                    os.path.join(work, "abdir", "sub" if name == "63" else "", "ab%s.sig.gz" % name))
    with zipfile.ZipFile(os.path.join(work, "track_abund.zip"), "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name in ("63", "47"):
            with open(os.path.join(data, "track_abund", name + ".fa.sig"), "rb") as src:
                z.writestr(zipfile.ZipInfo("signatures/%s.sig" % name, (2020, 1, 1, 0, 0, 0)), src.read())
    shutil.copy(os.path.join(data, "47.fa.sig"), os.path.join(work, "flat47.sig"))

    def placeholders(b):
        return b.replace(work.encode(), b"@WORK@").replace(data.encode(), b"@DATA@")

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=0):
        "the reference's command (stored outside LIVE) or this package's: (rc, ERROR lines, {file: sha256})"
        args = [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            out = recorded[key(args)]
            return out[RC], json.loads(out[STDERR].replace("@WORK@", work).replace("@DATA@", data)), \
                {rel: v for rel, v in out.items() if rel not in (STDERR, RC)}
        if args[0] == "scripts" and not LIVE:
            cmd = [sys.executable, "-m", "sourmash_b200.plugin"] + args[1:]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + args
        before = base._files(work)
        r = subprocess.run(cmd, capture_output=True, env=env, cwd=work, timeout=900)
        err = r.stderr.decode("utf-8", "replace")
        assert r.returncode == rc, " ".join(args) + "\n" + err[-3000:]
        after = base._files(work)
        files = {}
        for rel in sorted(after):
            if before.get(rel) != after[rel]:
                with open(os.path.join(work, rel), "rb") as fh:
                    files[rel] = _digest(placeholders(fh.read()))
        lines = error_lines(r.stdout.decode("utf-8", "replace") + "\n" + err)
        if args[0] != "scripts":
            out = dict(files)
            out[STDERR] = placeholders(json.dumps(lines).encode()).decode()
            out[RC] = r.returncode
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference did other than stored (%s)" % key(args)
        return r.returncode, lines, files

    def both(tag, *args, rc=0):
        "`search` and `scripts b200search` with the same arguments; @OUT@ names get the side's tag"
        def side(name):
            return [a.replace("@OUT@", "%s_%s" % (tag, name)) for a in map(str, args)]
        want = run("search", *side("ref"), rc=rc)
        got = run("scripts", "b200search", *side("b200"), rc=rc)
        assert got[0] == want[0], (tag, got[0], want[0])
        assert got[1] == want[1], (tag, "\n".join(got[1]), "\n".join(want[1]))
        rename = {rel.replace(tag + "_ref", tag + "_b200"): v for rel, v in want[2].items()}
        assert got[2] == rename, (tag, got[2], rename)
        return want

    run.work, run.data, run.both = work, data, both
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


def test_track_abund_databases(sk):
    ".sig.gz files, a .zip, several databases sharing sketches; --threshold 0, --best-only, -n"
    sk.both("files", "ab47.sig.gz", "ab47.sig.gz", "ab63.sig.gz", "--threshold", "0", "-o", "@OUT@.csv")
    sk.both("zip", "ab63.sig.gz", "track_abund.zip", "--threshold", "0", "-o", "@OUT@.csv")
    sk.both("shared", "ab47.sig.gz", "ab63.sig.gz", "track_abund.zip", "ab47.sig.gz", "--threshold", "0",
            "-o", "@OUT@.csv")
    sk.both("best", "ab47.sig.gz", "track_abund.zip", "ab63.sig.gz", "--threshold", "0", "--best-only", "-o", "@OUT@.csv")
    sk.both("n1", "ab47.sig.gz", "track_abund.zip", "--threshold", "0", "-n", "1", "-o", "@OUT@.csv")
    sk.both("n0", "ab47.sig.gz", "track_abund.zip", "--threshold", "0", "-n", "0", "-o", "@OUT@.csv")
    sk.both("default_threshold", "ab63.sig.gz", "track_abund.zip", "-o", "@OUT@.csv")


def test_two_scaled_values(sk):
    "abundance sketches at scaled 10 and 100 in one search: the query cut to the coarser group, the finer group cut"
    d = sk.data
    for scaled in ("10", "100"):
        for i, fa in enumerate(("short.fa", "short2.fa", "short3.fa")):
            sk("scripts", "b200sketch", os.path.join(d, fa), "-p", "k=31,scaled=%s,abund" % scaled,
               "-o", "s%s_%d.sig" % (scaled, i))
    sk.both("q10", "s10_0.sig", "s10_0.sig", "s100_1.sig", "s10_1.sig", "s100_2.sig", "s10_2.sig", "s100_0.sig",
            "--threshold", "0", "-o", "@OUT@.csv")
    sk.both("q100", "s100_1.sig", "s10_0.sig", "s10_1.sig", "s100_2.sig", "--threshold", "0.01", "-n", "0",
            "-o", "@OUT@.csv")


def test_error_paths(sk):
    "a flat subject in a database and --containment without --ignore-abundance: exit code and report"
    sk.both("flat_subject", "ab47.sig.gz", "ab63.sig.gz", "flat47.sig", "--threshold", "0", "-o", "@OUT@.csv", rc=255)
    sk.both("containment", "ab47.sig.gz", "ab63.sig.gz", "--containment", "-o", "@OUT@.csv", rc=255)


@pytest.mark.xfail(strict=True, reason="a directory's location column: each file's path in the reference (MultiIndex with "
                   "prepend_location), the directory in load_file_as_index's LinearIndex")
def test_directory_database(sk):
    sk.both("dir", "ab47.sig.gz", "abdir", "--threshold", "0", "-o", "@OUT@.csv")
