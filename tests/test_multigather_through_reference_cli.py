"""`sourmash scripts b200multigather` next to the reference's `sourmash multigather`, through the reference's command line.

The setting of tests/test_plugin_through_reference_cli.py (whose helpers this module uses): the reference's package runs
over the emulated library and finds this package's six plugin commands in a dist-info written next to it; both
commands run on the same inputs and every file they write -- per query the gather CSV, the matches and the unassigned
hashes -- must be byte-identical.  What the reference writes is stored in
tests/golden/multigather_cli_reference.json.gz; without the reference copy that build() makes the plugin command
(`python -m sourmash_b200.multigather`) is checked against the stored files, with it the live reference must write
exactly the stored files (SMB_PLUGIN_CLI_RECORD=1 rewrites them)."""
import base64
import glob
import gzip
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_plugin_through_reference_cli as base  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "multigather_cli_reference.json.gz")
ENTRY_POINTS = [(c.lower(), "sourmash_b200.plugin:Command_%s" % c) for c in base.COMMANDS] + \
               [("b200multigather", "sourmash_b200.multigather:Command_B200Multigather")]


@pytest.fixture(scope="module")
def mg(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refmg"))
    site = os.path.join(tmp, "site")
    data = base.DATA
    stored = {}
    if LIVE:
        over_abi._stub_package(tmp, emul_lib.build())
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(ROOT, "pyproject.toml")) as fh:
            declared = [line.split("=")[0].strip() for line in fh if "sourmash_b200." in line and ":Command_" in line]
        assert declared == [name for name, _ in ENTRY_POINTS]
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + "".join("%s = %s\n" % e for e in ENTRY_POINTS))
        recorded = {}
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
    os.makedirs(work)

    def placeholders(b):
        return b.replace(work.encode(), b"@WORK@").replace(data.encode(), b"@DATA@")

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=(0,)):
        if args[0] == "scripts" and not LIVE:
            cmd = [sys.executable, "-m", "sourmash_b200.multigather"] + [str(a) for a in args[2:]]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:                       # the reference's files, from the stored record
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            for rel, text in recorded[key(args)].items():
                out = os.path.join(work, rel)
                os.makedirs(os.path.dirname(out), exist_ok=True)
                with open(out, "wb") as fh:
                    fh.write(base64.b64decode(text).replace(b"@WORK@", work.encode()).replace(b"@DATA@", data.encode()))
            return None
        before = base._files(work)
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=work, timeout=900)
        assert r.returncode in rc, " ".join(map(str, args)) + "\n" + r.stdout[-2000:] + r.stderr[-3000:]
        if args[0] != "scripts":
            after = base._files(work)
            out = {}
            for rel in sorted(after):
                if before.get(rel) != after[rel]:
                    with open(os.path.join(work, rel), "rb") as fh:
                        out[rel] = base64.b64encode(placeholders(fh.read())).decode()
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference wrote other files than the stored ones (%s)" % key(args)
        return r

    def both(ref_dir, b200_dir, *args, rc=(0,)):
        "the reference's multigather and the plugin command, each writing into its own output directory"
        os.makedirs(os.path.join(work, ref_dir), exist_ok=True)
        os.makedirs(os.path.join(work, b200_dir), exist_ok=True)
        run("multigather", *args, "--output-dir", ref_dir, rc=rc)
        run("scripts", "b200multigather", *args, "--output-dir", b200_dir, rc=rc)
        want = {f: open(os.path.join(work, ref_dir, f), "rb").read() for f in sorted(os.listdir(os.path.join(work, ref_dir)))}
        got = {f: open(os.path.join(work, b200_dir, f), "rb").read() for f in sorted(os.listdir(os.path.join(work, b200_dir)))}
        assert sorted(got) == sorted(want), (sorted(got), sorted(want))
        for f in want:
            assert got[f] == want[f], f
        return want

    run.work, run.data, run.both = work, data, both
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


def _gcf(mg):
    return sorted(glob.glob(os.path.join(mg.data, "gather", "GCF*.sig")))


@pytest.mark.parametrize("threshold_bp", ["0", "50000"])
def test_multigather_writes_the_same_files(mg, threshold_bp):
    "combined.sig and three genomes as queries against the twelve genomes: CSV, matches and unassigned per query"
    sigs = _gcf(mg)
    queries = [os.path.join(mg.data, "gather", "combined.sig")] + sigs[:3]
    tag = "t%s" % threshold_bp
    files = mg.both(tag + "_ref", tag + "_b200", "--query", *queries, "--db", *sigs, "-k", "21", "--threshold-bp", threshold_bp)
    assert sum(f.endswith(".csv") for f in files) == 4
    assert sum(f.endswith(".unassigned.sig") for f in files) == 4
    assert all(files[f] for f in files if f.endswith(".csv"))


def test_multigather_scaled_and_queries_in_one_file(mg):
    "--scaled downsamples every query first; one file with three queries needs -U for distinct output names"
    sigs = _gcf(mg)
    if not os.path.exists(os.path.join(mg.work, "three.sig")):
        mg("sig", "cat", *sigs[3:6], "-o", "three.sig")
    files = mg.both("u_ref", "u_b200", "--query", "three.sig", "--db", *sigs, "-k", "21", "--threshold-bp", "0", "-U")
    assert sum(f.endswith(".csv") for f in files) == 3
    mg.both("sc_ref", "sc_b200", "--query", os.path.join(mg.data, "gather", "combined.sig"), sigs[1], "--db", *sigs,
            "-k", "21", "--threshold-bp", "0", "--scaled", "20000")


def test_multigather_abundance_query_and_a_query_without_match(mg):
    "a query with abundances (weighted columns, re-inflated unassigned hashes) and a query that matches nothing"
    d = mg.data
    files = mg.both("ab_ref", "ab_b200", "--query", os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "2.fa.sig"),
                    "--db", os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig"), "-k", "31", "--threshold-bp", "0")
    assert any(f.endswith(".unassigned.sig") for f in files)
    assert any(f.endswith(".csv") and not files[f] for f in files)          # the query without match: an empty CSV
