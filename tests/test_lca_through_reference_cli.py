"""`sourmash scripts b200lcaclassify | b200lcasummarize` next to the reference's `sourmash lca classify | lca summarize`,
through the reference's command line.

The setting of tests/test_sig_setops_through_reference_cli.py: the reference's package runs over the emulated library and
finds this package's commands in a dist-info written next to it; both commands run on the same inputs (the reference's
LCA test data, stored compressed under tests/golden/refdata/lca), and the files they write, their stdout, their exit codes and the
lines of their reports must be equal.  Progress lines ("... loading database", "... classifying") are left out: the next
line overwrites them on a terminal.

Cases: one and several --db (.lca.json and .lca.json.gz), --majority, --threshold 0, 1 and the default, --scaled
coarser than the databases, abundance queries with and without --ignore-abundance, --query-from-file, -o and stdout,
and the error paths: no --db, a missing file, an old-format database, mixed ksizes and a query coarser than the
databases.  A SQLite database, which the plugin refuses and the reference reads, is checked on the plugin side alone.
The reference's side is stored in tests/golden/lca_cli_reference.json.gz as the SHA-256 of every file it wrote, its
report lines and its exit code; without the reference copy that build() makes, `python -m sourmash_b200.lca` is checked
against the stored side, with it the live reference must do exactly what is stored (SMB_PLUGIN_CLI_RECORD=1 rewrites
the stored side)."""
import gzip
import hashlib
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lca_cases as C  # noqa: E402
import test_plugin_through_reference_cli as base  # noqa: E402
from test_sig_kmers_through_reference_cli import report_lines as _kmers_report_lines  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "lca_cli_reference.json.gz")
ENTRY = ("b200lcaclassify = sourmash_b200.lca:Command_B200LcaClassify\n"
         "b200lcasummarize = sourmash_b200.lca:Command_B200LcaSummarize\n")
STDERR, STDOUT, RC = "<stderr>", "<stdout>", "<rc>"


def report_lines(text):
    return [line for line in _kmers_report_lines(text) if not line.startswith("...")]


def _digest(b):
    return hashlib.sha256(b).hexdigest()


def _write_inputs(work):
    "the fixtures, plus an abundance query, a k=21 database, a coarser query and a query list, all derived from them"
    lca = C.unpack_fixtures(os.path.join(work, "lca"))
    with open(os.path.join(lca, "TARA_ASE_MAG_00031.sig")) as fh:
        sig = json.load(fh)
    for sk in sig[0]["signatures"]:
        sk["abundances"] = [1 + (i * 7) % 5 for i in range(len(sk["mins"]))]
    with open(os.path.join(work, "abund.sig"), "w") as fh:
        json.dump(sig, fh)
    with open(os.path.join(lca, "TARA_ASE_MAG_00031.sig")) as fh:
        sig = json.load(fh)
    for sk in sig[0]["signatures"]:
        sk["max_hash"] //= 10
        sk["mins"] = [h for h in sk["mins"] if h <= sk["max_hash"]]
        sk.pop("md5sum", None)
    sig[0]["name"] = "coarse"
    with open(os.path.join(work, "coarse.sig"), "w") as fh:
        json.dump(sig, fh)
    with open(os.path.join(lca, "delmont-1.lca.json")) as fh:
        text = fh.read()
    assert '"ksize": 31' in text
    with open(os.path.join(work, "k21.lca.json"), "w") as fh:
        fh.write(text.replace('"ksize": 31', '"ksize": 21'))
    with open(os.path.join(work, "db.sqldb"), "wb") as fh:
        fh.write(b"SQLite format 3\x00" + bytes(84))
    with open(os.path.join(work, "list.txt"), "w") as fh:
        fh.write("lca/TARA_PSW_MAG_00136.sig\n")


@pytest.fixture(scope="module")
def lc(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("reflca"))
    site = os.path.join(tmp, "site")
    stored, recorded = {}, {}
    if LIVE:
        over_abi._stub_package(tmp, emul_lib.build())
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + ENTRY)
        if os.path.exists(STORED) and not os.environ.get("SMB_PLUGIN_CLI_RECORD"):
            with gzip.open(STORED, "rt") as fh:
                stored = json.load(fh)
    else:
        emul_lib.build()
        os.makedirs(site)
        with gzip.open(STORED, "rt") as fh:
            recorded = json.load(fh)
    with open(os.path.join(site, "sitecustomize.py"), "w") as fh:
        fh.write("import sys\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport emulated_boot\nemulated_boot.install()\n"
                 % (os.path.join(HERE, "host_emul"), ROOT))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, os.path.join(tmp, "reftests")]), PYTHONDONTWRITEBYTECODE="1")
    work = os.path.join(tmp, "work")
    os.makedirs(work)
    _write_inputs(work)

    def placeholders(b):
        return b.replace(work.encode(), b"@WORK@")

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=0):
        "a reference command (stored outside LIVE) or the plugin command: (rc, report lines, {file: sha256})"
        args = [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            out = recorded[key(args)]
            return out[RC], json.loads(out[STDERR].replace("@WORK@", work)), \
                {rel: v for rel, v in out.items() if rel not in (STDERR, RC)}
        if args[0] == "scripts" and not LIVE:
            cmd = [sys.executable, "-m", "sourmash_b200.lca", args[1][len("b200lca"):]] + args[2:]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + args
        before = base._files(work)
        r = subprocess.run(cmd, capture_output=True, env=env, cwd=work, timeout=900)
        err = r.stderr.decode("utf-8", "replace")
        assert r.returncode == rc, " ".join(args) + "\n" + err[-3000:]
        after = base._files(work)
        files = {STDOUT: _digest(placeholders(r.stdout))}
        for rel in sorted(after):
            if before.get(rel) != after[rel]:
                with open(os.path.join(work, rel), "rb") as fh:
                    files[rel] = _digest(placeholders(fh.read()))
        lines = report_lines(err)
        if args[0] != "scripts":
            out = dict(files)
            out[STDERR] = placeholders(json.dumps(lines).encode()).decode()
            out[RC] = r.returncode
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference did other than stored (%s)" % key(args)
        return r.returncode, lines, files

    def both(op, tag, *args, rc=0):
        "`lca <op>` and the plugin command with the same arguments; @OUT@ names get the side's tag"
        def side(name):
            return [a.replace("@OUT@", "%s_%s" % (tag, name)) for a in map(str, args)]
        want = run("lca", op, *side("ref"), rc=rc)
        got = run("scripts", "b200lca" + op, *side("b200"), rc=rc)
        assert got[0] == want[0], (tag, got[0], want[0])
        want_lines = [line.replace(tag + "_ref", tag + "_b200") for line in want[1]]
        assert got[1] == want_lines, (tag, "\n".join(got[1]), "\n".join(want_lines))
        rename = {rel.replace(tag + "_ref", tag + "_b200"): v for rel, v in want[2].items()}
        assert got[2] == rename, (tag, got[2], rename)
        return want

    run.work, run.both, run.env = work, both, env
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


TARA = ["lca/TARA_ASE_MAG_00031.sig", "lca/TARA_PSW_MAG_00136.sig", "lca/TARA_ANW_MAG_00005.sig",
        "lca/TARA_ASE_MAG_00007.sig"]


def test_classify(lc):
    "one and several --db, .gz, --majority, --threshold 0 / 1 / default, --scaled, --query-from-file, -o and stdout"
    lc.both("classify", "one", "--db", "lca/delmont-1.lca.json", "--query", *TARA, "-o", "@OUT@.csv")
    lc.both("classify", "stdout", "--db", "lca/delmont-1.lca.json.gz", "lca/delmont-2.lca.json", "--query", *TARA)
    lc.both("classify", "many", "--db", "lca/dir1.lca.json", "lca/dir2.lca.json", "--db", "lca/both.lca.json",
            "--query", *TARA, "-o", "@OUT@.csv")
    lc.both("classify", "majority", "--db", "lca/both.lca.json", "lca/delmont-1.lca.json", "--query", *TARA,
            "--majority", "-o", "@OUT@.csv")
    for t in ("0", "1"):
        lc.both("classify", "thr" + t, "--db", "lca/both.lca.json", "lca/dir1.lca.json", "--query", *TARA,
                "--threshold", t, "-o", "@OUT@.csv")
        lc.both("classify", "majthr" + t, "--db", "lca/both.lca.json", "--query", *TARA, "--majority",
                "--threshold", t)
    lc.both("classify", "scaled", "--db", "lca/delmont-1.lca.json", "lca/dir2.lca.json", "--query", *TARA,
            "--scaled", "100000", "-o", "@OUT@.csv")
    lc.both("classify", "fromfile", "--db", "lca/delmont-1.lca.json", "--query", TARA[0], "--query-from-file",
            "list.txt", "-o", "@OUT@.csv")
    lc.both("classify", "47", "--db", "lca/47+63.lca.json", "--query", *TARA, "-o", "@OUT@.csv")


def test_summarize(lc):
    "one and several --db, abundance queries with and without --ignore-abundance, thresholds, --scaled, -o"
    lc.both("summarize", "one", "--db", "lca/delmont-1.lca.json", "--query", *TARA, "-o", "@OUT@.csv")
    lc.both("summarize", "many", "--db", "lca/dir1.lca.json", "lca/dir2.lca.json", "lca/both.lca.json",
            "--query", *TARA)
    lc.both("summarize", "abund", "--db", "lca/delmont-1.lca.json.gz", "lca/dir1.lca.json", "--query", "abund.sig",
            TARA[1], "-o", "@OUT@.csv")
    lc.both("summarize", "ignore", "--db", "lca/delmont-1.lca.json", "lca/dir1.lca.json", "--query", "abund.sig",
            TARA[1], "--ignore-abundance", "-o", "@OUT@.csv")
    for t in ("0", "1"):
        lc.both("summarize", "thr" + t, "--db", "lca/both.lca.json", "--query", *TARA, "--threshold", t,
                "-o", "@OUT@.csv")
    lc.both("summarize", "scaled", "--db", "lca/delmont-1.lca.json", "lca/dir2.lca.json", "--query", *TARA,
            "--scaled", "100000", "-o", "@OUT@.csv")
    lc.both("summarize", "fromfile", "--db", "lca/both.lca.json", "--query-from-file", "list.txt")


def test_error_paths(lc):
    "no --db, a missing file, the old-format database, mixed ksizes, a query coarser than the databases"
    for op in ("classify", "summarize"):
        lc.both(op, op + "_nodb", "--query", TARA[0], rc=255)
        lc.both(op, op + "_missingdb", "--db", "lca/nope.lca.json", "--query", TARA[0], rc=255)
        lc.both(op, op + "_missingq", "--db", "lca/delmont-1.lca.json", "--query", "nope.sig", rc=255)
        lc.both(op, op + "_noq", "--db", "lca/delmont-1.lca.json", rc=255)
        lc.both(op, op + "_old", "--db", "lca/old-db-format-1.json", "--query", TARA[0], rc=1)
        lc.both(op, op + "_ksizes", "--db", "lca/delmont-1.lca.json", "k21.lca.json", "--query", TARA[0], rc=1)
        lc.both(op, op + "_coarse", "--db", "lca/delmont-1.lca.json", "--query", TARA[0], "coarse.sig", TARA[1],
                "-o", "@OUT@.csv", rc=1)


def test_sqlite_database_is_refused(lc):
    "SQLite LCA databases are out of scope: refused with a clear error before any query is read"
    cmd = [sys.executable, "-m", "sourmash_b200.lca", "classify", "--db", "db.sqldb", "--query", TARA[0]]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=lc.work, timeout=900, env=lc.env)
    assert r.returncode == 1
    assert "is a SQLite LCA database; only JSON LCA databases" in r.stderr
