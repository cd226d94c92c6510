"""`sourmash scripts b200lcaindex` next to the reference's `sourmash lca index`, through the reference's command line.

The setting of tests/test_lca_through_reference_cli.py: the reference's package runs over the emulated library and
finds this package's commands in a dist-info written next to it; both commands run on the same inputs (the reference's
spreadsheets and genome signatures, stored compressed under tests/golden/refdata/lca_index and refdata/lca, and inputs
derived from them), and their exit codes, the lines of their reports and the files they write must be equal.

Files are compared as follows.  A database is parsed with its key order kept and each idx list sorted: the reference
writes list(set), CPython's set order, and this package ascending idx, which is the same list whenever every idx is
below 8 -- so an uncompressed database of fewer than 8 signatures must also be byte-identical.  A --report file is
compared with the lines of each section sorted, since the reference lists Python sets there.  The reference reads a
--from-file list into a set, so the compared --from-file case lists one entry; a longer list, read in file order
here, is checked on the plugin side.  Every database is then
used by `lca classify` on the reference's side and `b200lcaclassify` on the plugin's, whose CSVs must be identical.
The reference's side is stored in tests/golden/lca_index_cli_reference.json.gz; without the reference copy that
build() makes, `python -m sourmash_b200.lca` is checked against the stored side, with it the live reference must do
exactly what is stored (SMB_PLUGIN_CLI_RECORD=1 rewrites the stored side)."""
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lca_cases  # noqa: E402
import lca_index_cases as C  # noqa: E402
import test_plugin_through_reference_cli as base  # noqa: E402
from test_lca_through_reference_cli import report_lines  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "lca_index_cli_reference.json.gz")
ENTRY = ("b200lcaclassify = sourmash_b200.lca:Command_B200LcaClassify\n"
         "b200lcaindex = sourmash_b200.lca:Command_B200LcaIndex\n")
STDERR, STDOUT, RC = "<stderr>", "<stdout>", "<rc>"


def _digest(b):
    return hashlib.sha256(b).hexdigest()


def _normal_database(raw):
    "a database's members in file order, hashval_to_idx's keys in file order with sorted idx lists"
    d = json.loads(raw, object_pairs_hook=list)
    out = []
    for k, v in d:
        if k == "hashval_to_idx":
            v = [(h, sorted(ix)) for h, ix in v]
        out.append((k, v))
    return json.dumps(out).encode()


def _normal_report(raw):
    sections = raw.decode().split("----\n")
    return "----\n".join(s.split("\n", 1)[0] + "\n" + "\n".join(sorted(s.split("\n")[1:])) for s in sections).encode()


def _file_digests(rel, raw):
    "what of a written file must agree between the sides: {name: sha256}"
    if rel.endswith(".gz"):
        raw = gzip.decompress(raw)
    if ".lca.json" in rel:
        out = {rel: _digest(_normal_database(raw))}
        if not rel.endswith(".gz") and all(
                int(k) < 8 for k in json.loads(raw)["idx_to_lid"]) and len(json.loads(raw)["ident_to_idx"]) < 8:
            out[rel + "#bytes"] = _digest(raw)
        return out
    if rel.endswith(".report"):
        return {rel: _digest(_normal_report(raw))}
    return {rel: _digest(raw)}


def _write_inputs(work):
    "the fixtures, plus spreadsheets and signatures derived from them"
    lca_cases.unpack_fixtures(os.path.join(work, "lca"))
    C.unpack_fixtures(work)
    with open(os.path.join(work, "delmont-1.csv")) as fh:
        rows = [line.rstrip("\n").split(",") for line in fh]
    with open(os.path.join(work, "delmont-1-C3.csv"), "w") as fh:          # -C 3: one column before the ranks
        for r in rows:
            fh.write(",".join([r[0], "extra"] + r[1:]) + "\n")
    with open(os.path.join(work, "delmont-1-noheader.csv"), "w") as fh:
        for r in rows[1:]:
            fh.write(",".join(r) + "\n")
    with open(os.path.join(work, "genus-only.csv"), "w") as fh:           # 60 lineages, none at species
        fh.write(",".join(rows[0]) + "\n")
        for i in range(60):
            fh.write("g%d,Bacteria,P%d,C,O,F,G%d\n" % (i, i % 3, i) if i else ",".join(rows[1][:7]) + "\n")
    with open(os.path.join(work, "split.csv"), "w") as fh:
        fh.write(",".join(rows[0]) + "\n")
        fh.write(",".join(["TARA_ASE_MAG_00031"] + rows[1][1:]) + "\n")
        fh.write(",".join(["TARA_PSW_MAG_00136.2"] + rows[1][1:4]) + "\n")
    with open(os.path.join(work, "lca", "TARA_ASE_MAG_00031.sig")) as fh:
        sig = json.load(fh)
    renamed = json.loads(json.dumps(sig))
    renamed[0]["name"] = "TARA_ASE_MAG_00031.1 Alteromonas macleodii"
    with open(os.path.join(work, "renamed-31.sig"), "w") as fh:
        json.dump(renamed, fh)
    with open(os.path.join(work, "lca", "TARA_PSW_MAG_00136.sig")) as fh:
        other = json.load(fh)
    other[0]["name"] = "TARA_PSW_MAG_00136.2 second"
    with open(os.path.join(work, "renamed-136.sig"), "w") as fh:
        json.dump(other, fh)
    unnamed = json.loads(json.dumps(sig))
    unnamed[0].pop("name", None)
    unnamed[0]["filename"] = "TARA_ASE_MAG_00031"
    with open(os.path.join(work, "unnamed.sig"), "w") as fh:
        json.dump(unnamed, fh)
    num = json.loads(json.dumps(sig))
    for sk in num[0]["signatures"]:
        sk["num"], sk["max_hash"] = 100, 0
        sk["mins"] = sk["mins"][:100]
        sk.pop("md5sum", None)
    num[0]["name"] = "num-sketch"
    with open(os.path.join(work, "num.sig"), "w") as fh:
        json.dump(num, fh)
    os.makedirs(os.path.join(work, "mixed"))                                 # a directory with a file that is no .sig
    for name in sorted(os.listdir(os.path.join(work, "dir1")))[:3]:
        shutil.copy(os.path.join(work, "dir1", name), os.path.join(work, "mixed", name))
    shutil.copy(os.path.join(work, "dir1", name), os.path.join(work, "mixed", "copy.json"))
    with open(os.path.join(work, "mixed", "notes.txt"), "w") as fh:
        fh.write("not a signature\n")
    with open(os.path.join(work, "list.txt"), "w") as fh:                  # one entry: see test_index_inputs
        fh.write("dir2\n")
    with open(os.path.join(work, "list2.txt"), "w") as fh:
        fh.write("lca/TARA_PSW_MAG_00136.sig\ndir2\n")
    prot = os.path.join(HERE, "golden", "refdata", "prot")
    with open(os.path.join(work, "prot.csv"), "w") as fh:
        fh.write(",".join(rows[0]) + "\n")
        fh.write("GCA_001593925,Archaea,Euryarchaeota,Methanomicrobia,Methanomicrobiales,F,G,S1\n")
        fh.write("GCA_001593935,Archaea,Euryarchaeota,Methanomicrobia,Methanomicrobiales,F,G,S2\n")
    for m in ("protein", "dayhoff", "hp"):
        shutil.copy(os.path.join(prot, m + ".zip"), os.path.join(work, m + ".zip"))
    with open(os.path.join(work, "exists.lca.json"), "w") as fh:
        fh.write("{}")


@pytest.fixture(scope="module")
def lc(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("reflcaindex"))
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
                    files.update(_file_digests(rel, placeholders(fh.read())))
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

    def index(tag, *args, rc=0, query="lca/TARA_ASE_MAG_00031.sig"):
        "both sides' `lca index`, then `lca classify` of ``query`` against each side's database"
        both("index", tag, *args, rc=rc)
        out = [a for a in args if "@OUT@" in a]
        if rc == 0 and query:
            db = out[0] if out[0].endswith((".lca.json", ".lca.json.gz")) else out[0] + ".lca.json"
            both("classify", tag, "--db", db, "--query", query)

    run.work, run.both, run.index, run.env = work, both, index, env
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


TARA = ["lca/TARA_ASE_MAG_00031.sig", "lca/TARA_PSW_MAG_00136.sig", "lca/TARA_ANW_MAG_00005.sig",
        "lca/TARA_ASE_MAG_00007.sig"]


def test_index_spreadsheets(lc):
    "basic, .lca.json.gz, a name without extension, --tabs, -C 3, --no-headers, --split-identifiers"
    lc.index("basic", "delmont-1.csv", "@OUT@.lca.json", TARA[0])
    lc.index("gz", "delmont-1.csv", "@OUT@.lca.json.gz", *TARA)
    lc.index("noext", "delmont-2.csv", "@OUT@", *TARA)
    lc.index("tabs", "delmont-1.tsv", "@OUT@.lca.json", TARA[0], "--tabs", "--no-headers")
    lc.index("c3", "delmont-1-C3.csv", "@OUT@.lca.json", TARA[0], "-C", "3")
    lc.index("nohead", "delmont-1-noheader.csv", "@OUT@.lca.json", *TARA[:2], "--no-headers")
    lc.index("split", "split.csv", "@OUT@.lca.json", "renamed-31.sig", "renamed-136.sig", "--split-identifiers")
    lc.index("splitkeep", "split.csv", "@OUT@.lca.json", "renamed-31.sig", "renamed-136.sig",
             "--split-identifiers", "--keep-identifier-versions")
    lc.both("index", "c1", "delmont-1.csv", "@OUT@.lca.json", TARA[0], "-C", "1", rc=255)


def test_index_inputs(lc):
    "directories with and without -f, --from-file, the real spreadsheet with --report, duplicates, an empty name"
    lc.index("dirs", "tara-delmont-SuppTable3.csv", "@OUT@.lca.json", "dir1", "dir2", "-C", "3",
             "--split-identifiers", "-f", query="dir1/TARA_ANE_MAG_00044.fa.gz.sig")
    lc.index("report", "tara-delmont-SuppTable3.csv", "@OUT@.lca.json", "dir1", "dir2", TARA[0], "-C", "3",
             "--split-identifiers", "-f", "--report", "@OUT@.report")
    lc.index("mixed", "delmont-1.csv", "@OUT@.lca.json", "mixed", TARA[0])
    lc.index("mixedf", "delmont-1.csv", "@OUT@.lca.json", "mixed", TARA[0], "-f")
    # the reference reads a --from-file list into a set, so only a one-entry list gives it an order that does not
    # follow the string hash seed; a longer list is read in file order here (checked on the plugin side below)
    lc.index("fromfile", "delmont-1.csv", "@OUT@.lca.json", TARA[0], "--from-file", "list.txt")
    lc.index("dups", "delmont-1.csv", "@OUT@.lca.json", TARA[0], TARA[0], TARA[1], "--report", "@OUT@.report")
    lc.index("unnamed", "delmont-1.csv", "@OUT@.lca.json", "unnamed.sig", TARA[1])
    lc.index("root", "lca-root/tax.csv", "@OUT@.lca.json", "lca-root/TARA_MED_MAG_00029.fa.sig",
             "lca-root/TOBG_MED-875.fna.gz.sig", query="lca-root/TOBG_MED-875.fna.gz.sig")


def test_index_taxonomy_checks(lc):
    "--require-taxonomy, --fail-on-missing-taxonomy, too few species with and without -f, bad spreadsheets"
    lc.index("require", "delmont-1.csv", "@OUT@.lca.json", *TARA, "--require-taxonomy")
    lc.both("index", "failmissing", "delmont-1.csv", "@OUT@.lca.json", *TARA, "--require-taxonomy",
            "--fail-on-missing-taxonomy", rc=255)
    lc.both("index", "fewspecies", "genus-only.csv", "@OUT@.lca.json", TARA[0], rc=255)
    lc.index("fewspeciesf", "genus-only.csv", "@OUT@.lca.json", TARA[0], "-f")
    lc.index("bad1", "bad-spreadsheet.csv", "@OUT@.lca.json", TARA[0])
    lc.index("bad1f", "bad-spreadsheet.csv", "@OUT@.lca.json", TARA[0], "-f")
    lc.both("index", "bad2", "bad-spreadsheet-2.csv", "@OUT@.lca.json", TARA[0], rc=1)
    lc.index("bad2f", "bad-spreadsheet-2.csv", "@OUT@.lca.json", TARA[0], "-f")
    lc.index("bad3", "bad-spreadsheet-3.csv", "@OUT@.lca.json", TARA[0])


def test_index_errors(lc):
    "an existing output, a num sketch, --scaled finer than a sketch, no hashes, no signatures"
    lc.both("index", "exists", "delmont-1.csv", "exists.lca.json", TARA[0], rc=255)
    lc.both("index", "num", "delmont-1.csv", "@OUT@.lca.json", TARA[0], "num.sig", rc=255)
    lc.both("index", "fine", "delmont-1.csv", "@OUT@.lca.json", TARA[0], "--scaled", "1000", rc=255)
    lc.both("index", "nohash", "delmont-1.csv", "@OUT@.lca.json", TARA[0], "--scaled", "1e18", rc=1)
    lc.both("index", "nosig", "delmont-1.csv", "@OUT@.lca.json", rc=1)
    lc.index("coarse", "delmont-1.csv", "@OUT@.lca.json", *TARA, "--scaled", "100000")


def test_index_protein_moltypes(lc):
    "protein, dayhoff and hp sketches from .zip collections, k in residues"
    for m in ("protein", "dayhoff", "hp"):
        lc.index(m, "prot.csv", "@OUT@.lca.json", m + ".zip", "-k", "19", "--" + m, "--scaled", "100", query=None)


def test_sql_output_is_refused(lc):
    "SQLite output is out of scope: refused with exit -1 before anything is loaded"
    cmd = [sys.executable, "-m", "sourmash_b200.lca", "index", "delmont-1.csv", "sqlout", TARA[0], "-F", "sql"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=lc.work, timeout=900, env=lc.env)
    assert r.returncode == 255
    assert "SQLite LCA databases (-F sql) are not supported" in r.stderr
    assert not os.path.exists(os.path.join(lc.work, "sqlout.lca.sql"))


def test_from_file_list_is_read_in_file_order(lc):
    "a --from-file list of several entries gives idx in the list's order, after the command-line signatures"
    out = os.path.join(lc.work, "fileorder.lca.json")
    cmd = [sys.executable, "-m", "sourmash_b200.lca", "index", "delmont-1.csv", out, TARA[0], "--from-file",
           "list2.txt"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=lc.work, timeout=900, env=lc.env)
    assert r.returncode == 0, r.stderr[-3000:]
    with open(out) as fh:
        idents = list(json.load(fh)["ident_to_idx"])
    dir2 = sorted(n[:-len(".fa.gz.sig")] for n in os.listdir(os.path.join(lc.work, "dir2")))
    assert idents[:2] == ["TARA_ASE_MAG_00031", "TARA_PSW_MAG_00136"], idents
    assert idents[2:] == [n for n in dir2 if n not in idents[:2]], idents      # dir2's copy of 00031 is an md5 twin
