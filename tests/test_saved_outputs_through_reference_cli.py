"""The signature outputs of `sourmash scripts b200prefetch | b200gather | b200search` next to the reference's `prefetch |
gather | search`, through the reference's command line.

The setting of tests/test_sig_setops_through_reference_cli.py: the reference's package runs over the emulated library and
finds this package's commands in a dist-info written next to it; both commands run on the same inputs, and every file
they write (the SHA-256 of its bytes, of the decompressed bytes for a .gz file, whose gzip header stores a time), what
a `-` target writes to stdout, the exit codes and the report lines about the saved outputs must be equal.  The other
report lines differ by design (the plugin commands print a shorter report) and are covered by
tests/test_plugin_through_reference_cli.py.

Options: prefetch --save-matches --save-matching-hashes --save-unmatched-hashes; gather --save-matches --save-prefetch
--save-prefetch-csv --output-unassigned; search --save-matches.  Inputs: a flat query (47 / 63, the gather metagenome
against the 12 genomes), an abundance query with and without --ignore-abundance, --scaled coarser than the query, a
threshold no row reaches, a directory holding two copies of one signature under different names, two database
arguments, a database coarser than the query, .sig.gz and `-` targets; a .zip target is refused by the plugin commands.
The reference's side is stored in tests/golden/saved_outputs_cli_reference.json.gz; without the reference copy that
build() makes, `python -m sourmash_b200.plugin` is checked against it, with it the live reference must do exactly what is
stored (SMB_PLUGIN_CLI_RECORD=1 rewrites the stored side)."""
import base64
import gzip
import hashlib
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_plugin_through_reference_cli as base  # noqa: E402
from test_sig_kmers_through_reference_cli import report_lines as _kmers_report_lines  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "saved_outputs_cli_reference.json.gz")
STDERR, STDOUT, RC, FILES = "<stderr>", "<stdout>", "<rc>", "<files>"


def report_lines(text):
    "the lines about the saved outputs, and the last line of an error"
    lines = _kmers_report_lines(text)
    keep = [x for x in lines if x.startswith("saving ") or x.startswith("no unassigned hashes")]
    errors = [x for x in lines if x.startswith("ERROR") or "Error: " in x.split(" ")[0] + " "]
    return keep + errors[-1:]


def _digest(rel, b):
    return hashlib.sha256(gzip.decompress(b) if rel.endswith(".gz") else b).hexdigest()


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refsaved"))
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
    os.makedirs(os.path.join(work, "twins"))
    # one database directory holding 47 twice under two names: one md5, two signatures
    with open(os.path.join(data, "47.fa.sig")) as fh:
        sig = json.load(fh)
    for name in ("first", "second"):
        sig[0]["name"] = "47 as " + name
        with open(os.path.join(work, "twins", name + ".sig"), "w") as fh:
            json.dump(sig, fh)

    def placeholders(b):
        return b.replace(work.encode(), b"@WORK@").replace(data.encode(), b"@DATA@")

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=0):
        "a reference command (stored outside LIVE) or the plugin command: (rc, report lines, {file: sha256})"
        args = [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            out = recorded[key(args)]
            for rel, text in out.get(FILES, {}).items():            # the sketches later commands read
                with open(os.path.join(work, rel), "wb") as fh:
                    fh.write(base64.b64decode(text).replace(b"@WORK@", work.encode()).replace(b"@DATA@", data.encode()))
            return out[RC], json.loads(out[STDERR].replace("@WORK@", work).replace("@DATA@", data)), \
                {rel: v for rel, v in out.items() if rel not in (STDERR, RC, FILES)}
        if args[0] == "scripts" and not LIVE:
            cmd = [sys.executable, "-m", "sourmash_b200.plugin"] + args[1:]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + args
        before = base._files(work)
        r = subprocess.run(cmd, capture_output=True, env=env, cwd=work, timeout=900)
        err = r.stderr.decode("utf-8", "replace")
        assert r.returncode == rc, " ".join(args) + "\n" + err[-3000:]
        after = base._files(work)
        files = {STDOUT: _digest("", placeholders(r.stdout))} if "-" in args else {}
        for rel in sorted(after):
            if before.get(rel) != after[rel]:
                with open(os.path.join(work, rel), "rb") as fh:
                    files[rel] = _digest(rel, placeholders(fh.read()))
        lines = report_lines(err)
        if args[0] != "scripts":
            out = dict(files)
            out[STDERR] = placeholders(json.dumps(lines).encode()).decode()
            out[RC] = r.returncode
            if args[0] == "sig":
                out[FILES] = {}
                for rel in files:
                    if rel != STDOUT:
                        with open(os.path.join(work, rel), "rb") as fh:
                            out[FILES][rel] = base64.b64encode(placeholders(fh.read())).decode()
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference did other than stored (%s)" % key(args)
        return r.returncode, lines, files

    def both(cmd, tag, *args, rc=0):
        "the reference's command and the plugin command with the same arguments; @OUT@ names get the side's tag"
        def side(name):
            return [a.replace("@OUT@", "%s_%s" % (tag, name)) for a in map(str, args)]
        want = run(cmd, *side("ref"), rc=rc)
        got = run("scripts", "b200" + cmd, *side("b200"), rc=rc)
        assert got[0] == want[0], (tag, got[0], want[0])
        rename = [x.replace(tag + "_ref", tag + "_b200") for x in want[1]]
        assert got[1] == rename, (tag, "\n".join(got[1]), "\n".join(rename))
        rename = {rel.replace(tag + "_ref", tag + "_b200"): v for rel, v in want[2].items()}
        assert got[2] == rename, (tag, got[2], rename)
        return want

    run.work, run.data, run.both, run.env = work, data, both, env
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


def _gather(sk):
    d = os.path.join(sk.data, "gather")
    return [os.path.join(d, n) for n in sorted(os.listdir(d)) if n.startswith("GCF")]


PREFETCH_OUT = ["--save-matches", "@OUT@_m.sig", "--save-matching-hashes", "@OUT@_k.sig",
                "--save-unmatched-hashes", "@OUT@_u.sig.gz"]
GATHER_OUT = ["--save-matches", "@OUT@_m.sig", "--save-prefetch", "@OUT@_p.sig.gz", "--save-prefetch-csv", "@OUT@_p.csv",
              "--output-unassigned", "@OUT@_u.sig"]


def test_flat_queries(sk):
    "47 against 63, the gather metagenome against the 12 genomes; every option of the three commands"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    combined = os.path.join(d, "gather", "combined.sig")
    sk.both("prefetch", "pf47", sig47, sig63, "--threshold-bp", "0", *PREFETCH_OUT)
    sk.both("prefetch", "pfmeta", combined, *_gather(sk), "-k", "21", *PREFETCH_OUT)
    sk.both("gather", "g47", sig47, sig63, "--threshold-bp", "0", *GATHER_OUT)
    sk.both("gather", "gmeta", combined, *_gather(sk), "-k", "21", "--threshold-bp", "0", *GATHER_OUT)
    sk.both("search", "s47", sig47, sig63, os.path.join(d, "2.fa.sig"), "--save-matches", "@OUT@_m.sig")
    sk.both("search", "smeta", combined, *_gather(sk), "-k", "21", "--containment", "--save-matches", "@OUT@_m.sig.gz")


def test_abundance_queries(sk):
    "track_abund 47 / 63, with and without --ignore-abundance; --scaled coarser than the query"
    d = sk.data
    ab47, ab63 = os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "track_abund", "63.fa.sig")
    sk.both("prefetch", "pfab", ab47, ab63, "--threshold-bp", "0", *PREFETCH_OUT)
    sk.both("prefetch", "pfabsc", ab47, ab63, "--threshold-bp", "0", "--scaled", "2000", *PREFETCH_OUT)
    sk.both("gather", "gab", ab47, ab63, "--threshold-bp", "0", *GATHER_OUT)
    sk.both("gather", "gabig", ab47, ab63, "--threshold-bp", "0", "--ignore-abundance", *GATHER_OUT)
    sk.both("gather", "gabsc", ab47, ab63, "--threshold-bp", "0", "--scaled", "2000", *GATHER_OUT)
    sk.both("search", "sab", ab47, ab63, "--save-matches", "@OUT@_m.sig")
    sk.both("search", "sabig", ab47, ab63, "--ignore-abundance", "--save-matches", "@OUT@_m.sig")


def test_unreached_threshold(sk):
    "no row reaches the threshold: empty known, the whole query unknown, unassigned keeps the query's name"
    d = sk.data
    ab47, sig63 = os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "63.fa.sig")
    sig47 = os.path.join(d, "47.fa.sig")
    sk.both("prefetch", "pfnone", sig47, sig63, "--threshold-bp", "4000000", *PREFETCH_OUT)
    sk.both("prefetch", "pfnonesc", ab47, sig63, "--threshold-bp", "2000000", "--scaled", "2000", *PREFETCH_OUT)
    sk.both("gather", "gnone", sig47, sig63, "--threshold-bp", "4000000", *GATHER_OUT)
    sk.both("gather", "gnoneab", ab47, sig63, "--threshold-bp", "4000000", *GATHER_OUT)


def test_databases_md5_twins_and_two_arguments(sk):
    "a directory holding one signature twice under two names (--save-prefetch keeps one); two database arguments"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    sk.both("gather", "gtwins", sig47, "twins/", sig63, "--threshold-bp", "0", *GATHER_OUT)
    sk.both("gather", "gtwo", sig47, "twins/", sig63, "twins/", "--threshold-bp", "0", *GATHER_OUT)
    sk.both("prefetch", "pftwins", sig47, "twins/", sig63, "--threshold-bp", "0", *PREFETCH_OUT)
    sk.both("search", "stwins", sig47, "twins/", sig63, "--save-matches", "@OUT@_m.sig")


def test_a_database_coarser_than_the_query(sk):
    "63 downsampled to scaled=10000 as the database of the 47 query"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    sk("sig", "downsample", sig63, "--scaled", "10000", "-o", "63s10k.sig")
    sk.both("prefetch", "pfcoarse", sig47, "63s10k.sig", "--threshold-bp", "0", *PREFETCH_OUT)
    sk.both("search", "scoarse", sig47, "63s10k.sig", "--save-matches", "@OUT@_m.sig")
    sk.both("gather", "gcoarse", sig47, "63s10k.sig", "--threshold-bp", "0", "--save-matches", "@OUT@_m.sig")
    sk.both("gather", "gcoarsenone", sig47, "63s10k.sig", "--threshold-bp", "4000000", "--output-unassigned", "@OUT@_u.sig")
    sk.both("gather", "gcoarseu", sig47, "63s10k.sig", "--threshold-bp", "0", "--output-unassigned", "@OUT@_u.sig", rc=1)


def test_stdout_targets(sk):
    "`-` writes the signatures to stdout"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    sk.both("prefetch", "pfout", sig47, sig63, "--threshold-bp", "0", "--save-matching-hashes", "-")
    sk.both("prefetch", "pfoutm", sig47, sig63, "--threshold-bp", "0", "--save-matches", "-")


@pytest.mark.parametrize("target", ["out.zip", "out.sqldb", "outdir/"])
def test_collection_targets_are_refused(sk, target):
    "the plugin commands write .sig files only: a collection target is refused before anything is loaded, exit -1"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    for cmd, opt in (("b200prefetch", "--save-unmatched-hashes"), ("b200gather", "--save-prefetch"),
                     ("b200search", "--save-matches")):
        rc, lines, files = sk("scripts", cmd, sig47, sig63, opt, target, rc=255)
        assert files == {}, (cmd, files)
        assert len(lines) == 1 and lines[0].startswith("ERROR: cannot save signatures to") and target in lines[0], lines
