"""`sourmash scripts b200sketch | b200compare | b200search | b200gather | b200prefetch` through the REFERENCE's command line.

north_star asks for the hot paths "behind the reference's own plugin API": the reference loads command plugins from the
entry-point group `sourmash.cli_script` (src/sourmash/plugins.py:8-12, 91-186).  Here the reference's package (loaded in
place over this library, as in test_reference_python_over_abi.py) finds this package's entry points in a dist-info written
next to it, and every plugin command is run next to the reference's own command on the same inputs:

    sourmash sketch dna / protein / translate   vs   sourmash scripts b200sketch      -> equal signatures
    sourmash compare                            vs   sourmash scripts b200compare     -> equal matrix, labels, CSV
    sourmash search / gather / prefetch         vs   sourmash scripts b200search ...  -> byte-identical CSV files

Both sides run on the emulated library; the reference's commands go sketch by sketch and pair by pair through the C ABI,
the plugin commands through this package's batched entry points.

What the reference's commands write is stored in tests/golden/plugin_cli_reference.json.gz (paths of the inputs and of the
work directory replaced by placeholders), so without the reference the test runs the plugin commands
(`python -m sourmash_b200.plugin ...`) on the same inputs and compares them with the stored files.  With the reference
copy that build() makes (oracle/reference.py) the reference's commands run live, through its plugin loader, and what
they write must equal the stored files; SMB_PLUGIN_CLI_RECORD=1 rewrites the stored file instead."""
import base64
import csv
import glob
import gzip
import io
import json
import os
import shutil
import subprocess
import sys
import zipfile
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_reference_python_over_abi as over_abi  # noqa: E402

REF = over_abi.REF
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
LIVE = os.path.isdir(os.path.join(REF, "src", "sourmash"))
STORED = os.path.join(GOLDEN, "plugin_cli_reference.json.gz")
DATA = os.path.join(REF, "tests", "test-data")        # without the reference: a copy of the inputs in the reference's layout
DATA_FILES = (["genome-s10.fa.gz", "genome-s11.fa.gz", "genome-s12.fa.gz", "short.fa", "short2.fa", "short3.fa", "ecoli.faa",
               "ecoli.genes.fna", "47.fa.sig", "63.fa.sig", "2.fa.sig", "track_abund/47.fa.sig", "track_abund/63.fa.sig",
               "prot/protein/GCA_001593925.1_ASM159392v1_protein.faa.gz.sig",
               "prot/protein/GCA_001593935.1_ASM159393v1_protein.faa.gz.sig", "gather/combined.sig"]
              + ["gather/" + os.path.basename(p) for p in sorted(glob.glob(os.path.join(GOLDEN, "gather", "GCF*.sig")))])

COMMANDS = ("B200Sketch", "B200Compare", "B200Search", "B200Gather", "B200Prefetch")


def _stored_inputs(dest):
    "the reference's input files of this module, from tests/golden (as they are, or gzipped under refdata/)"
    for rel in DATA_FILES:
        out = os.path.join(dest, rel)
        os.makedirs(os.path.dirname(out), exist_ok=True)
        for src in (os.path.join(GOLDEN, "refdata", rel), os.path.join(GOLDEN, rel)):
            if os.path.exists(src):
                shutil.copy(src, out)
                break
        else:
            with gzip.open(os.path.join(GOLDEN, "refdata", rel + ".gz")) as fh, open(out, "wb") as o:
                o.write(fh.read())


def _comparable(rel, data):
    """What must be equal between two runs of a reference command: the bytes, except for a .zip archive, which records
    when it was written -- its members' names and contents (gzip members decompressed: their headers carry a time too)."""
    if not rel.endswith(".zip"):
        return data
    with zipfile.ZipFile(io.BytesIO(data)) as z:
        return sorted((i.filename, gzip.decompress(z.read(i)) if i.filename.endswith(".gz") else z.read(i))
                      for i in z.infolist())


def _files(work):
    found = {}
    for top, _dirs, names in os.walk(work):
        for n in names:
            path = os.path.join(top, n)
            found[os.path.relpath(path, work)] = os.stat(path).st_mtime_ns
    return found


@pytest.fixture(scope="module")
def cli(tmp_path_factory):
    global DATA
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refcli"))
    site = os.path.join(tmp, "site")
    if LIVE:
        over_abi._stub_package(tmp, emul_lib.build())
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")     # what `pip install .` writes from pyproject.toml
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(ROOT, "pyproject.toml")) as fh:
            declared = [line.split("=")[0].strip() for line in fh if "sourmash_b200.plugin:Command_" in line]
        assert declared == [c.lower() for c in COMMANDS]               # the entry points written below are the declared ones
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + "".join("%s = sourmash_b200.plugin:Command_%s\n" % (c.lower(), c) for c in COMMANDS))
        recorded = {}
        stored = {}
        if os.path.exists(STORED) and not os.environ.get("SMB_PLUGIN_CLI_RECORD"):
            with gzip.open(STORED, "rt") as fh:                         # what the live reference writes must match it
                stored = json.load(fh)
    else:
        emul_lib.build()
        os.makedirs(site)
        DATA = os.path.join(tmp, "test-data")
        _stored_inputs(DATA)
        with gzip.open(STORED, "rt") as fh:
            recorded = json.load(fh)
    with open(os.path.join(site, "sitecustomize.py"), "w") as fh:       # this package too binds the emulated library
        fh.write("import sys\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport emulated_boot\nemulated_boot.install()\n"
                 % (os.path.join(HERE, "host_emul"), ROOT))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, os.path.join(tmp, "reftests")]), PYTHONDONTWRITEBYTECODE="1")
    work = os.path.join(tmp, "work")
    os.makedirs(work)

    def placeholders(data):
        return data.replace(work.encode(), b"@WORK@").replace(DATA.encode(), b"@DATA@")

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=(0,)):
        if args[0] == "scripts" and not LIVE:                           # the plugin commands without the reference's loader
            cmd = [sys.executable, "-m", "sourmash_b200.plugin"] + [str(a) for a in args[1:]]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:                           # a reference command: what it wrote, from the stored file
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            for rel, text in recorded[key(args)].items():
                data = base64.b64decode(text).replace(b"@WORK@", work.encode()).replace(b"@DATA@", DATA.encode())
                os.makedirs(os.path.dirname(os.path.join(work, rel)), exist_ok=True)
                with open(os.path.join(work, rel), "wb") as fh:
                    fh.write(data)
            return None
        before = _files(work)
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=work, timeout=900)
        assert r.returncode in rc, " ".join(map(str, args)) + "\n" + r.stdout[-2000:] + r.stderr[-3000:]
        if args[0] != "scripts":                                        # LIVE: keep what the reference's command wrote
            after = _files(work)
            out = {}
            for rel in sorted(after):
                if before.get(rel) != after[rel]:
                    with open(os.path.join(work, rel), "rb") as fh:
                        out[rel] = base64.b64encode(placeholders(fh.read())).decode()
            recorded[key(args)] = out
            if key(args) in stored:
                assert sorted(stored[key(args)]) == sorted(out), "the reference wrote other files than the stored ones"
                for rel, text in out.items():
                    assert _comparable(rel, base64.b64decode(text)) == _comparable(rel, base64.b64decode(stored[key(args)][rel])), \
                        "the reference's %s differs from the stored one (%s)" % (rel, key(args))
        return r

    def load(path):                                                      # with the reference's own loader (or this package's)
        code = ("import %s as sourmash, sys, json\n"
                "print(json.dumps(sorted([ss.name, ss.filename, ss.md5sum(), ss.minhash.ksize, ss.minhash.moltype, "
                "ss.minhash.scaled, ss.minhash.num, int(ss.minhash.track_abundance), sorted(ss.minhash.hashes.items())] "
                "for ss in sourmash.load_file_as_signatures(sys.argv[1]))))") % ("sourmash" if LIVE else "sourmash_b200")
        r = subprocess.run([sys.executable, "-c", code, path], capture_output=True, text=True, env=env, cwd=work, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        return r.stdout

    def together(*cmdlines):
        "several command lines: the reference's one by one (what each writes is noted), then the plugin's at once"
        from concurrent.futures import ThreadPoolExecutor
        for c in cmdlines:
            if c[0] != "scripts":
                run(*c)
        plugin = [c for c in cmdlines if c[0] == "scripts"]
        with ThreadPoolExecutor(max(1, len(plugin))) as pool:
            return list(pool.map(lambda c: run(*c), plugin))

    def loads(*paths):
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(len(paths)) as pool:
            return list(pool.map(load, paths))

    run.work, run.load, run.loads, run.together = work, load, loads, together
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


@pytest.mark.skipif(not LIVE, reason="the reference's own plugin loader: needs the reference copy that build() makes (oracle/reference.py)")
def test_the_reference_lists_the_plugin_commands(cli):
    r = cli("scripts", rc=(0, 1))                          # no command given: the list of commands, exit status 1
    out = r.stderr + r.stdout
    for c in COMMANDS:
        assert "sourmash scripts %s" % c.lower() in out


@pytest.mark.parametrize("kind,params,files", [
    ("dna", "k=21,k=31,k=51,scaled=1000", ["genome-s10.fa.gz", "genome-s11.fa.gz", "genome-s12.fa.gz"]),
    ("dna", "k=31,scaled=100,abund", ["short.fa", "short2.fa"]),
    ("dna", "k=21,num=500", ["genome-s10.fa.gz"]),
    ("protein", "k=7,scaled=10", ["ecoli.faa"]),
    ("translate", "k=7,scaled=10,dayhoff", ["short.fa"]),
])
def test_sketch_commands_write_equal_signatures(cli, kind, params, files):
    paths = [os.path.join(DATA, f) for f in files]
    tag = "%s_%s" % (kind, zlib.crc32(params.encode()) % 10**6)
    extra, plugin_params = [], params
    if kind != "dna":
        moltype = "dayhoff" if "dayhoff" in params else "hp" if ",hp" in params else "protein"
        extra = ["--moltype", moltype] + (["--input-is-protein"] if kind == "protein" else [])
        plugin_params = params.replace(",dayhoff", "").replace(",hp", "")
    cli.together(["sketch", kind, "-p", params, *paths, "-o", tag + "_ref.sig"],
                 ["scripts", "b200sketch", "-p", plugin_params, *paths, "-o", tag + "_b200.sig", *extra])
    want, got = cli.loads(tag + "_ref.sig", tag + "_b200.sig")
    assert len(want) > 100 and got == want
    assert open(os.path.join(cli.work, tag + "_ref.sig")).read() == open(os.path.join(cli.work, tag + "_b200.sig")).read()   # the .sig files themselves


@pytest.mark.parametrize("flags,files", [
    (["--singleton"], ["short.fa"]),
    (["--name-from-first"], ["short.fa", "short2.fa"]),
    (["--merge", "all of them"], ["short.fa", "short2.fa", "short3.fa"]),
    (["--singleton", "--name-from-first"], ["ecoli.genes.fna"]),
])
def test_sketch_naming_modes_write_equal_signatures(cli, flags, files):
    "--singleton (one signature per record), --name-from-first, --merge NAME: names, filenames and sketches (command_sketch.py:662-789)"
    paths = [os.path.join(DATA, f) for f in files]
    tag = "naming_" + "".join(f.strip("-")[:4] for f in flags if f.startswith("--"))
    cli.together(["sketch", "dna", "-p", "k=21,k=31,scaled=10", *paths, "-o", tag + "_ref.sig", *flags],
                 ["scripts", "b200sketch", "-p", "k=21,k=31,scaled=10", *paths, "-o", tag + "_b200.sig", *flags])
    want, got = cli.loads(tag + "_ref.sig", tag + "_b200.sig")
    assert len(want) > 100 and got == want
    assert open(os.path.join(cli.work, tag + "_ref.sig")).read() == open(os.path.join(cli.work, tag + "_b200.sig")).read()   # the .sig files themselves


def test_sketch_of_fastq_and_invalid_bases(cli):
    "a FASTQ file; records with N and IUPAC codes (skipped k-mers, force = the CLI default)"
    reads = [("r1", "ACGTTGCAACGTTGCATGCATGCAAGCTNNACGTACGATCGATCGTACGATGCATGCA"),
             ("r2 second", "acgtacgtRYacgtagctagctagcatcgatcgatcgatgcatgcatgcatgcag")]
    with open(os.path.join(cli.work, "reads.fq"), "w") as fh:
        for name, seq in reads:
            fh.write("@%s\n%s\n+\n%s\n" % (name, seq, "I" * len(seq)))
    cli.together(["sketch", "dna", "-p", "k=11,scaled=1", "reads.fq", "-o", "fq_ref.sig"],
                 ["scripts", "b200sketch", "-p", "k=11,scaled=1", "reads.fq", "-o", "fq_b200.sig"])
    want, got = cli.loads("fq_ref.sig", "fq_b200.sig")
    assert len(want) > 100 and got == want


def test_compare_command_writes_the_same_matrix(cli):
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    cli.together(["compare", *sigs, "-k", "21", "-o", "ref.npy", "--csv", "ref_cmp.csv"],
                 ["scripts", "b200compare", *sigs, "-k", "21", "-o", "b200.npy", "--csv", "b200_cmp.csv"])
    w = cli.work
    a, b = np.load(os.path.join(w, "ref.npy")), np.load(os.path.join(w, "b200.npy"))
    assert a.shape == (12, 12) and np.array_equal(a, b) and 0 < a[a < 1].max() < 1
    assert open(os.path.join(w, "ref.npy.labels.txt")).read() == open(os.path.join(w, "b200.npy.labels.txt")).read()
    assert list(csv.reader(open(os.path.join(w, "ref_cmp.csv")))) == list(csv.reader(open(os.path.join(w, "b200_cmp.csv"))))


@pytest.mark.parametrize("flags", [["--containment"], ["--max-containment"], ["--avg-containment"], ["--estimate-ani"],
                                   ["--containment", "--estimate-ani"], ["--max-containment", "--estimate-ani"],
                                   ["--distance-matrix"], ["--scaled", "2000"]])
def test_compare_flags_write_the_same_matrix(cli, flags):
    "the other matrices of `sourmash compare`: containment forms, ANI, distances, a coarser --scaled"
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))[:6]
    tag = "cmp" + "".join(flags).replace("-", "")
    cli.together(["compare", *sigs, "-k", "21", "-o", tag + "_ref.npy", "--csv", tag + "_ref.csv", *flags],
                 ["scripts", "b200compare", *sigs, "-k", "21", "-o", tag + "_b200.npy", "--csv", tag + "_b200.csv", *flags])
    w = cli.work
    a, b = np.load(os.path.join(w, tag + "_ref.npy")), np.load(os.path.join(w, tag + "_b200.npy"))
    assert a.shape == (6, 6) and np.array_equal(a, b)
    assert open(os.path.join(w, tag + "_ref.csv")).read() == open(os.path.join(w, tag + "_b200.csv")).read()


@pytest.mark.parametrize("flags", [[], ["--ignore-abundance"], ["--containment"]])
def test_compare_of_abundance_sketches(cli, flags):
    "sketches with abundances: angular similarity unless --ignore-abundance; a flat sketch among them; containment ignores abundances"
    sigs = [os.path.join(DATA, "track_abund", f) for f in ("47.fa.sig", "63.fa.sig")] + [os.path.join(DATA, "2.fa.sig")]
    tag = "cmpab" + "".join(flags).replace("-", "")
    cli.together(["compare", *sigs, "-k", "31", "-o", tag + "_ref.npy", *flags],
                 ["scripts", "b200compare", *sigs, "-k", "31", "-o", tag + "_b200.npy", *flags])
    a, b = np.load(os.path.join(cli.work, tag + "_ref.npy")), np.load(os.path.join(cli.work, tag + "_b200.npy"))
    assert a.shape == (3, 3) and np.array_equal(a, b) and 0 < a[0, 1] < 1


def _same_file(cli, a, b, min_rows):
    ta, tb = open(os.path.join(cli.work, a)).read(), open(os.path.join(cli.work, b)).read()
    assert ta.count("\n") > min_rows and ta == tb


@pytest.mark.parametrize("flags", [[], ["--containment"], ["--max-containment"], ["--best-only"]])
def test_search_command_writes_the_same_csv(cli, flags):
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    tag = "search" + "".join(flags).replace("-", "")
    cli.together(["search", sigs[0], *sigs, "-k", "21", "--threshold", "0.01", "-o", tag + "_ref.csv", *flags],
                 ["scripts", "b200search", sigs[0], *sigs, "-k", "21", "--threshold", "0.01", "-o", tag + "_b200.csv", *flags])
    _same_file(cli, tag + "_ref.csv", tag + "_b200.csv", 1 if "--best-only" in flags else 5)


@pytest.mark.parametrize("threshold_bp", ["0", "50000"])
def test_gather_and_prefetch_commands_write_the_same_csv(cli, threshold_bp):
    query = os.path.join(DATA, "gather", "combined.sig")
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    for cmd in ("gather", "prefetch"):
        tag = "%s_%s" % (cmd, threshold_bp)
        cli.together([cmd, query, *sigs, "-k", "21", "--threshold-bp", threshold_bp, "-o", tag + "_ref.csv"],
                     ["scripts", "b200" + cmd, query, *sigs, "-k", "21", "--threshold-bp", threshold_bp, "-o", tag + "_b200.csv"])
        _same_file(cli, tag + "_ref.csv", tag + "_b200.csv", 5)


def test_gather_of_an_abundance_query_writes_the_same_csv(cli):
    "weighted columns (average_abund, f_unique_weighted, ...): a query with abundances against flat genomes"
    query = os.path.join(DATA, "track_abund", "47.fa.sig")
    dbs = [os.path.join(DATA, f) for f in ("47.fa.sig", "63.fa.sig", "2.fa.sig")]
    cli.together(["gather", query, *dbs, "-k", "31", "--threshold-bp", "0", "-o", "abund_ref.csv"],
                 ["scripts", "b200gather", query, *dbs, "-k", "31", "--threshold-bp", "0", "-o", "abund_b200.csv"])
    _same_file(cli, "abund_ref.csv", "abund_b200.csv", 1)


@pytest.mark.parametrize("flags", [[], ["--best-only"], ["--containment", "--best-only"]])
def test_search_of_one_multi_signature_database(cli, flags):
    "all subjects in ONE file (made with the reference's `sig cat`): --best-only ratchets its threshold inside a database"
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    if not os.path.exists(os.path.join(cli.work, "all12.sig")):
        cli("sig", "cat", *sigs[::-1], "-o", "all12.sig")              # reversed: the query's own sketch comes last
    tag = "one" + "".join(flags).replace("-", "")
    cli.together(["search", sigs[3], "all12.sig", "-k", "21", "--threshold", "0.01", "-o", tag + "_ref.csv", *flags],
                 ["scripts", "b200search", sigs[3], "all12.sig", "-k", "21", "--threshold", "0.01", "-o", tag + "_b200.csv", *flags])
    _same_file(cli, tag + "_ref.csv", tag + "_b200.csv", 1)
    if flags:
        rows = open(os.path.join(cli.work, tag + "_ref.csv")).read().count("\n") - 1
        assert 1 <= rows < 8                                            # fewer than without the ratchet


def test_a_zip_collection_as_the_database(cli):
    "the twelve genomes in one .zip (written by the reference's `sig cat`): every command, same files; a zip reports its absolute path"
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    query = os.path.join(DATA, "gather", "combined.sig")
    cli("sig", "cat", *sigs, "-o", "all12.zip")
    cli.together(["gather", query, "all12.zip", "-k", "21", "--threshold-bp", "0", "-o", "zip_gather_ref.csv"],
                 ["scripts", "b200gather", query, "all12.zip", "-k", "21", "--threshold-bp", "0", "-o", "zip_gather_b200.csv"],
                 ["prefetch", query, "all12.zip", "-k", "21", "--threshold-bp", "0", "-o", "zip_prefetch_ref.csv"],
                 ["scripts", "b200prefetch", query, "all12.zip", "-k", "21", "--threshold-bp", "0", "-o", "zip_prefetch_b200.csv"])
    cli.together(["search", sigs[0], "all12.zip", "-k", "21", "--threshold", "0.01", "-o", "zip_search_ref.csv"],
                 ["scripts", "b200search", sigs[0], "all12.zip", "-k", "21", "--threshold", "0.01", "-o", "zip_search_b200.csv"],
                 ["compare", "all12.zip", "-k", "21", "-o", "zip_ref.npy"],
                 ["scripts", "b200compare", "all12.zip", "-k", "21", "-o", "zip_b200.npy"])
    for name in ("gather", "prefetch", "search"):
        _same_file(cli, "zip_%s_ref.csv" % name, "zip_%s_b200.csv" % name, 5)
    assert np.array_equal(np.load(os.path.join(cli.work, "zip_ref.npy")), np.load(os.path.join(cli.work, "zip_b200.npy")))
    assert open(os.path.join(cli.work, "zip_ref.npy.labels.txt")).read() == open(os.path.join(cli.work, "zip_b200.npy.labels.txt")).read()


def test_a_directory_as_the_database_and_the_scaled_option(cli):
    """A directory (with a sub-directory) of .sig files is one database whose matches report the file they came from; --scaled
    downsamples the query first, and the reports then quote that sketch; protein sketches."""
    import shutil
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    query = os.path.join(DATA, "gather", "combined.sig")
    db = os.path.join(cli.work, "dbdir")
    os.makedirs(os.path.join(db, "sub"))
    for i, p in enumerate(sigs):
        shutil.copy(p, os.path.join(db, "sub") if i % 3 == 0 else db)
    cli.together(["gather", query, "dbdir", "-k", "21", "--threshold-bp", "0", "-o", "dir_gather_ref.csv"],
                 ["scripts", "b200gather", query, "dbdir", "-k", "21", "--threshold-bp", "0", "-o", "dir_gather_b200.csv"],
                 ["search", sigs[0], "dbdir", "--best-only", "-k", "21", "--threshold", "0.01", "-o", "dir_search_ref.csv"],
                 ["scripts", "b200search", sigs[0], "dbdir", "--best-only", "-k", "21", "--threshold", "0.01", "-o", "dir_search_b200.csv"])
    cli.together(["gather", query, *sigs, "-k", "21", "--threshold-bp", "0", "--scaled", "20000", "-o", "sc_gather_ref.csv"],
                 ["scripts", "b200gather", query, *sigs, "-k", "21", "--threshold-bp", "0", "--scaled", "20000", "-o", "sc_gather_b200.csv"],
                 ["compare", "dbdir", "-k", "21", "-o", "dir_ref.npy"],
                 ["scripts", "b200compare", "dbdir", "-k", "21", "-o", "dir_b200.npy"])
    _same_file(cli, "dir_gather_ref.csv", "dir_gather_b200.csv", 5)
    _same_file(cli, "dir_search_ref.csv", "dir_search_b200.csv", 1)
    _same_file(cli, "sc_gather_ref.csv", "sc_gather_b200.csv", 3)
    assert np.array_equal(np.load(os.path.join(cli.work, "dir_ref.npy")), np.load(os.path.join(cli.work, "dir_b200.npy")))
    prot = sorted(glob.glob(os.path.join(DATA, "prot", "protein", "*.sig")))
    cli.together(["search", prot[0], *prot, "--protein", "--threshold", "0.0", "-o", "prot_search_ref.csv"],
                 ["scripts", "b200search", prot[0], *prot, "--moltype", "protein", "--threshold", "0.0", "-o", "prot_search_b200.csv"],
                 ["gather", prot[0], *prot, "--protein", "--threshold-bp", "0", "-o", "prot_gather_ref.csv"],
                 ["scripts", "b200gather", prot[0], *prot, "--moltype", "protein", "--threshold-bp", "0", "-o", "prot_gather_b200.csv"])
    _same_file(cli, "prot_search_ref.csv", "prot_search_b200.csv", 1)
    _same_file(cli, "prot_gather_ref.csv", "prot_gather_b200.csv", 0)


def test_confidence_interval_columns(cli):
    "--estimate-ani-ci: the four (gather, prefetch) / two (containment search) extra columns"
    query = os.path.join(DATA, "gather", "combined.sig")
    sigs = sorted(glob.glob(os.path.join(DATA, "gather", "GCF*.sig")))
    pairs = []
    for cmd, first, flags in (("gather", query, ["--threshold-bp", "0"]), ("prefetch", query, ["--threshold-bp", "0"]),
                              ("search", sigs[0], ["--threshold", "0.01", "--containment"])):
        pairs += [[cmd, first, *sigs, "-k", "21", "--estimate-ani-ci", "-o", "ci_%s_ref.csv" % cmd, *flags],
                  ["scripts", "b200" + cmd, first, *sigs, "-k", "21", "--estimate-ani-ci", "-o", "ci_%s_b200.csv" % cmd, *flags]]
    cli.together(*pairs)
    for cmd in ("gather", "prefetch", "search"):
        _same_file(cli, "ci_%s_ref.csv" % cmd, "ci_%s_b200.csv" % cmd, 5)
        assert "ani_low" in open(os.path.join(cli.work, "ci_%s_ref.csv" % cmd)).readline()
