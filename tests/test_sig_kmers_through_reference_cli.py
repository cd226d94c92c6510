"""`sourmash scripts b200sigkmers` next to the reference's `sourmash sig kmers`, through the reference's command line.

The setting of tests/test_multigather_through_reference_cli.py: the reference's package runs over the emulated library
and finds this package's plugin commands in a dist-info written next to it; both commands run on the same inputs, and
every file they write (--save-kmers CSV, --save-sequences FASTA), their exit codes and the lines of their reports must be
equal.  The inputs follow the shapes of the reference's test_sig_kmers_* cases (short.fa, ecoli.faa; DNA, num, low
scaled, translate and protein sketches, an empty sequence file, an empty query) plus several files, FASTQ, gzip, abundance
signatures, several merged signatures, --from-file, -k, --check-sequence with and without --force, and the error paths.
What the reference does is stored in tests/golden/sig_kmers_cli_reference.json.gz; without the reference copy that build()
makes, `python -m sourmash_b200.sigkmers` is checked against the stored side, with it the live reference must do exactly
what is stored (SMB_PLUGIN_CLI_RECORD=1 rewrites the stored side)."""
import base64
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
STORED = os.path.join(GOLDEN, "sig_kmers_cli_reference.json.gz")
ENTRY = "b200sigkmers = sourmash_b200.sigkmers:Command_B200SigKmers\n"
STDERR = "<stderr>"
RC = "<rc>"


def report_lines(text):
    """The report of a run: every line as the terminal shows it (the text after the last carriage return), without the
    reference's banner, blank lines, the reference's per-file loading messages and the frames of a traceback (their
    paths differ)."""
    out = []
    for line in text.splitlines():
        line = line.split("\r")[-1].replace("\x1b[K", "").rstrip()
        if not line or line.startswith("==") or line.startswith("Traceback") or line.startswith("  "):
            continue
        if line.startswith("Loaded ") and " sigs from " in line or line.startswith("loaded ") and (
                " signatures from " in line or " signatures total" in line):
            continue
        out.append(line)
    return out


def _extra_inputs(d):
    "FASTA / FASTQ / gzip inputs with lower case and N, written the same way with and without the reference"
    import random
    rng = random.Random(5)
    with open(os.path.join(base.DATA if LIVE else d, "short.fa")) as fh:
        short = "".join(line.strip() for line in fh if not line.startswith(">"))
    def mutate(s, n):
        s = list(s)
        for _ in range(n):
            s[rng.randrange(len(s))] = rng.choice("ACGTacgt")
        return "".join(s)
    reads = [short[i:i + 150] for i in range(0, len(short) - 150, 37)]
    recs = [(("r%d read %d" % (i, i)), mutate(r, 3)) for i, r in enumerate(reads)]
    recs[3] = (recs[3][0], recs[3][1].lower())
    with_n = list(recs)
    with_n[5] = (with_n[5][0], with_n[5][1][:70] + "N" + with_n[5][1][71:])
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "reads1.fa"), "w") as fh:
        fh.write("".join(">%s\n%s\n" % r for r in recs[:20]))
    with gzip.GzipFile(os.path.join(d, "reads2.fq.gz"), "wb", mtime=0) as fh:
        fh.write("".join("@%s\n%s\n+\n%s\n" % (n, s, "I" * len(s)) for n, s in recs[20:]).encode())
    with open(os.path.join(d, "withn.fq"), "w") as fh:
        fh.write("".join("@%s\n%s\n+\n%s\n" % (n, s, "I" * len(s)) for n, s in with_n[:12]))
    with open(os.path.join(d, "tiny.fa"), "w") as fh:
        fh.write(">tiny\nACGTACGTAC\n")
    with open(os.path.join(d, "empty.fa"), "w") as fh:
        pass


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refsk"))
    site = os.path.join(tmp, "site")
    data = base.DATA
    stored = {}
    if LIVE:
        over_abi._stub_package(tmp, emul_lib.build())
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + ENTRY)
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

    def unplace(b):
        return b.replace(b"@WORK@", work.encode()).replace(b"@DATA@", data.encode())

    def key(args):
        return placeholders(json.dumps([str(a) for a in args]).encode()).decode()

    def run(*args, rc=0):
        "a reference command (stored outside LIVE) or the plugin command; returns (rc, report lines, written files)"
        args = [str(a) for a in args]
        if args[0] != "scripts" and not LIVE:
            assert key(args) in recorded, "no stored outputs of the reference for %s" % key(args)
            out = recorded[key(args)]
            files = {}
            for rel, text in out.items():
                if rel in (STDERR, RC):
                    continue
                files[rel] = unplace(base64.b64decode(text))
                path = os.path.join(work, rel)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                with open(path, "wb") as fh:
                    fh.write(files[rel])
            return out[RC], json.loads(unplace(out[STDERR].encode()).decode()), files
        if args[0] == "scripts" and not LIVE:
            cmd = [sys.executable, "-m", "sourmash_b200.sigkmers"] + args[2:]
        else:
            cmd = [sys.executable, "-m", "sourmash"] + args
        before = base._files(work)
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=work, timeout=900)
        assert r.returncode == rc, " ".join(args) + "\n" + r.stdout[-2000:] + r.stderr[-3000:]
        after = base._files(work)
        files = {}
        for rel in sorted(after):
            if before.get(rel) != after[rel]:
                with open(os.path.join(work, rel), "rb") as fh:
                    files[rel] = fh.read()
        lines = report_lines(r.stderr)
        if args[0] != "scripts":
            out = {rel: base64.b64encode(placeholders(b)).decode() for rel, b in files.items()}
            out[STDERR] = placeholders(json.dumps(lines).encode()).decode()
            out[RC] = r.returncode
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference did other than stored (%s)" % key(args)
        return r.returncode, lines, files

    def both(tag, *args, rc=0):
        "`sig kmers` and the plugin command with the same arguments; --save-* names get the side's tag"
        def side(name):
            return [a.replace("@OUT@", "%s_%s" % (tag, name)) for a in map(str, args)]
        want = run("sig", "kmers", *side("ref"), rc=rc)
        got = run("scripts", "b200sigkmers", *side("b200"), rc=rc)
        assert got[0] == want[0], (tag, got[0], want[0])
        assert got[1] == want[1], (tag, "\n".join(got[1]), "\n".join(want[1]))
        rename = {rel.replace(tag + "_ref", tag + "_b200"): b for rel, b in want[2].items()}
        assert sorted(got[2]) == sorted(rename), (tag, sorted(got[2]), sorted(rename))
        for rel in rename:
            assert got[2][rel] == rename[rel], (tag, rel)
        return want

    run.work, run.data, run.both = work, data, both
    if not LIVE:
        # the generated inputs were stored with the reference's side; put them in place
        for k, out in recorded.items():
            if k == key(["<inputs>"]):
                for rel, text in out.items():
                    path = os.path.join(work, rel)
                    os.makedirs(os.path.dirname(path), exist_ok=True)
                    with open(path, "wb") as fh:
                        fh.write(base64.b64decode(text))
    else:
        _extra_inputs(os.path.join(work, "in"))
        ins = {}
        for name in sorted(os.listdir(os.path.join(work, "in"))):
            with open(os.path.join(work, "in", name), "rb") as fh:
                ins[os.path.join("in", name)] = base64.b64encode(fh.read()).decode()
        recorded[key(["<inputs>"])] = ins
    yield run
    if LIVE and os.environ.get("SMB_PLUGIN_CLI_RECORD"):
        with gzip.GzipFile(STORED, "wb", mtime=0) as fh:
            fh.write(json.dumps(recorded, sort_keys=True, indent=0).encode())


def _sketch(sk, *args):
    "a query signature, made by the reference's `sourmash sketch` (its files come from the stored side without it)"
    sk("sketch", *args)


SAVE = ["--save-kmers", "@OUT@.csv", "--save-sequences", "@OUT@.fa"]


def test_dna_query_shapes(sk):
    "test_sig_kmers_1_dna / _more_in_query / _single_sig / _lowscaled / _num, and --save-kmers or --save-sequences alone"
    d = sk.data
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "scaled=1", "-o", "short.sig")
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "scaled=5", "-o", "short100.sig")
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "num=50", "-o", "shortnum.sig")
    _sketch(sk, "dna", os.path.join(d, "short.fa"), os.path.join(d, "short2.fa"), "-p", "scaled=1", "-o", "more.sig")
    sk.both("dna", "--sig", "short.sig", "--seq", os.path.join(d, "short.fa"), *SAVE)
    sk.both("more", "--sig", "more.sig", "--seq", os.path.join(d, "short.fa"), *SAVE)
    sk.both("low", "--sig", "short100.sig", "--seq", os.path.join(d, "short.fa"), os.path.join(d, "short2.fa"), *SAVE)
    sk.both("num", "--sig", "shortnum.sig", "--seq", os.path.join(d, "short.fa"), *SAVE)
    sk.both("kmersonly", "--sig", "short.sig", "--seq", os.path.join(d, "short.fa"), "--save-kmers", "@OUT@.csv")
    sk.both("nosave", "--sig", "short.sig", "--seq", os.path.join(d, "short.fa"))


@pytest.mark.parametrize("mol", ["protein", "dayhoff", "hp"])
def test_protein_family_shapes(sk, mol):
    "test_sig_kmers_1_dna_translate_* and test_sig_kmers_2_*: no moltype flag, residues and translated DNA"
    d = sk.data
    _sketch(sk, "protein", os.path.join(d, "ecoli.faa"), "-p", "%s,k=7,scaled=5" % mol, "-o", "ecoli_%s.sig" % mol)
    _sketch(sk, "translate", os.path.join(d, "short.fa"), "-p", "%s,k=7,scaled=5" % mol, "-o", "tr_%s.sig" % mol)
    sk.both("prot_" + mol, "--sig", "ecoli_%s.sig" % mol, "--seq", os.path.join(d, "ecoli.faa"), *SAVE)
    sk.both("tr_" + mol, "--sig", "tr_%s.sig" % mol, "--seq", os.path.join(d, "short.fa"), "--translate", *SAVE)


def test_reads_files_abundance_merge_and_selection(sk):
    "several files (FASTA + FASTQ.gz), an abundance signature, two merged signatures, --from-file and -k"
    d = sk.data
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "k=21,k=31,scaled=5,abund", "-o", "ab.sig")
    _sketch(sk, "dna", os.path.join(d, "short2.fa"), "-p", "k=31,scaled=5", "-o", "s2.sig")
    reads = ["in/reads1.fa", "in/reads2.fq.gz"]
    sk.both("ab", "--sig", "ab.sig", "-k", "31", "--seq", *reads, *SAVE)
    sk.both("merged", "--sig", "ab.sig", "s2.sig", "-k", "31", "--seq", *reads, *SAVE)
    with open(os.path.join(sk.work, "list.txt"), "w") as fh:
        fh.write("ab.sig\ns2.sig\n")
    sk.both("fromfile", "--from-file", "list.txt", "-k", "31", "--seq", *reads, *SAVE)


def test_invalid_dna(sk):
    "--check-sequence without and with --force, and --save-kmers meeting an N in a matching record"
    _sketch(sk, "dna", os.path.join(sk.data, "short.fa"), "-p", "scaled=2", "-o", "s10.sig")
    sk.both("check", "--sig", "s10.sig", "--seq", "in/withn.fq", "--check-sequence", *SAVE, rc=255)
    sk.both("checkf", "--sig", "s10.sig", "--seq", "in/withn.fq", "--check-sequence", "-f", *SAVE)
    sk.both("nocheck", "--sig", "s10.sig", "--seq", "in/withn.fq", "--save-sequences", "@OUT@.fa")
    sk.both("nocheckkmers", "--sig", "s10.sig", "--seq", "in/withn.fq", *SAVE, rc=1)


def test_error_paths(sk):
    "empty sequence file, empty query, no signatures, --translate with a DNA sketch, incompatible signatures"
    d = sk.data
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "scaled=1", "-o", "e_short.sig")
    _sketch(sk, "dna", "in/tiny.fa", "-o", "tiny.sig")
    _sketch(sk, "dna", os.path.join(d, "short.fa"), "-p", "k=31,scaled=500", "-o", "s500.sig")
    sk.both("emptyseq", "--sig", "e_short.sig", "--seq", "in/empty.fa", rc=255)
    sk.both("emptysig", "--sig", "tiny.sig", "--seq", os.path.join(d, "short.fa"), rc=255)
    sk.both("nosig", "--sig", "e_short.sig", "-k", "21", "--seq", os.path.join(d, "short.fa"), rc=255)
    sk.both("translatedna", "--sig", "e_short.sig", "--seq", os.path.join(d, "short.fa"), "--translate", rc=255)
    sk.both("incompatible", "--sig", "e_short.sig", "s500.sig", "--seq", os.path.join(d, "short.fa"), rc=255)
