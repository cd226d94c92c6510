"""`sourmash scripts b200sigmerge | b200sigintersect | b200sigsubtract` next to the reference's `sourmash sig merge |
intersect | subtract`, through the reference's command line.

The setting of tests/test_sig_kmers_through_reference_cli.py: the reference's package runs over the emulated library and
finds this package's commands in a dist-info written next to it; both commands run on the same inputs, and the
signature files they write, what they write to stdout (-o -), their exit codes and the lines of their reports must be
equal.  Progress lines ("...loading from", "...N sigs so far") are left out of the comparison: they depend on the
terminal width and the loading interval, not on the result.

Inputs: 47/63 (flat and track_abund), the 12 gather genomes, protein sketches, a .zip collection, num sketches, a
directory and --from-file; the options --flatten, -A, --set-name / --name, -k and the moltype flags; the error paths of
k-size / scaled / num / abundance mismatches, subtract of abundance sketches, -A with a flat signature, and no signatures
at all.  The reference's side is stored in tests/golden/sig_setops_cli_reference.json.gz as the SHA-256 of every file it
wrote, its report lines and its exit code; without the reference copy that build() makes, `python -m
sourmash_b200.sigsetops` is checked against the stored side, with it the live reference must do exactly what is stored
(SMB_PLUGIN_CLI_RECORD=1 rewrites the stored side)."""
import base64
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_plugin_through_reference_cli as base  # noqa: E402
from test_sig_kmers_through_reference_cli import report_lines as _kmers_report_lines  # noqa: E402

over_abi = base.over_abi
HERE, ROOT, GOLDEN, LIVE = base.HERE, base.ROOT, base.GOLDEN, base.LIVE
STORED = os.path.join(GOLDEN, "sig_setops_cli_reference.json.gz")
ENTRY = ("b200sigmerge = sourmash_b200.sigsetops:Command_B200SigMerge\n"
         "b200sigintersect = sourmash_b200.sigsetops:Command_B200SigIntersect\n"
         "b200sigsubtract = sourmash_b200.sigsetops:Command_B200SigSubtract\n")
STDERR, STDOUT, RC, FILES = "<stderr>", "<stdout>", "<rc>", "<files>"


def report_lines(text):
    return [line for line in _kmers_report_lines(text) if not line.startswith("...") and not line.startswith("<<<")]


def _digest(b):
    return hashlib.sha256(b).hexdigest()


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    tmp = str(tmp_path_factory.mktemp("refsetops"))
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
            fh.write("[sourmash.cli_script]\n" + ENTRY)
        if os.path.exists(STORED) and not os.environ.get("SMB_PLUGIN_CLI_RECORD"):
            with gzip.open(STORED, "rt") as fh:
                stored = json.load(fh)
    else:
        emul_lib.build()
        os.makedirs(site)
        data = os.path.join(tmp, "test-data")
        base._stored_inputs(data)
        os.makedirs(os.path.join(data, "prot"), exist_ok=True)
        shutil.copy(os.path.join(GOLDEN, "refdata", "prot", "protein.zip"), os.path.join(data, "prot", "protein.zip"))
        with gzip.open(STORED, "rt") as fh:
            recorded = json.load(fh)
    with open(os.path.join(site, "sitecustomize.py"), "w") as fh:
        fh.write("import sys\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport emulated_boot\nemulated_boot.install()\n"
                 % (os.path.join(HERE, "host_emul"), ROOT))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, os.path.join(tmp, "reftests")]), PYTHONDONTWRITEBYTECODE="1")
    work = os.path.join(tmp, "work")
    os.makedirs(os.path.join(work, "dir", "sub"))
    for i, name in enumerate(sorted(n for n in os.listdir(os.path.join(data, "gather")) if n.startswith("GCF"))[:5]):
        shutil.copy(os.path.join(data, "gather", name), os.path.join(work, "dir", "sub" if i % 2 else "", name))
    with open(os.path.join(work, "list.txt"), "w") as fh:
        fh.write("%s\n%s\n" % (os.path.join(data, "47.fa.sig"), os.path.join(data, "63.fa.sig")))

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
            cmd = [sys.executable, "-m", "sourmash_b200.sigsetops", args[1][len("b200sig"):]] + args[2:]
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
            if args[0] == "sketch":
                out[FILES] = {}
                for rel in files:
                    if rel != STDOUT:
                        with open(os.path.join(work, rel), "rb") as fh:
                            out[FILES][rel] = base64.b64encode(placeholders(fh.read())).decode()
            recorded[key(args)] = out
            if key(args) in stored:
                assert stored[key(args)] == out, "the reference did other than stored (%s)" % key(args)
        return r.returncode, lines, files

    def both(op, tag, *args, rc=0):
        "`sig <op>` and the plugin command with the same arguments; @OUT@ names get the side's tag"
        def side(name):
            return [a.replace("@OUT@", "%s_%s" % (tag, name)) for a in map(str, args)]
        want = run("sig", op, *side("ref"), rc=rc)
        got = run("scripts", "b200sig" + op, *side("b200"), rc=rc)
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


def _gather(sk):
    d = os.path.join(sk.data, "gather")
    return [os.path.join(d, n) for n in sorted(os.listdir(d)) if n.startswith("GCF")]


def test_merge(sk):
    "47 + 63, abundance sketches, --flatten, the 12 gather genomes, a .zip, a directory, --from-file, -k, --name, stdout"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    ab47, ab63 = os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "track_abund", "63.fa.sig")
    sk.both("merge", "flat", sig47, sig63, "-o", "@OUT@.sig")
    sk.both("merge", "stdout", sig47, sig63, "--set-name", "both")
    sk.both("merge", "abund", ab47, ab63, ab47, "-o", "@OUT@.sig.gz", "--name", "twice")
    sk.both("merge", "flatten", ab47, sig63, "--flatten", "-o", "@OUT@.sig")
    sk.both("merge", "gather", *_gather(sk), "-k", "31", "--dna", "-o", "@OUT@.sig")
    sk.both("merge", "zip", os.path.join(d, "prot", "protein.zip"), "--protein", "-o", "@OUT@.sig")
    sk.both("merge", "dir", "dir", "-k", "31", "-o", "@OUT@.sig")
    sk.both("merge", "fromfile", "--from-file", "list.txt", "-k", "31", "-o", "@OUT@.sig")


def test_intersect_and_subtract(sk):
    "intersect and subtract of flat, protein and directory inputs, -A, --flatten and --set-name"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    ab47, ab63 = os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "track_abund", "63.fa.sig")
    prot = [os.path.join(d, "prot", "protein", n) for n in sorted(os.listdir(os.path.join(d, "prot", "protein")))]
    sk.both("intersect", "isect", sig47, sig63, "-o", "@OUT@.sig")
    sk.both("intersect", "isectab", ab47, ab63, "-A", ab47, "--set-name", "common", "-o", "@OUT@.sig")
    sk.both("intersect", "isectprot", *prot, "--protein", "-o", "@OUT@.sig")
    sk.both("intersect", "isectdir", "dir", *_gather(sk)[:3], "-k", "31", "-o", "@OUT@.sig")
    sk.both("intersect", "isectfrom", "--from-file", "list.txt", "-o", "@OUT@.sig")
    sk.both("intersect", "isectout", sig47, sig63)
    sk.both("subtract", "sub", sig47, sig63, "-o", "@OUT@.sig")
    sk.both("subtract", "subflat", ab47, ab63, "--flatten", "-o", "@OUT@.sig", "--set-name", "rest")
    sk.both("subtract", "subA", ab47, sig63, "-A", ab47, "-o", "@OUT@.sig")
    sk.both("subtract", "submany", _gather(sk)[0], *_gather(sk)[1:], "-k", "31", "-o", "@OUT@.sig.gz")
    sk.both("subtract", "subprot", prot[0], os.path.join(d, "prot", "protein.zip"), "--protein", "-o", "@OUT@.sig")


def test_num_sketches(sk):
    "num sketches of different num: merge keeps the first sketch's num; intersect and subtract take them"
    d = sk.data
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "num=500", "-o", "n500a.sig")
    sk("sketch", "dna", os.path.join(d, "short2.fa"), "-p", "num=500", "-o", "n500b.sig")
    sk("sketch", "dna", os.path.join(d, "short3.fa"), "-p", "num=200", "-o", "n200.sig")
    sk.both("merge", "num", "n500a.sig", "n500b.sig", "n200.sig", "-o", "@OUT@.sig")
    sk.both("merge", "num200", "n200.sig", "n500a.sig", "-o", "@OUT@.sig")
    sk.both("intersect", "numisect", "n500a.sig", "n500b.sig", "-o", "@OUT@.sig")
    sk.both("subtract", "numsub", "n500a.sig", "n500b.sig", "n200.sig", "-o", "@OUT@.sig")


def test_error_paths(sk):
    "k-size, scaled, num and abundance mismatches, subtract of abundance sketches, -A with a flat signature, nothing"
    d = sk.data
    sig47, sig63 = os.path.join(d, "47.fa.sig"), os.path.join(d, "63.fa.sig")
    ab47, ab63 = os.path.join(d, "track_abund", "47.fa.sig"), os.path.join(d, "track_abund", "63.fa.sig")
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "k=21,scaled=10", "-o", "k21.sig")
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "k=31,scaled=10", "-o", "k31.sig")
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "k=31,scaled=20", "-o", "s20.sig")
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "k=31,num=100", "-o", "n100.sig")
    sk("sketch", "dna", os.path.join(d, "short.fa"), "-p", "k=31,scaled=10,abund", "-o", "ab31.sig")
    for op in ("merge", "intersect"):
        sk.both(op, op + "_k", "k31.sig", "k21.sig", "-o", "@OUT@.sig", rc=255)
        sk.both(op, op + "_scaled", "k31.sig", "s20.sig", "-o", "@OUT@.sig", rc=255)
        sk.both(op, op + "_num", "k31.sig", "n100.sig", "-o", "@OUT@.sig", rc=255)
        sk.both(op, op + "_none", "k31.sig", "-k", "51", "-o", "@OUT@.sig", rc=255)
        sk.both(op, op + "_empty", "-o", "@OUT@.sig", rc=255)
    sk.both("merge", "merge_abund", sig47, ab63, "-o", "@OUT@.sig", rc=255)
    sk.both("merge", "merge_abund2", "k31.sig", "ab31.sig", "-o", "@OUT@.sig", rc=255)
    sk.both("intersect", "isect_flatA", sig47, sig63, "-A", sig47, "-o", "@OUT@.sig", rc=255)
    sk.both("subtract", "sub_abund", ab47, sig63, "-o", "@OUT@.sig", rc=1)
    sk.both("subtract", "sub_abund2", sig47, ab63, "-o", "@OUT@.sig", rc=1)
    sk.both("subtract", "sub_k", "k31.sig", "k21.sig", "-o", "@OUT@.sig", rc=255)
    sk.both("subtract", "sub_scaled", "k31.sig", "s20.sig", "-o", "@OUT@.sig", rc=255)
    sk.both("subtract", "sub_none", "k31.sig", "k21.sig", "-k", "31", "-o", "@OUT@.sig", rc=255)
    sk.both("subtract", "sub_flatA", sig47, sig63, "-A", sig63, "-o", "@OUT@.sig", rc=255)
