"""Randomised differential test: the reference's Python (its per-pair loops over this library's ABI) against this package's
batched functions, on the same random signature lists, in one process.

Both packages are importable side by side (`sourmash` = the reference loaded in place, as in
test_reference_python_over_abi.py; `sourmash_b200` = this package), both bound to the emulated library.  For every random
list -- equal or mixed scaled, flat and abundance sketches, empty sketches, num sketches -- the matrices of
compare_all_pairs / compare_serial_containment / _max_containment / _avg_containment (with and without ANI) must be equal
bit for bit, and LinearIndex.search / search_abund / prefetch and a gather loop must return the same matches with the same
scores.  Then random FASTA files are sketched both ways (every molecule type), and random query / database sets go through
the reference's `gather`, `prefetch` and `search` commands and the plugin's: the CSV files must be byte-identical (query at a
finer, equal or coarser scaled than the databases; abundance queries with and without --ignore-abundance; thresholds).

The reference's side of every comparison is stored, as a digest of its outcome, in tests/golden/differential_seed<N>.json, so
the test runs without the reference: it recomputes this package's side and compares it, comparison by comparison, with the
stored digests.  With the reference copy that build() makes (oracle/reference.py) it runs the reference's side live as well (and checks that
it still gives the stored digests);

    SMB_REFERENCE=<checkout> python tests/test_differential_vs_reference_python.py <seed>

rewrites the stored file of a seed."""
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_reference_python_over_abi as over_abi  # noqa: E402

REF = over_abi.REF
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

GOLDEN = os.path.join(HERE, "golden")

TRIALS = r'''
import hashlib
import json
import sys
import warnings
import numpy as np
import sourmash_b200 as smb
import sourmash_b200.compare as our_compare
import sourmash_b200.index as our_index
from sourmash_b200.plugin import main as plugin_main

seed, n_trials, golden_path, LIVE = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4] == "live"
if LIVE:                                                            # the reference's side is computed, not read back
    import sourmash as ref
    import sourmash.compare as ref_compare
    import sourmash.index as ref_index
    from sourmash.__main__ import main as sourmash_main
else:
    ref = ref_compare = ref_index = None
    with open(golden_path) as fh:
        STORED = json.load(fh)
    assert STORED["seed"] == seed and STORED["n_trials"] == n_trials, (STORED["seed"], STORED["n_trials"])
RECORDS = []                                                        # [what, digest of the reference's outcome] in order
rng = np.random.default_rng(seed)
stats = {"compare": 0, "containment": 0, "ani": 0, "search": 0, "prefetch": 0, "gather": 0, "errors": 0}   # comparisons made


def canonical(v):
    "a JSON-able form in which two outcomes are equal exactly when same() below accepts them"
    if isinstance(v, np.ndarray):
        a = np.asarray(v, dtype=np.float64) + 0.0                  # -0.0 == 0.0
        a = np.where(np.isnan(a), np.nan, a)                        # one NaN
        return ["nd", list(a.shape), hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()]
    if isinstance(v, (bool, np.bool_)):
        return ["b", bool(v)]
    if isinstance(v, (int, np.integer)):
        return ["i", str(int(v))]
    if isinstance(v, (float, np.floating)):
        f = float(v)
        return ["i", str(int(f))] if f.is_integer() and abs(f) < 2**63 else ["f", f.hex()]
    if isinstance(v, (list, tuple)):
        return [canonical(x) for x in v]
    if isinstance(v, dict):
        return ["d", sorted([canonical(k), canonical(x)] for k, x in v.items())]
    if v is None or isinstance(v, str):
        return v
    raise TypeError("no canonical form for %r" % type(v))


def digest(o):
    key = ["raises", o[1]] if o[0] == "raises" else ["ok", canonical(o[1])]
    return hashlib.sha256(json.dumps(key).encode()).hexdigest()[:16]


def stored(what):
    "the stored digest of the next comparison, which must be this one"
    i = len(RECORDS)
    want = STORED["records"][i] if i < len(STORED["records"]) else None
    if not want or want[0] != what:
        raise AssertionError("comparison %d is %r here, %r in %s" % (i, what, want and want[0], golden_path))
    return want[1]


def make(pkg, spec):
    mh = pkg.MinHash(n=spec["num"], ksize=spec["ksize"], scaled=spec["scaled"], track_abundance=spec["abund"])
    if spec["abund"]:
        mh.set_abundances(dict(zip(spec["hashes"], spec["abunds"])))
    else:
        mh.add_many(spec["hashes"])
    return pkg.SourmashSignature(mh, name=spec["name"], filename=spec["name"] + ".fa").to_frozen()   # what loading a file gives


def random_list(rng):
    n = int(rng.integers(2, 8))
    kind = rng.choice(["scaled", "scaled", "mixed_scaled", "num", "abund"])
    pool = rng.integers(1, 2**64 - 1, size=int(rng.integers(20, 400)), dtype=np.uint64)
    specs = []
    for i in range(n):
        scaled, num = 1000, 0
        if kind == "mixed_scaled":
            scaled = int(rng.choice([500, 1000, 2000]))
        if kind == "num":
            scaled, num = 0, 50
        hashes = rng.choice(pool, size=int(rng.integers(0, len(pool))), replace=False)
        if scaled:
            hashes = hashes[hashes <= np.uint64((2**64 - 1) // scaled)] if rng.random() < 0.5 else hashes % np.uint64((2**64) // scaled)
        hashes = np.unique(hashes)
        if rng.random() < 0.08:
            hashes = hashes[:0]                                     # an empty sketch
        abund = kind == "abund" and rng.random() < 0.8
        specs.append(dict(num=num, ksize=21, scaled=scaled, abund=bool(abund), name="s%d" % i,
                          hashes=[int(h) for h in hashes], abunds=[int(a) for a in rng.integers(1, 30, size=len(hashes))]))
    return kind, specs


def outcome(fn):
    "('ok', value) or ('raises', exception type name, message)"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return ("ok", fn())
        except Exception as exc:                                    # noqa: BLE001 -- the comparison IS about what is raised
            return ("raises", type(exc).__name__, str(exc))


def check(what, ours, theirs, specs):
    "ours / theirs: zero-argument functions; theirs (the reference) runs only when it is present"
    b = outcome(ours)
    if LIVE:
        a = outcome(theirs)
        same(a, b, what, specs)
        RECORDS.append([what, digest(a)])
        return
    if digest(b) != stored(what):
        raise AssertionError("%s differs from the reference's stored outcome\nhere %r\n%r" % (what, b[:3], specs))
    RECORDS.append([what, digest(b)])
    if b[0] == "raises":
        stats["errors"] += 1


def same(a, b, what, specs):
    if a[0] != b[0]:
        raise AssertionError("%s: reference %r, here %r\n%r" % (what, a[:3], b[:3], specs))
    if a[0] == "raises":
        if a[1] != b[1]:
            raise AssertionError("%s raises %s(%s) in the reference, %s(%s) here" % (what, a[1], a[2], b[1], b[2]))
        stats["errors"] += 1
        return
    if isinstance(a[1], np.ndarray):
        if not (a[1].shape == b[1].shape and np.array_equal(a[1], b[1], equal_nan=True)):
            raise AssertionError("%s differs\nreference\n%r\nhere\n%r\n%r" % (what, a[1], b[1], specs))
    elif a[1] != b[1]:
        raise AssertionError("%s differs\nreference %r\nhere      %r\n%r" % (what, a[1], b[1], specs))


for trial in range(n_trials):
    kind, specs = random_list(rng)
    R, O = [make(ref, s) for s in specs] if LIVE else None, [make(smb, s) for s in specs]
    down = kind == "mixed_scaled"
    for ignore in (True, False):
        check("compare_all_pairs(ignore_abundance=%s) on %s" % (ignore, kind),
              lambda: our_compare.compare_all_pairs(O, ignore, downsample=down, n_jobs=None),
              lambda: ref_compare.compare_all_pairs(R, ignore, downsample=down, n_jobs=None), specs)
        stats["compare"] += 1
    for name in ("compare_serial_containment", "compare_serial_max_containment", "compare_serial_avg_containment"):
        check("%s on %s" % (name, kind), lambda: getattr(our_compare, name)(O, downsample=down),
              lambda: getattr(ref_compare, name)(R, downsample=down), specs)
        stats["containment"] += 1
        if kind in ("scaled", "mixed_scaled"):
            check("%s(return_ani) on %s" % (name, kind), lambda: getattr(our_compare, name)(O, downsample=down, return_ani=True),
                  lambda: getattr(ref_compare, name)(R, downsample=down, return_ani=True), specs)
            stats["ani"] += 1
    if kind == "mixed_scaled":             # without the flag the avg ANI form downsamples anyway (FracMinHashComparison)
        for name in ("compare_serial_avg_containment",):
            check("%s(return_ani, no downsample) on %s" % (name, kind), lambda: getattr(our_compare, name)(O, return_ani=True),
                  lambda: getattr(ref_compare, name)(R, return_ani=True), specs)
            stats["ani"] += 1
    if kind in ("scaled", "mixed_scaled"):
        check("compare_all_pairs(return_ani) on %s" % kind,
              lambda: our_compare.compare_all_pairs(O, True, downsample=down, return_ani=True, n_jobs=None),
              lambda: ref_compare.compare_all_pairs(R, True, downsample=down, return_ani=True, n_jobs=None), specs)
        stats["ani"] += 1
    # one-vs-many: the first signature against an index of the rest
    if kind in ("scaled", "mixed_scaled") and len(specs[0]["hashes"]):
        ri, oi = ref_index.LinearIndex(R[1:], "db") if LIVE else None, our_index.LinearIndex(O[1:], "db")

        def names(results):
            return [(float(r.score), r.signature.name, r.location) for r in results]
        for kw in (dict(threshold=0.0), dict(threshold=0.05, do_containment=True), dict(threshold=0.05, do_max_containment=True),
                   dict(threshold=0.0, best_only=True)):
            check("LinearIndex.search(%r) on %s" % (kw, kind), lambda: names(oi.search(O[0], **kw)),
                  lambda: names(ri.search(R[0], **kw)), specs)
            stats["search"] += 1
        check("LinearIndex.prefetch on %s" % kind, lambda: names(oi.prefetch(O[0], threshold_bp=0)),
              lambda: names(ri.prefetch(R[0], threshold_bp=0)), specs)
        stats["prefetch"] += 1

        def best(index, query, tbp):
            r = index.best_containment(query, threshold_bp=tbp)
            return None if not r else (float(r.score), r.signature.name, r.location)
        for tbp in (0, 5000):
            check("LinearIndex.best_containment(threshold_bp=%d) on %s" % (tbp, kind), lambda: best(oi, O[0], tbp),
                  lambda: best(ri, R[0], tbp), specs)
            stats["search"] += 1

        def gather_rounds(index, query):
            counter = index.counter_gather(query, 0)
            cur, out = query.minhash.flatten().to_mutable(), []
            while True:
                res = counter.peek(cur)
                if not res:
                    return out
                sr, intersect = res
                out.append((float(sr.score), sr.signature.name, len(intersect)))
                counter.consume(intersect)
                cur = cur.downsample(scaled=counter.scaled).to_mutable() if counter.scaled > cur.scaled else cur
                cur.remove_many(intersect.downsample(scaled=cur.scaled) if intersect.scaled < cur.scaled else intersect)
        check("gather rounds on %s" % kind, lambda: gather_rounds(oi, O[0]), lambda: gather_rounds(ri, R[0]), specs)
        stats["gather"] += 1
    if kind == "abund":
        ri, oi = ref_index.LinearIndex(R[1:], "db") if LIVE else None, our_index.LinearIndex(O[1:], "db")
        check("LinearIndex.search_abund", lambda: [(float(r.score), r.signature.name) for r in oi.search_abund(O[0], threshold=0.0)],
              lambda: [(float(r.score), r.signature.name) for r in ri.search_abund(R[0], threshold=0.0)], specs)
        stats["search"] += 1
# ---- sketching: the reference's record-by-record add_sequence / add_protein against this package's batched file sketcher
import gzip
from sourmash_b200.sketch import sketch_fasta_files
stats["sketch"] = 0
for trial in range(max(4, n_trials // 5)):
    mode = rng.choice(["dna", "dna", "dna_abund_num", "protein", "dayhoff", "hp", "translate"])
    n_files = int(rng.integers(1, 4))
    paths, records = [], []
    for f in range(n_files):
        recs = []
        for r in range(int(rng.integers(0, 5))):
            L = int(rng.choice([0, 5, 20, 21, 60, 300, 2500]))
            if mode in ("protein", "dayhoff", "hp"):
                seq = "".join(rng.choice(list("ACDEFGHIKLMNPQRSTVWYX*"), size=L))
            else:
                seq = "".join(rng.choice(list("ACGT"), size=L))
                if L and rng.random() < 0.5:                       # invalid bases, lower case
                    pos = rng.integers(0, L, size=max(1, L // 40))
                    seq = "".join(("N" if i in set(pos.tolist()) else c) for i, c in enumerate(seq))
                if rng.random() < 0.3:
                    seq = seq.lower()
            recs.append(("f%dr%d some description" % (f, r), seq))
        path = "sk%d_%d.fa%s" % (trial, f, ".gz" if rng.random() < 0.3 else "")
        text = "".join(">%s\n%s\n" % (n, "\n".join(sq[i:i + 70] for i in range(0, len(sq), 70))) for n, sq in recs)
        (gzip.open if path.endswith(".gz") else open)(path, "wt").write(text)
        paths.append(path); records.append(recs)
    if mode in ("dna", "dna_abund_num"):
        ksizes, kw = [21, 31, 51], dict(is_protein=False)
    else:
        ksizes, kw = [7, 10], dict(is_protein=mode in ("protein", "translate"), dayhoff=mode == "dayhoff", hp=mode == "hp")
    scaled, num, abund = (0, 30, True) if mode == "dna_abund_num" else (int(rng.choice([1, 10, 100])), 0, bool(rng.random() < 0.3))
    ours = sketch_fasta_files(paths, ksizes=ksizes, scaled=scaled, num=num, track_abundance=abund,
                              moltype={"dna": "dna", "dna_abund_num": "dna", "translate": "protein"}.get(mode, mode),
                              input_is_protein=mode in ("protein", "dayhoff", "hp"))
    got = sorted((ss.filename, mh.ksize, sorted(mh.hashes.items())) for ss in ours for mh in ss.sketches())   # one signature per file

    def want():
        out = []
        for path, recs in zip(paths, records):
            if not recs:
                continue                                            # no sequences found: no signature
            for k in ksizes:
                mh = ref.MinHash(n=num, ksize=k, scaled=scaled, track_abundance=abund, **kw)
                for _name, seq in recs:
                    if mode in ("protein", "dayhoff", "hp"):
                        mh.add_protein(seq)
                    else:
                        mh.add_sequence(seq, force=True)            # translate: is_protein sketch fed DNA = six frames
                out.append((path, k, sorted(mh.hashes.items())))
        return sorted(out)
    check("sketch (%s, scaled=%s num=%s abund=%s)" % (mode, scaled, num, abund), lambda: got, want, records)
    stats["sketch"] += 1
# ---- reports: the reference's gather / prefetch / search commands against the plugin commands, CSV files byte for byte
import contextlib, io
stats["reports"] = 0


def cli(main, *args):
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        try:
            main([str(a) for a in args])
        except SystemExit as exc:
            return exc.code or 0
        except Exception as exc:                                    # noqa: BLE001
            return type(exc).__name__
    return 0


# the input .sig files: written by the reference when it is present, else by this package (same layout, same bytes)
WRITER = ref if LIVE else smb


def save(ss, path):
    if LIVE:
        with open(path, "w") as fp:
            ref.save_signatures([ss], fp)
    else:
        with open(path, "wb") as fp:
            smb.save_signatures_to_json([ss], fp)


def read(path):
    try:
        return open(path).read()
    except FileNotFoundError:
        return None


for trial in range(max(3, n_trials // 8)):
    top = (2**64 - 1) // 1000
    pool = np.unique(rng.integers(1, top, size=3000, dtype=np.uint64))
    n_subj = int(rng.integers(2, 9))
    # one scaled per database set, finer / equal / coarser than the query's 1000 (databases of DIFFERENT scaled values are
    # the one case the plugin does not follow: the reference lowers the resolution as coarser matches get picked, DESIGN 8)
    db_scaled = int(rng.choice([500, 1000, 2000]))
    subjects, files = [], []
    for i in range(n_subj):
        own = rng.choice(pool, size=int(rng.integers(30, 600)), replace=False)
        mh = WRITER.MinHash(n=0, ksize=31, scaled=db_scaled)
        mh.add_many([int(h) for h in own])
        ss = WRITER.SourmashSignature(mh, name="subject %d" % i, filename="subj%d.fa" % i)
        subjects.append(ss)
        path = "rep%d_s%d.sig" % (trial, i)
        save(ss, path)
        files.append(path)
    qh = {}
    for ss in subjects[: max(1, n_subj - 1)]:                      # the query: parts of most subjects + hashes of its own
        for h in list(ss.minhash.hashes)[:: int(rng.integers(1, 4))]:
            qh[h] = int(rng.integers(1, 40))
    for h in rng.integers(1, top, size=int(rng.integers(0, 200)), dtype=np.uint64):
        qh[int(h)] = int(rng.integers(1, 5))
    abund = bool(rng.random() < 0.6)
    qmh = WRITER.MinHash(n=0, ksize=31, scaled=1000, track_abundance=abund)
    if abund:
        qmh.set_abundances(qh)
    else:
        qmh.add_many(list(qh))
    qpath = "rep%d_query.sig" % trial
    save(WRITER.SourmashSignature(qmh, name="the query", filename="query.fa"), qpath)
    tbp = int(rng.choice([0, 20000, 100000]))
    runs = [("gather", ["--threshold-bp", tbp] + (["--ignore-abundance"] if abund and rng.random() < 0.4 else [])),
            ("prefetch", ["--threshold-bp", tbp]),
            ("search", ["--threshold", "0.02"] + ([[], ["--containment"], ["--max-containment"]][int(rng.integers(0, 3))])
             + (["--ignore-abundance"] if abund and rng.random() < 0.6 else []))]
    for cmd, flags in runs:
        what = "%s %r (abund query: %s, %d subjects, db scaled %d)" % (cmd, flags, abund, n_subj, db_scaled)
        a, b = "rep%d_%s_ref.csv" % (trial, cmd), "rep%d_%s_b200.csv" % (trial, cmd)
        rb = cli(plugin_main, "b200" + cmd, qpath, *files, "-o", b, *flags)
        tb = read(b)
        if not LIVE:
            want = stored(what)
            if want != "skipped" and digest(("ok", [rb == 0, tb])) != want:
                raise AssertionError("%s: exit %r, the CSV or the exit status differs from the reference's stored outcome\n%s"
                                     % (what, rb, (tb or "")[:2000]))
            RECORDS.append([what, want])
            stats["reports"] += want != "skipped"
            continue
        ra = cli(sourmash_main, cmd, qpath, *files, "-o", a, *flags)
        ta = read(a)
        if ra == "AssertionError":                                  # an `assert` of the reference's own tripped: nothing to follow
            RECORDS.append([what, "skipped"])
            continue
        RECORDS.append([what, digest(("ok", [ra == 0, ta]))])
        if (ra == 0) != (rb == 0) or ta != tb:
            la, lb = (ta or "").splitlines(), (tb or "").splitlines()
            diff = [(x, y) for x, y in zip(la, lb) if x != y][:2] or [("%d lines" % len(la), "%d lines" % len(lb))]
            raise AssertionError("%s %r (abund query: %s, %d subjects, db scaled %d): exit %r / %r\n%s\n%s" % (
                cmd, flags, abund, n_subj, db_scaled, ra, rb, la[:1],
                "\n".join("reference %s\nplugin    %s" % d for d in diff)))
        stats["reports"] += 1
if LIVE:
    with open(golden_path, "w") as fh:                              # one comparison per line
        fh.write('{"seed": %d, "n_trials": %d, "records": [\n%s\n]}\n' % (seed, n_trials, ",\n".join(json.dumps(r) for r in RECORDS)))
else:
    assert len(RECORDS) == len(STORED["records"]), (len(RECORDS), len(STORED["records"]))
print("DIFFERENTIAL OK", stats, len(RECORDS), "comparisons")
'''


def _run_trials(tmp, seed, n_trials, golden_path, live):
    "the trial script against the emulated library; live: the reference's side too, its digests written to golden_path"
    sys.path.insert(0, os.path.join(HERE, "host_emul"))
    try:
        import emul_lib
    finally:
        sys.path.pop(0)
    site = os.path.join(tmp, "site")
    if live:
        over_abi._stub_package(tmp, emul_lib.build())
    else:
        emul_lib.build()
        os.makedirs(site)
    with open(os.path.join(site, "sitecustomize.py"), "w") as fh:       # this package binds the emulated library too
        fh.write("import sys\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport emulated_boot\nemulated_boot.install()\n"
                 % (os.path.join(HERE, "host_emul"), ROOT))
    if live:
        info = os.path.join(site, "sourmash_b200-0.1.0.dist-info")     # the plugin commands, as the reference finds them
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as fh:
            fh.write("Metadata-Version: 2.1\nName: sourmash_b200\nVersion: 0.1.0\n")
        with open(os.path.join(info, "entry_points.txt"), "w") as fh:
            fh.write("[sourmash.cli_script]\n" + "".join("b200%s = sourmash_b200.plugin:Command_B200%s\n" % (c.lower(), c)
                                                          for c in ("Sketch", "Compare", "Search", "Gather", "Prefetch")))
    script = os.path.join(tmp, "trials.py")
    with open(script, "w") as fh:
        fh.write(TRIALS)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([site, os.path.join(tmp, "reftests")]), PYTHONDONTWRITEBYTECODE="1")
    return subprocess.run([sys.executable, script, str(seed), str(n_trials), golden_path, "live" if live else "stored"],
                          capture_output=True, text=True, env=env, cwd=tmp, timeout=int(os.environ.get("SMB_DIFF_TIMEOUT", "1500")))


def _golden(seed):
    return os.path.join(GOLDEN, "differential_seed%d.json" % seed)


REFERENCE_PRESENT = os.path.isdir(os.path.join(REF, "src", "sourmash"))


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("seed", [int(x) for x in os.environ.get("SMB_DIFF_SEEDS", "1").split(",")])   # longer campaigns by hand
def test_batched_functions_equal_the_reference_loops_on_random_lists(tmp_path, seed):
    n_trials = int(os.environ.get("SMB_DIFF_TRIALS", "40"))
    if not REFERENCE_PRESENT and not os.path.exists(_golden(seed)):
        pytest.skip("seed %d: no stored outcomes and no reference copy (oracle/reference.py)" % seed)
    if REFERENCE_PRESENT:                                           # the reference live; its digests must still be the stored ones
        live = str(tmp_path / "live.json")
        r = _run_trials(str(tmp_path / "live"), seed, n_trials, live, True)
        assert r.returncode == 0 and "DIFFERENTIAL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
        if os.path.exists(_golden(seed)):
            with open(live) as a, open(_golden(seed)) as b:
                assert json.load(a) == json.load(b), "the reference's outcomes differ from the stored ones"
    if os.path.exists(_golden(seed)):
        r = _run_trials(str(tmp_path / "stored"), seed, n_trials, _golden(seed), False)
        assert r.returncode == 0 and "DIFFERENTIAL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]


if __name__ == "__main__":                                         # SMB_REFERENCE=<checkout> python <this file> <seed> [trials]
    import tempfile
    assert REFERENCE_PRESENT, "needs the reference copy (oracle/reference.py) or SMB_REFERENCE"
    seed_arg, trials_arg = int(sys.argv[1]), int(sys.argv[2]) if len(sys.argv) > 2 else 40
    with tempfile.TemporaryDirectory() as d:
        r = _run_trials(d, seed_arg, trials_arg, _golden(seed_arg), True)
    print(r.stdout[-2000:], r.stderr[-4000:])
    sys.exit(r.returncode)
