"""`sourmash scripts b200sigmerge | b200sigintersect | b200sigsubtract`: union, intersection and difference of many
sketches in one device sort.

The reference's `sourmash sig merge` (src/sourmash/sig/__main__.py:459-523) calls ``MinHash.merge`` once per signature,
and every call copies the running union into a new vector (src/core/src/sketch/minhash.rs:432-516): merging n sketches
moves O(n |union|) hashes.  `sig intersect` and `sig subtract` (:526-592, :643-712) build a Python set of every hash
of every signature.  Here the sketches are parsed natively into one CSR (``SignatureSet.from_files``), uploaded in one
copy, and combined by ``batch.combine``: one stable radix sort of the whole set and one pass over its runs of equal
hashes.  Only the compatibility checks run on the host, on the per-sketch metadata arrays; hashes never pass through
Python objects.

``merge_minhashes``, ``intersect_minhashes`` and ``subtract_minhashes`` do the same for a list of ``MinHash`` or
``SourmashSignature`` objects, with the reference commands' semantics: the first sketch is the template
(``copy_and_clear``), intersect and subtract flatten the result, and incompatible sketches raise the errors
``MinHash.merge`` / ``is_compatible`` would.

The commands take the reference's options and give its outputs, messages and exit codes:

    sourmash scripts b200sigmerge a.sig b.sig.gz c.zip dir/ -k 31 --dna --flatten --set-name all -o merged.sig
    sourmash scripts b200sigintersect a.sig b.sig -A a.sig -o common.sig
    sourmash scripts b200sigsubtract a.sig b.sig c.sig --flatten -o rest.sig

Also ``python -m sourmash_b200.sigsetops merge|intersect|subtract ...``.  The command classes are not yet declared as
``sourmash.cli_script`` entry points in pyproject.toml, whose declared list the test suite pins to the six existing
commands; ``sourmash scripts ...`` finds them once they are.  Inputs are .sig / .sig.gz files, .zip
collections and directories of .sig files, named on the command line or (merge, intersect) listed in --from-file.
Not supported, and refused by the argument parser: picklists (--picklist, --picklist-require-all), -f/--force, and
writing a .zip collection with -o.  Any other -o path is written as a .sig JSON file (gzip-compressed for .gz).
"""
import argparse
import sys

import numpy as np

from . import batch as B
from .plugin import CommandLinePlugin, _expand
from .sigkmers import _error


def _notify(args, msg, end="\n"):
    "the reference's notify: clears the terminal line first; end='\\r' messages are overwritten by the next one"
    if not getattr(args, "quiet", False):
        print("\r\033[K", end="", file=sys.stderr)
        print(msg, end=end, file=sys.stderr)


class IncompatibleSketches(ValueError):
    """A sketch the operation cannot take.  ``index``: its position in the input; ``exit_code``: what the reference's
    command exits with on it."""

    def __init__(self, msg, index, exit_code=-1):
        super().__init__(msg)
        self.index, self.exit_code = index, exit_code


_MERGE_MISMATCH = ((lambda ss, r, t: ss.ksize[r] != ss.ksize[t], "different ksizes cannot be compared"),
                   (lambda ss, r, t: ss.hash_function[r] != ss.hash_function[t], "DNA/prot minhashes cannot be compared"),
                   (lambda ss, r, t: ss.max_hash[r] != ss.max_hash[t], "mismatch in scaled; comparison fail"),
                   (lambda ss, r, t: ss.seed[r] != ss.seed[t], "mismatch in seed; comparison fail"))


def _first_mismatch(ss, rows):
    """(position, message) of the first row that KmerMinHash::check_compatible (minhash.rs:886-912) refuses against
    rows[0] -- ksize, hash function, max_hash, seed, in that order -- or None"""
    rows = np.asarray(rows)
    bad = np.zeros(len(rows), bool)
    for test, _ in _MERGE_MISMATCH:
        bad |= test(ss, rows, rows[0])
    if not bad.any():
        return None
    i = int(np.argmax(bad))
    msg = next(m for test, m in _MERGE_MISMATCH if test(ss, rows[i], rows[0]))
    return i, msg


def _minhash_from(template, hashes, abunds):
    "a copy_and_clear()-ed template filled with the given sorted hashes (and abundances)"
    from ._lowlevel import ffi, lib
    n = len(hashes)
    if not n:
        return template
    h = np.ascontiguousarray(hashes, dtype=np.uint64)
    if abunds is not None:
        a = np.ascontiguousarray(abunds, dtype=np.uint64)
        template._methodcall(lib.kmerminhash_set_abundances, ffi.cast("uint64_t *", h.ctypes.data),
                             ffi.cast("uint64_t *", a.ctypes.data), n, True)
    else:
        template.add_many(h)
    return template


def merge_rows(ss, rows, *, flatten=False):
    """`sig merge` of the sketches ``rows`` of a ``SignatureSet``, in that order.  Raises IncompatibleSketches at the
    first sketch the reference's loop refuses: a different track_abundance than the first (unless ``flatten``), then
    check_compatible."""
    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    track = bool(ss.has_abund[rows[0]]) and not flatten
    refused = []                              # (position, message); the abundance check runs first for a sketch
    if not flatten:
        differs = np.nonzero(ss.has_abund[rows] != ss.has_abund[rows[0]])[0]
        if len(differs):
            i = int(differs[0])
            refused.append((i, "incompatible signatures: track_abundance is %s in first sig, %s in second"
                            % (bool(ss.has_abund[rows[0]]), bool(ss.has_abund[rows[i]]))))
    mismatch = _first_mismatch(ss, rows)
    if mismatch is not None:
        refused.append(mismatch)
    if refused:
        raise IncompatibleSketches(*min(refused, key=lambda r: r[0])[::-1])
    mh = ss.minhash(int(rows[0])).copy_and_clear()
    if flatten:
        mh.track_abundance = False
    hashes, abunds = B.combine(ss.to_sketchset(rows, with_abunds=track), "union", num=int(ss.num[rows[0]]))
    return _minhash_from(mh, hashes, abunds if track else None)


def _check_compatible(ss, rows):
    found = _first_mismatch(ss, rows)
    if found is not None:
        raise IncompatibleSketches("incompatible minhashes; specify -k and/or molecule type.", found[0])


def intersect_rows(ss, rows):
    "`sig intersect` of the sketches ``rows``: the hashes every one holds, in a flat copy_and_clear() of the first"
    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    _check_compatible(ss, rows)
    hashes, _ = B.combine(ss.to_sketchset(rows), "all")
    return _minhash_from(ss.minhash(int(rows[0])).copy_and_clear().flatten(), hashes, None)


def subtract_rows(ss, rows, *, flatten=False):
    """`sig subtract`: the hashes of sketch rows[0] that none of the others holds, in a flat copy_and_clear() of it.
    Sketches with abundances are refused (exit code 1) unless ``flatten``."""
    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    abund_msg = "Cannot use subtract on signatures with abundance tracking, sorry!"
    if ss.has_abund[rows[0]] and not flatten:
        raise IncompatibleSketches(abund_msg, 0, exit_code=1)
    refused = []                              # (position, message, exit code); compatibility is checked first
    mismatch = _first_mismatch(ss, rows)
    if mismatch is not None:
        refused.append((mismatch[0], "incompatible minhashes; specify -k and/or molecule type.", -1))
    tracked = np.nonzero(ss.has_abund[rows])[0] if not flatten else []
    if len(tracked):
        refused.append((int(tracked[0]), abund_msg, 1))
    if refused:
        i, msg, code = min(refused, key=lambda r: r[0])
        raise IncompatibleSketches(msg, i, exit_code=code)
    hashes, _ = B.combine(ss.to_sketchset(rows), "first_only")
    return _minhash_from(ss.minhash(int(rows[0])).copy_and_clear().flatten(), hashes, None)


def _object_set(objs):
    from .sigset import SignatureSet
    objs = list(objs)
    if not objs:
        raise ValueError("no sketches given")
    ss = SignatureSet.from_objects(objs)
    if ss is None:
        raise TypeError("expected a list of MinHash or of SourmashSignature objects")
    return ss, np.arange(len(ss), dtype=np.uint32)


def merge_minhashes(objs, *, flatten=False):
    """The union of a list of MinHash / SourmashSignature objects as one MinHash, as `sig merge` builds it: a
    copy_and_clear() of the first, abundances summed (unless ``flatten``), a num sketch's bottom num kept."""
    return merge_rows(*_object_set(objs), flatten=flatten)


def intersect_minhashes(objs):
    "The hashes common to all of a list of MinHash / SourmashSignature objects, as `sig intersect` builds them (flat)"
    return intersect_rows(*_object_set(objs))


def subtract_minhashes(objs, *, flatten=False):
    "The hashes of the first of a list of MinHash / SourmashSignature objects that none of the others holds (flat)"
    return subtract_rows(*_object_set(objs), flatten=flatten)


# ---------------------------------------------------------------------------------------------------- commands
def _moltype_args(p):
    "the reference's add_ksize_arg / add_moltype_args (cli/utils.py)"
    p.add_argument("-k", "--ksize", metavar="K", default=None, type=int, help="k-mer size to select; no default.")
    for name, flags in (("protein", ["--protein"]), ("dayhoff", ["--dayhoff"]),
                        ("hp", ["--hp", "--hydrophobic-polar"])):
        p.add_argument(*flags, dest=name, action="store_true", help="choose %s signatures" % name)
        p.add_argument(*[f.replace("--", "--no-", 1) for f in flags], dest=name, action="store_false",
                       help="do not choose %s signatures" % name)
        p.set_defaults(**{name: False})
    p.add_argument("--dna", "--rna", "--nucleotide", dest="dna", default=None, action="store_true",
                   help="choose a nucleotide signature")
    p.add_argument("--no-dna", "--no-rna", "--no-nucleotide", dest="dna", action="store_false",
                   help="do not choose a nucleotide signature")
    p.set_defaults(dna=None)


def _common_args(p, *, set_name_alias=False):
    p.add_argument("-o", "--output", metavar="FILE", default="-", help="output signature to this file (default stdout)")
    if set_name_alias:
        p.add_argument("--set-name", "--name", help="rename merged signature")
    else:
        p.add_argument("--set-name", help="set name for output signature")
    _moltype_args(p)


def _moltype(args):
    "calculate_moltype (sourmash_args.py): at most one moltype flag"
    picked = [m for m, on in (("DNA", args.dna), ("dayhoff", args.dayhoff), ("hp", args.hp),
                               ("protein", args.protein)) if on]
    if len(picked) > 1:
        _error("cannot specify more than one of --dna/--rna/--nucleotide/--protein/--hp/--dayhoff")
        raise SystemExit(-1)
    return picked[-1] if picked else None


def _check_output(parser, args):
    if str(args.output).endswith(".zip"):
        parser.error("writing a .zip collection is not supported; use a .sig or .sig.gz path, or - for stdout")


def _load(paths, ksize, moltype):
    """All sketches of the given locations in the reference's load order (location, signature, sketch), selected
    by -k (residues for protein-family sketches) and moltype: (SignatureSet, rows, files, origin), where sketch r
    was read from files[ss.file[r]], named by argument origin[ss.file[r]]"""
    from .sigset import SignatureSet
    files, origin = _expand(paths)
    ss = SignatureSet.from_files(files)
    keep = np.ones(len(ss), bool)
    if ksize is not None:
        dna = ss.hash_function == 1
        keep &= np.where(dna, ss.ksize == ksize, ss.ksize == 3 * ksize)
    if moltype is not None:
        code = {"DNA": 1, "protein": 2, "dayhoff": 3, "hp": 4}[moltype]
        keep &= ss.hash_function == code
    rows = np.nonzero(keep)[0].astype(np.uint32)
    return ss, rows, files, np.asarray(origin, dtype=np.int64)


def _save(args, mh):
    from .signature import SourmashSignature, save_signatures_to_json
    sig = SourmashSignature(mh, name=args.set_name or "")
    if args.output == "-":
        save_signatures_to_json([sig], sys.stdout)
        sys.stdout.flush()
        return
    gz = args.output.endswith(".gz")
    with open(args.output, "wb" if gz else "w", encoding=None if gz else "utf-8") as fp:
        save_signatures_to_json([sig], fp, compression=1 if gz else 0)


def _abundances_from(args, moltype, mh):
    "-A: abundances of exactly one signature, through MinHash.inflate"
    _notify(args, f"loading signature from {args.abundances_from}, keeping abundances")
    ss, rows, _, _ = _load([args.abundances_from], args.ksize, moltype)
    if len(rows) == 0:
        raise ValueError(f"no signatures in '{args.abundances_from}'? expected exactly one.")
    if len(rows) > 1:
        raise ValueError(f"more than one signature in '{args.abundances_from}'; expected exactly one")
    abund_mh = ss.minhash(int(rows[0]))
    if not abund_mh.track_abundance:
        _error("--track-abundance not set on loaded signature?! exiting.")
        raise SystemExit(-1)
    return mh.inflate(abund_mh)


def _signature_paths(args):
    paths = list(args.signatures)
    if args.from_file:
        with open(args.from_file) as fh:
            paths += [line.strip() for line in fh if line.strip()]
    return paths


class _SetOpCommand(CommandLinePlugin):
    def __init__(self, p):
        super().__init__(p)
        self._parser = p


class Command_B200SigMerge(_SetOpCommand):
    command = "b200sigmerge"
    description = "merge signatures (sig merge): the union of all their hashes, in one sort on a GPU"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("signatures", nargs="*")
        p.add_argument("--flatten", action="store_true", help="remove abundances from all signatures")
        p.add_argument("--from-file", help="a text file containing a list of files to load signatures from")
        _common_args(p, set_name_alias=True)

    def main(self, args):
        super().main(args)
        _check_output(self._parser, args)
        moltype = _moltype(args)
        ss, rows, files, _ = _load(_signature_paths(args), args.ksize, moltype)
        if not len(rows):
            _error("no signatures to merge!?")
            raise SystemExit(-1)
        try:
            mh = merge_rows(ss, rows, flatten=args.flatten)
        except IncompatibleSketches as exc:
            r = int(rows[exc.index])
            name = ss.name(r) or ss.filename(r) or ss.md5sum(r)[:8]
            _error(f"ERROR when merging signature '{name}' ({ss.md5sum(r)[:8]}) from file {files[int(ss.file[r])]}")
            _error(str(exc))
            raise SystemExit(exc.exit_code)
        _save(args, mh)
        _notify(args, f"loaded and merged {len(rows)} signatures")
        return 0


class Command_B200SigIntersect(_SetOpCommand):
    command = "b200sigintersect"
    description = "intersect signatures (sig intersect): the hashes all of them hold, in one sort on a GPU"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("signatures", nargs="*")
        p.add_argument("-A", "--abundances-from", metavar="FILE",
                       help="intersect with & take abundances from this signature")
        p.add_argument("--from-file", help="a text file containing a list of files to load signatures from")
        _common_args(p)

    def main(self, args):
        super().main(args)
        _check_output(self._parser, args)
        moltype = _moltype(args)
        ss, rows, _, _ = _load(_signature_paths(args), args.ksize, moltype)
        if not len(rows):
            _notify(args, "no signatures provided to intersect!?")
            raise SystemExit(-1)
        try:
            mh = intersect_rows(ss, rows)
        except IncompatibleSketches as exc:
            _error(str(exc))
            raise SystemExit(exc.exit_code)
        if args.abundances_from:
            mh = _abundances_from(args, moltype, mh)
        _save(args, mh)
        _notify(args, f"loaded and intersected {len(rows)} signatures")
        return 0


class Command_B200SigSubtract(_SetOpCommand):
    command = "b200sigsubtract"
    description = "subtract signatures (sig subtract): the hashes of the first that no other holds, on a GPU"

    def __init__(self, p):
        super().__init__(p)
        p.add_argument("signature_from")
        p.add_argument("subtraction_sigs", nargs="+")
        p.add_argument("--flatten", action="store_true", help="remove abundance from signatures before subtracting")
        p.add_argument("-A", "--abundances-from", metavar="FILE",
                       help="intersect with & take abundances from this signature")
        _common_args(p)

    def main(self, args):
        super().main(args)
        _check_output(self._parser, args)
        moltype = _moltype(args)
        if args.abundances_from:
            args.flatten = True
        ss, rows, _, origin = _load([args.signature_from] + list(args.subtraction_sigs), args.ksize, moltype)
        first = rows[origin[ss.file[rows]] == 0]
        if len(first) != 1:
            raise ValueError(f"no signatures in '{args.signature_from}'? expected exactly one." if not len(first) else
                             f"more than one signature in '{args.signature_from}'; expected exactly one")
        if ss.has_abund[first[0]] and not args.flatten:
            _error("Cannot use subtract on signatures with abundance tracking, sorry!")
            raise SystemExit(1)
        _notify(args, f"loaded signature from {args.signature_from}...", end="\r")
        rows = np.concatenate([first, rows[origin[ss.file[rows]] != 0]]).astype(np.uint32)
        if len(rows) == 1:
            _error("no signatures to subtract!?")
            raise SystemExit(-1)
        try:
            mh = subtract_rows(ss, rows, flatten=args.flatten)
        except IncompatibleSketches as exc:
            _error(str(exc))
            raise SystemExit(exc.exit_code)
        if args.abundances_from:
            mh = _abundances_from(args, moltype, mh)
        _save(args, mh)
        _notify(args, f"loaded and subtracted {len(rows) - 1} signatures")
        return 0


_COMMANDS = {"merge": Command_B200SigMerge, "intersect": Command_B200SigIntersect, "subtract": Command_B200SigSubtract}


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    parser = argparse.ArgumentParser(prog="python -m sourmash_b200.sigsetops")
    sub = parser.add_subparsers(dest="op", required=True)
    cmds = {name: cls(sub.add_parser(name, description=cls.description)) for name, cls in _COMMANDS.items()}
    args = parser.parse_args(argv)
    return cmds[args.op].main(args)


if __name__ == "__main__":
    sys.exit(main())
