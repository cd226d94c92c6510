"""`sourmash sketch dna | protein | translate` driver on the batched GPU path.

Counterpart of the record loop of sourmash/src/sourmash/command_sketch.py:662-789
(`_compute_individual`: screed record loop -> ``sig.add_sequence(seq, force=not check_sequence)``
or ``sig.add_protein(seq)`` when ``input_is_protein``): the input files are read natively
(``smb_records_read``: FASTA/FASTQ, plain or gzip, one thread per file, sequence bytes in
page-locked memory), all records go to the GPU in one ``smb_sketch_records`` call, and one
``SourmashSignature`` per file (or per record with ``singleton=True``) comes back carrying one
sketch per ksize.
"""
import numpy as np

from . import batch as B
from ._ffi import rustcall
from ._lowlevel import ffi, lib
from .minhash import MinHash
from .signature import SourmashSignature


class RecordBatch:
    """Sequence records of a set of FASTA/FASTQ(.gz) files, parsed by the library."""

    def __init__(self, paths, n_threads=0):
        self.paths = [str(p) for p in paths]
        keep = [ffi.new("char[]", p.encode("utf-8")) for p in self.paths]
        self._ptr = rustcall(lib.smb_records_read, ffi.new("char *[]", keep), len(keep), int(n_threads))
        n = int(lib.smb_records_len(self._ptr))
        self.starts = np.frombuffer(ffi.buffer(lib.smb_records_starts(self._ptr), n * 8), dtype=np.uint64) if n else np.zeros(0, np.uint64)
        self.lengths = np.frombuffer(ffi.buffer(lib.smb_records_lengths(self._ptr), n * 8), dtype=np.uint64) if n else np.zeros(0, np.uint64)
        self.files = np.frombuffer(ffi.buffer(lib.smb_records_files(self._ptr), n * 4), dtype=np.uint32) if n else np.zeros(0, np.uint32)
        self.total_bytes = int(lib.smb_records_total_bytes(self._ptr))

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:
            self.starts = self.lengths = self.files = None
            lib.smb_records_free(p)

    def __len__(self):
        return len(self.files)

    def names(self):
        noff = ffi.new("uint64_t **")
        base = lib.smb_records_names(self._ptr, noff)
        n = len(self)
        off = np.frombuffer(ffi.buffer(noff[0], (n + 1) * 8), dtype=np.uint64)
        blob = bytes(ffi.buffer(base, int(off[-1]))) if n and off[-1] else b""
        return [blob[int(off[i]):int(off[i + 1])].decode("utf-8", "replace") for i in range(n)]

    def sequence(self, i):
        lo, n = int(self.starts[i]), int(self.lengths[i])
        return bytes(ffi.buffer(lib.smb_records_data(self._ptr) + lo, n)) if n else b""

    def sketch(self, rec_to_sketch, n_sketches, ksizes, *, moltype="DNA", input_is_protein=False, scaled=0, num=0,
               seed=42, track_abundance=False):
        ks = np.ascontiguousarray(ksizes, dtype=np.uint32)
        hf = B._HASH_FUNCTIONS[moltype.lower()]
        if hf != 1:
            ks = np.ascontiguousarray(ks * np.uint32(3))
        elif input_is_protein:
            raise ValueError("cannot add protein sequence to DNA MinHash")
        r2s = np.ascontiguousarray(rec_to_sketch, dtype=np.uint32)
        nk = ffi.new("uint64_t *")
        p = rustcall(lib.smb_sketch_records, self._ptr, ffi.cast("uint32_t *", r2s.ctypes.data) if len(r2s) else ffi.NULL,
                     int(n_sketches), ffi.cast("uint32_t *", ks.ctypes.data), len(ks), hf, bool(input_is_protein),
                     int(scaled), int(num), int(seed), bool(track_abundance), nk)
        return B.SketchSet(p), int(nk[0])


def read_sequences(path):
    """[(name, sequence bytes)] of a FASTA or FASTQ file (optionally gzipped)."""
    rb = RecordBatch([path])
    return list(zip(rb.names(), (rb.sequence(i) for i in range(len(rb)))))


def _signature_from_rows(rows, abunds, ksizes, scaled, num, seed, track, name, filename, moltype="DNA"):
    sig = SourmashSignature.__new__(SourmashSignature)
    sig._objptr = lib.signature_new()
    sig._shared = False
    mol = moltype.lower()
    for i, k in enumerate(ksizes):
        mh = MinHash(num, k, scaled=scaled, seed=seed, track_abundance=track, is_protein=mol == "protein",
                     dayhoff=mol == "dayhoff", hp=mol == "hp")
        if track:
            mh.set_abundances(dict(zip(rows[i].tolist(), abunds[i].tolist())))
        else:
            mh.add_many(rows[i])
        rustcall(lib.signature_push_mh, sig._get_objptr(), mh._get_objptr())
    if name:
        sig._name = name
    if filename:
        sig.filename = filename
    return sig


def sketch_fasta_files(filenames, *, ksizes=(21, 31, 51), scaled=1000, num=0, seed=42, track_abundance=False,
                       singleton=False, name_from_first=False, check_sequence=False, moltype="DNA",
                       input_is_protein=False, n_threads=0, merge=None):
    """Sketch every input file on the GPU; returns a list of SourmashSignature (one sketch per ksize).

    ``moltype`` "protein" / "dayhoff" / "hp" with ``input_is_protein`` is `sketch protein`; without
    it the DNA is translated in six frames (`sketch translate`); ksizes are then in residues.
    ``check_sequence=True`` reproduces ``--check-sequence`` (force=False: the first invalid k-mer
    raises ValueError) through the per-record ABI call; the default skips invalid k-mers like
    the reference CLI (command_sketch.py:827-832).  ``merge="name"`` is ``--merge``: every record of
    every file goes into one signature with that name, filename = the last input
    (_compute_merged, command_sketch.py:791-824)."""
    ksizes = list(ksizes)
    rb = RecordBatch(filenames, n_threads)
    rec_names = rb.names() if (singleton or name_from_first) else None
    names, files = [], []
    if merge is not None:
        if singleton:
            raise ValueError("cannot specify both 'singleton' and 'merge'")
        if len(rb) == 0:
            return []                                      # "no sequences found": nothing is saved
        owner = np.zeros(len(rb), dtype=np.uint32)
        names, files = [merge], [rb.paths[-1]]
    elif singleton:
        owner = np.arange(len(rb), dtype=np.uint32)
        names = rec_names
        files = [rb.paths[int(f)] for f in rb.files]
    else:
        owner = rb.files.copy()
        first_of = {}
        if name_from_first:
            for i, f in enumerate(rb.files):
                first_of.setdefault(int(f), rec_names[i])
        names = [first_of.get(i, "") for i in range(len(rb.paths))]
        files = list(rb.paths)
    n_sk = len(names)
    # a file without records gives no signature ("no sequences found in ...", command_sketch.py:697-700)
    keep = [bool(c) for c in np.bincount(owner, minlength=n_sk)] if (merge is None and not singleton) else [True] * n_sk
    if check_sequence and moltype.lower() == "dna":
        sigs = []
        empty = [np.zeros(0, np.uint64)] * len(ksizes)
        for s in range(n_sk):
            sig = _signature_from_rows(empty, empty, ksizes, scaled, num, seed, track_abundance, names[s], files[s])
            for i in np.nonzero(owner == s)[0]:
                sig.add_sequence(rb.sequence(int(i)), force=False)
            sigs.append(sig)
        return [sig for sig, k in zip(sigs, keep) if k]
    nk = len(ksizes)
    if len(rb) == 0:                                       # no records anywhere: nothing to save
        return []
    sset, _ = rb.sketch(owner, n_sk, ksizes, moltype=moltype, input_is_protein=input_is_protein, scaled=scaled,
                        num=num, seed=seed, track_abundance=track_abundance)
    hf = B._HASH_FUNCTIONS[moltype.lower()]
    ks = np.ascontiguousarray(ksizes, dtype=np.uint32) * np.uint32(3 if hf != 1 else 1)
    size = ffi.new("uintptr_t *")
    arr = rustcall(lib.smb_signatures_from_sketchset, sset._ptr, ffi.cast("uint32_t *", ks.ctypes.data), nk, hf,
                   int(scaled), int(num), int(seed), size)
    sigs = [SourmashSignature._from_objptr(arr[i]) for i in range(size[0])]
    lib.signatures_array_free(arr, size[0])
    for s_, sig in enumerate(sigs):
        if names[s_]:
            sig._name = names[s_]
        if files[s_]:
            sig.filename = files[s_]
    return [sig for sig, k in zip(sigs, keep) if k]
