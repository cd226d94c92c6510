"""Bulk .sig loading straight into a GPU-resident SketchSet (SURVEY §8 f1).

The reference loads N signatures as N Python objects (signature.py:383-527), and ``compare`` /
``search`` / ``gather`` then pull every sketch's hashes back out through the FFI one object at a
time.  Here the library parses all files in parallel threads into one CSR (csrc/ingest.cu) and the
rows go to HBM in one copy; Python only sees per-sketch metadata.
"""
import numpy as np

from . import batch as B
from ._ffi import decode_str, rustcall
from ._lowlevel import ffi, lib

_MOLTYPES = {1: "DNA", 2: "protein", 3: "dayhoff", 4: "hp"}
# layout of SmbSketchInfo (include/sourmash_b200.h), natural C alignment
_INFO_DTYPE = np.dtype({"names": ["sig_index", "file", "ksize", "num", "max_hash", "seed", "hash_function",
                                  "has_abund", "n_mins"],
                        "formats": ["<u4", "<u4", "<u4", "<u4", "<u8", "<u8", "<u4", "u1", "<u8"],
                        "offsets": [0, 4, 8, 12, 16, 24, 32, 36, 40], "itemsize": 48})


class SignatureSet:
    """Parsed .sig files: per-sketch metadata on the host, hashes as CSR (numpy views), and
    ``to_sketchset`` to put any selection of rows on the GPU."""

    def __init__(self, ptr):
        self._ptr = ptr
        n = int(lib.smb_sigs_n_sketches(ptr))
        info = ffi.new("SmbSketchInfo[]", max(n, 1))       # one call for all sketches
        lib.smb_sigs_sketch_info_all(ptr, info)
        rec = np.frombuffer(ffi.buffer(info, n * ffi.sizeof("SmbSketchInfo")), dtype=_INFO_DTYPE) if n else \
            np.zeros(0, dtype=_INFO_DTYPE)
        self.ksize, self.num = rec["ksize"].copy(), rec["num"].copy()
        self.max_hash, self.seed = rec["max_hash"].copy(), rec["seed"].copy()
        self.hash_function, self.has_abund = rec["hash_function"].copy(), rec["has_abund"].astype(bool)
        self.sig_index, self.file, self.n_mins = rec["sig_index"].copy(), rec["file"].copy(), rec["n_mins"].copy()
        self.offsets = np.frombuffer(ffi.buffer(lib.smb_sigs_offsets(ptr), (n + 1) * 8), dtype=np.uint64)
        tot = int(self.offsets[-1]) if n else 0
        self.mins = np.frombuffer(ffi.buffer(lib.smb_sigs_mins(ptr), tot * 8), dtype=np.uint64) if tot else np.zeros(0, np.uint64)
        self.abunds = np.frombuffer(ffi.buffer(lib.smb_sigs_abunds(ptr), tot * 8), dtype=np.uint64) if tot else np.zeros(0, np.uint64)

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:
            self.offsets = self.mins = self.abunds = None
            lib.smb_sigs_free(p)

    @classmethod
    def from_files(cls, paths, n_threads=0, *, use_manifest=True, traverse_yield_all=False, loose=None):
        """Parse .sig / .sig.gz files and .zip collections of them.  A zip contributes the members
        ZipFileLinearIndex.signatures() of the reference would yield (index/__init__.py:639-683);
        the two keywords are that class's options.  ``loose``: one flag per path; a flagged path is read as
        one JSON file and contributes nothing when it does not parse (a forced directory's other files)."""
        paths = [str(p).encode("utf-8") for p in paths]
        keep = [ffi.new("char[]", p) for p in paths]
        arr = ffi.new("char *[]", keep)
        flags = (0 if use_manifest else 1) | (2 if traverse_yield_all else 0)
        if loose is None:
            return cls(rustcall(lib.smb_sigs_read_opts, arr, len(paths), int(n_threads), flags))
        mask = np.ascontiguousarray(loose, dtype=np.uint8)
        if len(mask) != len(paths):
            raise ValueError("one loose flag per path")
        return cls(rustcall(lib.smb_sigs_read_loose, arr, len(paths), int(n_threads), flags,
                            ffi.cast("uint8_t *", mask.ctypes.data) if len(mask) else ffi.NULL))

    @classmethod
    def from_objects(cls, objs):
        """Batch of SourmashSignature objects (their first sketch) or of MinHash objects, pulled out of
        the library in one call.  Returns None for mixed / foreign lists (callers fall back)."""
        from .minhash import MinHash
        from .signature import SourmashSignature
        objs = list(objs)
        if objs and all(isinstance(o, SourmashSignature) for o in objs):
            arr = ffi.new("SourmashSignature *[]", [o._get_objptr() for o in objs])
            return cls(rustcall(lib.smb_sigs_from_signatures, arr, len(objs)))
        if objs and all(isinstance(o, MinHash) for o in objs):
            arr = ffi.new("SourmashKmerMinHash *[]", [o._get_objptr() for o in objs])
            return cls(rustcall(lib.smb_sigs_from_minhashes, arr, len(objs)))
        return None

    def python_scaled(self):
        "MinHash.scaled of every sketch (minhash.py:63-67: round((2**64-1)/max_hash), 0 for num sketches)."
        out = np.zeros(len(self), dtype=np.uint64)
        for mx in np.unique(self.max_hash):
            if mx:
                out[self.max_hash == mx] = min(int(round((2**64 - 1) / int(mx), 0)), 2**64 - 1)
        return out

    def csr_host(self, max_hash=0, with_abunds=False):
        """(hashes, offsets[, abunds]) of all sketches on the host, every row cut at max_hash
        (0: as stored) -- rows are sorted, so the cut is a prefix (downsample_scaled)."""
        n = len(self)
        if not max_hash:
            h, off = self.mins, self.offsets
            return (h, off, self.abunds) if with_abunds else (h, off)
        keep = self.mins <= np.uint64(max_hash)
        csum = np.concatenate([[0], np.cumsum(keep, dtype=np.int64)])
        off = csum[self.offsets.astype(np.int64)].astype(np.uint64)
        h = self.mins[keep]
        return (h, off, self.abunds[keep]) if with_abunds else (h, off)

    @classmethod
    def from_json(cls, data):
        buf = data.encode("utf-8") if isinstance(data, str) else bytes(data)
        return cls(rustcall(lib.smb_sigs_parse, buf, len(buf)))

    def __len__(self):
        return len(self.ksize)

    def moltype(self, i):
        return _MOLTYPES[int(self.hash_function[i])]

    def name(self, i):
        return decode_str(lib.smb_sigs_sig_name(self._ptr, int(self.sig_index[i])))

    def filename(self, i):
        return decode_str(lib.smb_sigs_sig_filename(self._ptr, int(self.sig_index[i])))

    def location(self, i):
        "Zip member the sketch was stored in (the manifest's internal_location); '' for plain files."
        return decode_str(lib.smb_sigs_sig_location(self._ptr, int(self.sig_index[i])))

    def locations(self):
        "location(i) of every sketch (one lookup per signature object, cached)."
        if getattr(self, "_locs", None) is None:
            per_sig = {}
            self._locs = [per_sig[j] if j in per_sig else per_sig.setdefault(
                j, decode_str(lib.smb_sigs_sig_location(self._ptr, j))) for j in self.sig_index.tolist()]
        return self._locs

    def md5sums(self):
        "md5 of every sketch, computed from its hashes (what SourmashSignature.md5sum() returns)."
        if getattr(self, "_md5s", None) is None:
            n = len(self)
            buf = ffi.new("char[]", max(32 * n, 1))
            rustcall(lib.smb_sigs_md5_all, self._ptr, buf)
            raw = bytes(ffi.buffer(buf, 32 * n)).decode("ascii")
            self._md5s = [raw[32 * i:32 * i + 32] for i in range(n)]
        return self._md5s

    def md5sum(self, i):
        return decode_str(lib.smb_sigs_sketch_md5(self._ptr, int(i)))

    def row(self, i):
        return self.mins[int(self.offsets[i]):int(self.offsets[i + 1])]

    def select(self, ksize=None, moltype=None, scaled=None, num=None):
        """Indices of the sketches matching the filters (ksize as stored; scaled: sketches that can
        be downsampled to it, i.e. stored scaled <= requested)."""
        keep = np.ones(len(self), bool)
        if ksize is not None:
            keep &= self.ksize == ksize
        if moltype is not None:
            code = {v.lower(): k for k, v in _MOLTYPES.items()}[moltype.lower()]
            keep &= self.hash_function == code
        if scaled is not None:
            keep &= (self.max_hash >= np.uint64(B.max_hash_for_scaled(scaled))) & (self.max_hash != 0)
        if num is not None:
            keep &= self.num == num
        return np.nonzero(keep)[0].astype(np.uint32)

    def signatures(self, rows=None):
        "Rows (default: all) as FrozenSourmashSignature objects, one per sketch, built in one call."
        from .signature import FrozenSourmashSignature
        size = ffi.new("uintptr_t *")
        if rows is None:
            arr = rustcall(lib.smb_sigs_signatures, self._ptr, ffi.NULL, 0, size)
        else:
            rows = np.ascontiguousarray(rows, dtype=np.uint32)
            arr = rustcall(lib.smb_sigs_signatures, self._ptr, ffi.cast("uint32_t *", rows.ctypes.data), len(rows), size)
        try:
            return [FrozenSourmashSignature._from_objptr(arr[i]) for i in range(size[0])]
        finally:
            lib.signatures_array_free(arr, size[0])

    def minhash(self, i):
        "One sketch as a (frozen) MinHash object."
        from .minhash import FrozenMinHash
        return FrozenMinHash._from_objptr(rustcall(lib.smb_sigs_minhash, self._ptr, int(i)))

    def to_sketchset(self, rows=None, scaled=None, with_abunds=False):
        """Rows (default: all) as a GPU-resident SketchSet; ``scaled`` downsamples every row
        (prefix h <= max_hash_for_scaled(scaled), sketch/minhash.rs:777-798)."""
        max_hash = B.max_hash_for_scaled(scaled) if scaled else 0
        if rows is None:
            p = rustcall(lib.smb_sigs_to_sketchset, self._ptr, ffi.NULL, 0, max_hash, bool(with_abunds))
        else:
            rows = np.ascontiguousarray(rows, dtype=np.uint32)
            p = rustcall(lib.smb_sigs_to_sketchset, self._ptr, ffi.cast("uint32_t *", rows.ctypes.data),
                         len(rows), max_hash, bool(with_abunds))
        return B.SketchSet(p)


def compare_signature_files(paths, *, ksize=None, moltype="DNA", scaled=None, n_threads=0):
    """`sourmash compare *.sig` without per-object Python: parse all files natively, downsample to
    the coarsest scaled (commands.py:167-194), one N x N launch.  Returns (matrix, labels)."""
    ss = SignatureSet.from_files(paths, n_threads)
    rows = ss.select(ksize=ksize, moltype=moltype)
    if len(rows) == 0:
        raise ValueError("no signatures match the selection")
    nums = set(int(x) for x in ss.num[rows])
    is_scaled = bool((ss.max_hash[rows] != 0).all())
    if not is_scaled and (len(nums) != 1 or (ss.max_hash[rows] != 0).any()):
        raise ValueError("cannot mix scaled signatures with num signatures / different nums")
    if len(set(int(x) for x in ss.ksize[rows])) != 1:
        raise ValueError("multiple k-mer sizes loaded; please specify one with ksize")
    labels = [ss.name(i) or ss.filename(i) or ss.md5sum(i)[:8] for i in rows]
    if is_scaled:
        coarsest = int(ss.max_hash[rows].min())                     # largest scaled == smallest max_hash
        if scaled:
            coarsest = min(coarsest, B.max_hash_for_scaled(scaled))
        p = rustcall(lib.smb_sigs_to_sketchset, ss._ptr, ffi.cast("uint32_t *", rows.ctypes.data), len(rows),
                     coarsest, False)
        return B.compare_jaccard(B.SketchSet(p)), labels
    return B.compare_jaccard(ss.to_sketchset(rows), num=nums.pop()), labels
