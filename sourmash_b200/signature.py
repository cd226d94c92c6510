"""SourmashSignature: named container of sketches over the C ABI.

Mirrors the part of sourmash/src/sourmash/signature.py (:29-527) that sits on the
hot path: construction from a MinHash, ``add_sequence`` (every sketch of the signature sees
the sequence), the comparison delegates, md5sum identity, and ``.sig`` JSON I/O through the
library's native reader / writer (csrc/ingest.cu; format: signature.rs:401-445).
"""
import contextlib
import os

from ._lowlevel import ffi, lib
from .minhash import FrozenMinHash, MinHash
from ._ffi import RustObject, decode_str, rustcall

SIGNATURE_VERSION = 0.4


class SourmashSignature(RustObject):
    "A sketch (or several) plus name / filename metadata."

    __dealloc_func__ = lib.signature_free

    def __init__(self, minhash, name="", filename=""):
        self._objptr = lib.signature_new()
        if name:
            self._name = name
        if filename:
            self.filename = filename
        self.minhash = minhash

    # -- sketch access (signature_first_mh clones: ffi/signature.rs:169-185) -------------------
    @property
    def minhash(self):
        return FrozenMinHash._from_objptr(self._methodcall(lib.signature_first_mh))

    @minhash.setter
    def minhash(self, value):
        self._methodcall(lib.signature_set_mh, value._get_objptr())

    def sketches(self):
        "All sketches of this signature (clones)."
        size = ffi.new("uintptr_t *")
        arr = self._methodcall(lib.signature_get_mhs, size)
        try:
            return [FrozenMinHash._from_objptr(arr[i]) for i in range(size[0])]
        finally:
            lib.smb_mh_array_free(arr)                     # the pointer array; the clones now belong to the wrappers

    def __len__(self):
        return self._methodcall(lib.signature_len)

    # -- metadata ----------------------------------------------------------------------------
    @property
    def name(self):
        return decode_str(self._methodcall(lib.signature_get_name))

    @name.setter
    def name(self, value):
        self._methodcall(lib.signature_set_name, value.encode("utf-8"))

    @property
    def _name(self):
        return self.name

    @_name.setter
    def _name(self, value):
        self._methodcall(lib.signature_set_name, value.encode("utf-8"))

    @property
    def filename(self):
        return decode_str(self._methodcall(lib.signature_get_filename))

    @filename.setter
    def filename(self, value):
        self._methodcall(lib.signature_set_filename, value.encode("utf-8"))

    @property
    def license(self):
        return decode_str(self._methodcall(lib.signature_get_license))

    def md5sum(self):
        "md5 of the (first) sketch: the signature's identity key."
        return self.minhash.md5sum()

    def __hash__(self):
        return hash(self.md5sum())

    def __str__(self):
        n, fn, md5 = self.name, self.filename, self.md5sum()
        return n or fn or md5[:8]

    def __repr__(self):
        return f"SourmashSignature({self.name!r}, {self.md5sum()[:8]})"

    def __eq__(self, other):
        return self._methodcall(lib.signature_eq, other._get_objptr())

    def __ne__(self, other):
        return not self == other

    # -- hot path ----------------------------------------------------------------------------
    def add_sequence(self, sequence, force=False):
        "Hash the sequence into every sketch of the signature (GPU)."
        seq = sequence.encode("utf-8") if isinstance(sequence, str) else bytes(sequence)
        self._methodcall(lib.signature_add_sequence, seq, force)

    def add_protein(self, sequence):
        self._methodcall(lib.signature_add_protein, sequence.encode("utf-8"))

    def similarity(self, other, ignore_abundance=False, downsample=False):
        return self.minhash.similarity(other.minhash, ignore_abundance=ignore_abundance, downsample=downsample)

    def jaccard(self, other):
        return self.minhash.similarity(other.minhash, ignore_abundance=True, downsample=False)

    def contained_by(self, other, downsample=False):
        return self.minhash.contained_by(other.minhash, downsample)

    def max_containment(self, other, downsample=False):
        return self.minhash.max_containment(other.minhash, downsample)

    def avg_containment(self, other, downsample=False):
        return self.minhash.avg_containment(other.minhash, downsample=downsample)

    @classmethod
    def from_params(cls, params):
        "Empty signature with one sketch per ksize of a ComputeParameters (signature_from_params)."
        rv = object.__new__(cls)
        rv._objptr = rustcall(lib.signature_from_params, params._get_objptr())
        rv._shared = False
        return rv

    # -- ANI delegates (signature.py:186-222 of the reference) ---------------------------------
    def jaccard_ani(self, other, *, downsample=False, jaccard=None, prob_threshold=1e-3, err_threshold=1e-4):
        return self.minhash.jaccard_ani(other.minhash, downsample=downsample, jaccard=jaccard,
                                        prob_threshold=prob_threshold, err_threshold=err_threshold)

    def containment_ani(self, other, *, downsample=False, containment=None, confidence=0.95, estimate_ci=False):
        return self.minhash.containment_ani(other.minhash, downsample=downsample, containment=containment,
                                            confidence=confidence, estimate_ci=estimate_ci)

    def max_containment_ani(self, other, *, downsample=False, max_containment=None, confidence=0.95,
                            estimate_ci=False):
        return self.minhash.max_containment_ani(other.minhash, downsample=downsample,
                                                max_containment=max_containment, confidence=confidence,
                                                estimate_ci=estimate_ci)

    def avg_containment_ani(self, other, *, downsample=False):
        return self.minhash.avg_containment_ani(other.minhash, downsample=downsample)

    # -- copies, pickling, freezing (signature.py:236-290) --------------------------------------
    def __getstate__(self):
        return (self.minhash, self.name, self.filename)

    def __setstate__(self, tup):
        mh, name, filename = tup
        self.__del__()
        self._objptr = lib.signature_new()
        self._shared = False
        if name:
            self._methodcall(lib.signature_set_name, name.encode("utf-8"))
        if filename:
            self._methodcall(lib.signature_set_filename, filename.encode("utf-8"))
        self._methodcall(lib.signature_set_mh, mh._get_objptr())

    def __reduce__(self):
        return (SourmashSignature, (self.minhash, self.name, self.filename))

    def __copy__(self):
        return SourmashSignature(self.minhash, name=self.name, filename=self.filename)

    copy = __copy__

    def to_frozen(self):
        "Frozen copy of this signature."
        new_ss = self.copy()
        new_ss.__class__ = FrozenSourmashSignature
        return new_ss

    def to_mutable(self):
        "Mutable copy of this signature."
        return self.copy()

    def into_frozen(self):
        "Freeze this signature in place."
        self.__class__ = FrozenSourmashSignature


class FrozenSourmashSignature(SourmashSignature):
    "Immutable signature (signature.py:293-352 of the reference): what the loaders return."

    @SourmashSignature.minhash.setter
    def minhash(self, value):
        raise ValueError("cannot set .minhash on FrozenSourmashSignature")

    @SourmashSignature._name.setter
    def _name(self, value):
        raise ValueError("cannot set ._name on FrozenSourmashSignature")

    @SourmashSignature.name.setter
    def name(self, value):
        raise ValueError("cannot set .name on FrozenSourmashSignature")

    @SourmashSignature.filename.setter
    def filename(self, value):
        raise ValueError("cannot set .filename on FrozenSourmashSignature")

    def add_sequence(self, sequence, force=False):
        raise ValueError("cannot add sequence data to FrozenSourmashSignature")

    def add_protein(self, sequence):
        raise ValueError("cannot add protein sequence to FrozenSourmashSignature")

    def __copy__(self):
        return self

    copy = __copy__

    def to_frozen(self):
        return self

    def to_mutable(self):
        mut = SourmashSignature.__new__(SourmashSignature)
        mut._objptr = None
        mut.__setstate__(self.__getstate__())
        return mut

    def into_frozen(self):
        self.__class__ = FrozenSourmashSignature

    @contextlib.contextmanager
    def update(self):
        "Context manager yielding a mutable copy that is frozen again on exit."
        new_copy = self.to_mutable()
        yield new_copy
        new_copy.into_frozen()


class ComputeParameters(RustObject):
    "Parameter bag used by ``sketch`` to build template sketches (command_sketch.py:864-1085)."

    __dealloc_func__ = lib.computeparams_free

    def __init__(self, *, ksizes=(21, 31, 51), seed=42, dna=True, num_hashes=0, track_abundance=False, scaled=1000):
        self._objptr = lib.computeparams_new()
        self.ksizes = list(ksizes)
        self.seed, self.dna = seed, dna
        self.num_hashes, self.track_abundance, self.scaled = num_hashes, track_abundance, scaled

    @property
    def ksizes(self):
        size = ffi.new("uintptr_t *")
        ptr = self._methodcall(lib.computeparams_ksizes, size)
        out = list(ffi.unpack(ptr, size[0]))
        lib.computeparams_ksizes_free(ptr, size[0])
        return out

    @ksizes.setter
    def ksizes(self, v):
        self._methodcall(lib.computeparams_set_ksizes, list(v), len(v))

    seed = property(lambda s: s._methodcall(lib.computeparams_seed),
                    lambda s, v: s._methodcall(lib.computeparams_set_seed, v))
    dna = property(lambda s: s._methodcall(lib.computeparams_dna),
                   lambda s, v: s._methodcall(lib.computeparams_set_dna, v))
    protein = property(lambda s: s._methodcall(lib.computeparams_protein),
                       lambda s, v: s._methodcall(lib.computeparams_set_protein, v))
    dayhoff = property(lambda s: s._methodcall(lib.computeparams_dayhoff),
                       lambda s, v: s._methodcall(lib.computeparams_set_dayhoff, v))
    hp = property(lambda s: s._methodcall(lib.computeparams_hp),
                  lambda s, v: s._methodcall(lib.computeparams_set_hp, v))
    num_hashes = property(lambda s: s._methodcall(lib.computeparams_num_hashes),
                          lambda s, v: s._methodcall(lib.computeparams_set_num_hashes, v))
    scaled = property(lambda s: s._methodcall(lib.computeparams_scaled),
                      lambda s, v: s._methodcall(lib.computeparams_set_scaled, int(v)))
    track_abundance = property(lambda s: s._methodcall(lib.computeparams_track_abundance),
                               lambda s, v: s._methodcall(lib.computeparams_set_track_abundance, v))


# ---------------------------------------------------------------------------------------------
# .sig JSON (signature.rs:401-445; sketch fields sketch/minhash.rs:103-184): parsed and written
# by the library (csrc/ingest.cu) through the reference's own entry points
# signatures_load_path / signatures_load_buffer / signatures_save_buffer
# (signature.py:383-527 -> ffi/signature.rs:219-343).
# ---------------------------------------------------------------------------------------------
def load_signatures_from_json(data, ksize=None, select_moltype=None, ignore_md5sum=False, do_raise=False):
    """Yield SourmashSignature objects (one per sketch) from a .sig / .sig.gz path, JSON text,
    bytes (optionally gzipped) or a file object.  ``ksize`` is compared with the stored value
    (3 x residues for protein-family sketches), like the reference (signature.rs:611-616).
    What counts as which kind of input, and which failures are swallowed unless ``do_raise``, follow
    signature.py:350-471: anything with read / fileno / mode is read (a failing read is swallowed too), text or bytes
    holding "sourmash_signature" or starting with the gzip magic is a buffer, an existing path is a path, the rest is an error."""
    if not data:
        return
    file_like = hasattr(data, "read") or hasattr(data, "fileno") or hasattr(data, "mode")
    is_buffer = False
    if not file_like and hasattr(data, "find"):
        try:
            is_buffer = data.find("sourmash_signature") > 0
        except TypeError:
            is_buffer = data.find(b"sourmash_signature") > 0 or data.startswith(b"\x1f\x8b")
    is_path = False
    if not file_like and not is_buffer:
        try:
            is_path = os.path.exists(data)
        except (ValueError, TypeError):
            is_path = False
        if not is_path:
            if do_raise:
                raise ValueError("Error in parsing signature; quitting. Cannot open file or invalid signature")
            return
    moltype = select_moltype
    if moltype is None:
        moltype = ffi.NULL
    elif hasattr(moltype, "encode"):
        moltype = moltype.encode("utf-8")
    size = ffi.new("uintptr_t *")
    try:
        if file_like:
            if hasattr(data, "mode") and "t" in data.mode:      # text handle: the bytes underneath
                data = data.buffer
            buf = data.read()
            data.close()
            data = buf
        if is_path:
            arr = rustcall(lib.signatures_load_path, os.fspath(data).encode("utf-8"), ignore_md5sum, int(ksize or 0), moltype, size)
        else:
            buf = data.encode("utf-8") if hasattr(data, "encode") else bytes(data)
            arr = rustcall(lib.signatures_load_buffer, buf, len(buf), ignore_md5sum, int(ksize or 0), moltype, size)
        sigs = [FrozenSourmashSignature._from_objptr(arr[i]) for i in range(size[0])]
        lib.signatures_array_free(arr, size[0])
    except Exception:
        if do_raise:
            raise
        return
    yield from sigs


load_signatures = load_signatures_from_json


def load_one_signature_from_json(data, ksize=None, select_moltype=None, ignore_md5sum=False):
    it = load_signatures_from_json(data, ksize=ksize, select_moltype=select_moltype, ignore_md5sum=ignore_md5sum)
    try:
        first = next(it)
    except StopIteration:
        raise ValueError("no signatures to load")
    try:
        next(it)
    except StopIteration:
        return first
    raise ValueError("expected to load exactly one signature")


def save_signatures_to_json(siglist, fp=None, compression=0):
    """Serialise signatures in the reference's .sig JSON layout (compact, serde field order);
    returns bytes if fp is None, like the reference (signature.py:487-527)."""
    siglist = list(siglist)
    ptrs = ffi.new("SourmashSignature *[]", [sig._get_objptr() for sig in siglist])
    size = ffi.new("uintptr_t *")
    raw = rustcall(lib.signatures_save_buffer, ptrs, len(siglist), int(compression), size)
    try:
        result = bytes(ffi.buffer(raw, size[0]))
    finally:
        lib.nodegraph_buffer_free(raw, size[0])
    if fp is None:
        return result
    try:
        fp.write(result)
    except TypeError:
        fp.write(result.decode("utf-8"))
    return None
