"""MinHash / FrozenMinHash: the sketch object model over the C ABI.

Same public surface and semantics as the reference's ``sourmash.minhash``
(sourmash/src/sourmash/minhash.py:162-1258) so that code written against
``sourmash.MinHash`` runs unchanged; every method is a thin call into
``libsourmash_b200.so`` (include/sourmash_b200.h part 1), where hashing and intersections
execute on the GPU.  Float formulas that the reference evaluates in Python
(bias-corrected containment, minhash.py:819-959) are evaluated here in Python too, in the
same operation order, so results are bit-identical.

Protein / dayhoff / hp sketches hash on the GPU as well (``add_protein`` for residues,
``add_sequence`` for DNA translated in six frames; csrc/aa_kmers.cuh).
"""
from collections.abc import Mapping

import numpy as np

from ._lowlevel import ffi, lib
from ._ffi import RustObject, decode_str, rustcall

MINHASH_DEFAULT_SEED = 42
MINHASH_MAX_HASH = 0xFFFFFFFFFFFFFFFF

__all__ = ["MinHash", "FrozenMinHash", "hash_murmur", "translate_codon", "get_minhash_default_seed", "get_minhash_max_hash",
           "flatten_and_downsample_scaled", "flatten_and_downsample_num", "flatten_and_intersect_scaled"]


def get_minhash_default_seed():
    "Default murmurhash seed (42)."
    return MINHASH_DEFAULT_SEED


def _deprecated(name, details):
    "what the reference's @deprecated decorator does once the version is reached: a DeprecationWarning"
    import warnings
    warnings.warn("%s is deprecated. %s" % (name, details), DeprecationWarning, stacklevel=3)


def get_minhash_max_hash():
    "Largest possible hash value (2**64 - 1)."
    return MINHASH_MAX_HASH


def _get_max_hash_for_scaled(scaled):
    # python-side twin of max_hash_for_scaled (minhash.py:53-60); only used to round-trip scaled
    if scaled == 0:
        return 0
    if scaled == 1:
        return MINHASH_MAX_HASH
    return min(int(round(MINHASH_MAX_HASH / scaled, 0)), MINHASH_MAX_HASH)


def _get_scaled_for_max_hash(max_hash):
    if max_hash == 0:
        return 0
    return min(int(round(MINHASH_MAX_HASH / max_hash, 0)), MINHASH_MAX_HASH)


_RC_TABLE = str.maketrans("ACGTNacgtn", "TGCANtgcan")     # screed.rc equivalent


def to_bytes(s):
    "str / bytes / single int -> bytes"
    if isinstance(s, bytes):
        return s
    if isinstance(s, str):
        return s.encode("utf-8")
    if isinstance(s, int):
        return bytes([s])
    if isinstance(s, (bytearray, memoryview, np.ndarray)):
        return bytes(s)
    raise TypeError("Requires a string-like sequence")


def translate_codon(codon):
    "Translate a codon into an amino acid (minhash.py:96-101)."
    from .exceptions import SourmashError
    try:
        return rustcall(lib.sourmash_translate_codon, to_bytes(codon)).decode("utf-8")
    except SourmashError as e:
        raise ValueError(e.message)


def hash_murmur(kmer, seed=MINHASH_DEFAULT_SEED):
    "murmurhash3_x64_128(kmer, seed) low word, computed by the library (on the GPU)."
    return rustcall(lib.hash_murmur, to_bytes(kmer), seed)


def flatten_and_downsample_scaled(mh, *scaled_vals):
    "Flatten and downsample to the max of the given scaled values."
    assert mh.scaled
    assert all(x > 0 for x in scaled_vals)
    mh = mh.flatten()
    scaled = max(scaled_vals)
    if scaled > mh.scaled:
        return mh.downsample(scaled=scaled)
    return mh


def flatten_and_downsample_num(mh, *num_vals):
    "Flatten and downsample to the min of the given num values."
    assert mh.num
    assert all(x > 0 for x in num_vals)
    mh = mh.flatten()
    num = min(num_vals)
    if num < mh.num:
        return mh.downsample(num=num)
    return mh


def flatten_and_intersect_scaled(mh1, mh2):
    "Flatten + downsample both to the coarser scaled, return the intersection sketch."
    scaled = max(mh1.scaled, mh2.scaled)
    return mh1.flatten().downsample(scaled=scaled) & mh2.flatten().downsample(scaled=scaled)


class _HashesWrapper(Mapping):
    "Read-only {hash: abundance} view returned by MinHash.hashes."

    def __init__(self, h):
        self._data = h

    def __getitem__(self, key):
        return self._data[key]

    def __repr__(self):
        return repr(self._data)

    def __len__(self):
        return len(self._data)

    def __iter__(self):
        return iter(self._data)

    def __eq__(self, other):
        return list(self.items()) == list(other.items())

    def __setitem__(self, k, v):
        raise RuntimeError("cannot modify hashes directly; use 'add' methods")


def _hash_function_for(is_protein, dayhoff, hp):
    if dayhoff:
        return lib.HASH_FUNCTIONS_MURMUR64_DAYHOFF
    if hp:
        return lib.HASH_FUNCTIONS_MURMUR64_HP
    if is_protein:
        return lib.HASH_FUNCTIONS_MURMUR64_PROTEIN
    return lib.HASH_FUNCTIONS_MURMUR64_DNA


class MinHash(RustObject):
    """The core sketch object.

    ``MinHash(n, ksize)`` makes a bottom-``n`` MinHash; ``MinHash(0, ksize, scaled=s)`` makes a
    FracMinHash keeping every hash ``<= 2**64 / s``.

    >>> mh1 = MinHash(n=20, ksize=3)
    >>> mh1.add_sequence('ATGAGAGACGATAGACAGATGAC')            # doctest: +SKIP
    """

    __dealloc_func__ = lib.kmerminhash_free

    def __init__(self, n, ksize, *, is_protein=False, dayhoff=False, hp=False, track_abundance=False,
                 seed=MINHASH_DEFAULT_SEED, max_hash=0, mins=None, scaled=0):
        if max_hash:
            if scaled:
                raise ValueError("cannot set both max_hash and scaled")
            scaled = _get_scaled_for_max_hash(max_hash)
        if scaled and n:
            raise ValueError("cannot set both n and max_hash")
        if not n and not scaled:
            raise ValueError("cannot omit both n and scaled")
        if dayhoff or hp:
            is_protein = False
        hash_function = _hash_function_for(is_protein, dayhoff, hp)
        if hash_function != lib.HASH_FUNCTIONS_MURMUR64_DNA:
            ksize = ksize * 3          # protein-family sketches carry ksize*3 below the ABI
        self._objptr = lib.kmerminhash_new(scaled, ksize, hash_function, seed, track_abundance, n)
        if mins:
            if track_abundance:
                self.set_abundances(mins)
            else:
                self.add_many(mins)

    # ------------------------------------------------------------------ copying / pickling
    def _blank_like(self, *, track_abundance=None, num=None, max_hash=None):
        return MinHash(
            self.num if num is None else num, self.ksize, is_protein=self.is_protein, dayhoff=self.dayhoff,
            hp=self.hp, track_abundance=self.track_abundance if track_abundance is None else track_abundance,
            seed=self.seed, max_hash=self._max_hash if max_hash is None else max_hash)

    def __copy__(self):
        "A new, mutable copy."
        a = self._blank_like()
        a.merge(self)
        return a

    copy = __copy__

    def copy_and_clear(self):
        "An empty sketch with the same parameters."
        return self._blank_like()

    def __getstate__(self):
        return (self.num, self.ksize if self.is_dna else self.ksize * 3, self.is_protein, self.dayhoff,
                self.hp, self.hashes, None, self.track_abundance, self._max_hash, self.seed)

    def __setstate__(self, tup):
        (n, ksize, is_protein, dayhoff, hp, mins, _, track_abundance, max_hash, seed) = tup
        self.__del__()
        self._shared = False
        self._objptr = lib.kmerminhash_new(_get_scaled_for_max_hash(max_hash), ksize,
                                           _hash_function_for(is_protein, dayhoff, hp), seed,
                                           track_abundance, n)
        if track_abundance:
            MinHash.set_abundances(self, mins)      # explicit: self may be a FrozenMinHash
        else:
            MinHash.add_many(self, mins)

    def __eq__(self, other):
        return self.__getstate__() == other.__getstate__()

    # ------------------------------------------------------------------ adding data
    def add_sequence(self, sequence, force=False):
        "Hash all k-mers of a DNA sequence into the sketch (runs on the GPU)."
        self._methodcall(lib.kmerminhash_add_sequence, to_bytes(sequence), force)

    def seq_to_hashes(self, sequence, *, force=False, bad_kmers_as_zeroes=False, is_protein=False):
        "Hashes of the sequence's k-mers in order, without adding them."
        if is_protein and self.moltype not in ("protein", "dayhoff", "hp"):
            raise ValueError("cannot add protein sequence to DNA MinHash")
        if bad_kmers_as_zeroes and not force:
            raise ValueError("cannot represent invalid kmers as 0 while force is not set to True")
        size = ffi.new("uintptr_t *")
        seq = to_bytes(sequence)
        ptr = self._methodcall(lib.kmerminhash_seq_to_hashes, seq, len(seq), force, bad_kmers_as_zeroes,
                               is_protein, size)
        n = size[0]
        try:
            return ffi.unpack(ptr, n)
        finally:
            lib.kmerminhash_slice_free(ptr, n)

    def kmers_and_hashes(self, sequence, *, force=False, is_protein=False):
        """Yield (kmer, hash) for every k-mer without adding them (minhash.py:392-456).
        DNA into a protein-family sketch is translated in six frames; with ``force`` invalid
        k-mers come out with hash None."""
        bad_kmers_as_zeroes = bool(force)
        sequence = (to_bytes(sequence).decode("utf-8") if not isinstance(sequence, str) else sequence).upper()
        hashvals = self.seq_to_hashes(sequence, force=force, is_protein=is_protein,
                                      bad_kmers_as_zeroes=bad_kmers_as_zeroes)
        if bad_kmers_as_zeroes:
            hashvals = [None if h == 0 else h for h in hashvals]
        ksize = self.ksize
        translate = False
        if self.moltype == "DNA" or is_protein:
            pass
        else:                                   # DNA into protein / dayhoff / hp: translate
            translate = True
            ksize = self.ksize * 3
        if translate:
            # forward AND reverse complement => twice the k-mers
            n_kmers = (len(sequence) - ksize + 1) * 2
            assert n_kmers == len(hashvals)
            seqrc = sequence[::-1].translate(_RC_TABLE)
            hash_i = 0
            for frame in (0, 1, 2):
                for strand in (sequence, seqrc):
                    for start in range(0, len(strand) - ksize + 1 - frame, 3):
                        yield strand[start + frame:start + frame + ksize], hashvals[hash_i]
                        hash_i += 1
        else:
            n_kmers = len(sequence) - ksize + 1
            assert n_kmers == len(hashvals)
            for i, hashval in zip(range(0, n_kmers), hashvals):
                yield sequence[i:i + ksize], hashval

    def add_kmer(self, kmer):
        "Add one k-mer."
        want = self.ksize if self.is_dna else self.ksize * 3
        if len(kmer) != want:
            raise ValueError(f"kmer to add is not {want} in length")
        self.add_sequence(kmer)

    def add_many(self, hashes):
        "Add hashes from an iterable or another MinHash."
        if isinstance(hashes, MinHash):
            self._methodcall(lib.kmerminhash_add_from, hashes._get_objptr())
            return
        arr = np.fromiter(hashes, dtype=np.uint64) if not isinstance(hashes, np.ndarray) else \
            np.ascontiguousarray(hashes, dtype=np.uint64)
        self._methodcall(lib.kmerminhash_add_many, ffi.cast("uint64_t *", arr.ctypes.data), len(arr))

    def remove_many(self, hashes):
        "Remove hashes given by an iterable or another MinHash."
        if isinstance(hashes, MinHash):
            self._methodcall(lib.kmerminhash_remove_from, hashes._get_objptr())
            return
        arr = np.fromiter(hashes, dtype=np.uint64) if not isinstance(hashes, np.ndarray) else \
            np.ascontiguousarray(hashes, dtype=np.uint64)
        self._methodcall(lib.kmerminhash_remove_many, ffi.cast("uint64_t *", arr.ctypes.data), len(arr))

    def add_hash(self, h):
        return self._methodcall(lib.kmerminhash_add_hash, h)

    def add_hash_with_abundance(self, h, a):
        if not self.track_abundance:
            raise RuntimeError("Use track_abundance=True when constructing the MinHash to use "
                               "add_hash_with_abundance.")
        return self._methodcall(lib.kmerminhash_add_hash_with_abundance, h, a)

    def add_protein(self, sequence):
        self._methodcall(lib.kmerminhash_add_protein, to_bytes(sequence))

    def clear(self):
        return self._methodcall(lib.kmerminhash_clear)

    def set_abundances(self, values, clear=True):
        "values[hash] = abundance; abundance 0 removes the hash."
        if not self.track_abundance:
            raise RuntimeError("Use track_abundance=True when constructing the MinHash to use set_abundances.")
        hashes, abunds = [], []
        for h, v in values.items():
            if v < 0:
                raise ValueError("Abundance cannot be set to a negative value.")
            hashes.append(h)
            abunds.append(v)
        self._methodcall(lib.kmerminhash_set_abundances, hashes, abunds, len(hashes), clear)

    # ------------------------------------------------------------------ inspection
    def __len__(self):
        return self._methodcall(lib.kmerminhash_get_mins_size)

    def _mins_array(self):
        "Sorted hashes as a numpy uint64 array."
        size = ffi.new("uintptr_t *")
        ptr = self._methodcall(lib.kmerminhash_get_mins, size)
        n = size[0]
        try:
            return np.frombuffer(ffi.buffer(ptr, n * 8), dtype=np.uint64).copy() if n else np.zeros(0, np.uint64)
        finally:
            lib.kmerminhash_slice_free(ptr, n)

    def _abunds_array(self):
        size = ffi.new("uintptr_t *")
        ptr = self._methodcall(lib.kmerminhash_get_abunds, size)
        n = size[0]
        try:
            return np.frombuffer(ffi.buffer(ptr, n * 8), dtype=np.uint64).copy() if n else np.zeros(0, np.uint64)
        finally:
            lib.kmerminhash_slice_free(ptr, n)

    @property
    def hashes(self):
        "{hash: abundance} (abundance 1 for flat sketches), in ascending hash order."
        mins = self._mins_array().tolist()
        if self.track_abundance:
            return _HashesWrapper(dict(zip(mins, self._abunds_array().tolist())))
        return _HashesWrapper({k: 1 for k in mins})

    def get_mins(self, with_abundance=False):
        "Deprecated in the reference (minhash.py:498-511: since 3.5, 'Use .hashes property instead.'); warns like it."
        _deprecated("get_mins", "Use .hashes property instead.")
        return self.hashes if with_abundance else self.hashes.keys()

    def get_hashes(self):
        "Deprecated in the reference (minhash.py:513-521); warns like it."
        _deprecated("get_hashes", "Use .hashes property instead.")
        return self.hashes.keys()

    @property
    def scaled(self):
        "Python-visible scaled = round(2**64 / max_hash) (0 for num sketches)."
        mx = self._max_hash
        return _get_scaled_for_max_hash(mx) if mx else 0

    @property
    def is_dna(self):
        return not (self.is_protein or self.dayhoff or self.hp)

    @property
    def ksize(self):
        "k in residues: protein-family sketches store 3*k below the ABI."
        k = self._methodcall(lib.kmerminhash_ksize)
        if self.is_dna:
            return k
        assert k % 3 == 0
        return k // 3

    @property
    def moltype(self):
        if self.is_protein:
            return "protein"
        if self.dayhoff:
            return "dayhoff"
        if self.hp:
            return "hp"
        return "DNA"

    @property
    def track_abundance(self):
        return self._methodcall(lib.kmerminhash_track_abundance)

    @track_abundance.setter
    def track_abundance(self, b):
        if self.track_abundance == b:
            return
        if b is False:
            self._methodcall(lib.kmerminhash_disable_abundance)
        elif len(self) > 0:
            raise RuntimeError("Can only set track_abundance=True if the MinHash is empty")
        else:
            self._methodcall(lib.kmerminhash_enable_abundance)

    def md5sum(self):
        return decode_str(self._methodcall(lib.kmerminhash_md5sum))

    # ------------------------------------------------------------------ resizing
    def downsample(self, *, num=None, scaled=None):
        "A new sketch downsampled to ``num`` or ``scaled``."
        if num is None and scaled is None:
            raise ValueError("must specify either num or scaled to downsample")
        if num is not None and scaled is not None:
            raise ValueError("cannot specify both num and scaled")
        if num is not None:
            if self.scaled:
                raise ValueError("cannot downsample a scaled MinHash using num")
            if self.num < num:
                raise ValueError("new sample num is higher than current sample num")
            max_hash = 0
        else:
            if self.num:
                raise ValueError("cannot downsample a num MinHash using scaled")
            if self.scaled > scaled:
                raise ValueError(f"new scaled {scaled} is lower than current sample scaled {self.scaled}")
            max_hash = _get_max_hash_for_scaled(scaled)
            num = 0
        a = self._blank_like(num=num, max_hash=max_hash)
        if self.track_abundance:
            a.set_abundances(self.hashes)
        else:
            a.add_many(self)
        return a

    def flatten(self):
        "Drop abundances (returns self if already flat)."
        if not self.track_abundance:
            return self
        a = self._blank_like(track_abundance=False)
        a.add_many(self)
        return a

    # ------------------------------------------------------------------ comparison (GPU)
    def is_compatible(self, other):
        return self._methodcall(lib.kmerminhash_is_compatible, other._get_objptr())

    def count_common(self, other, downsample=False):
        "Number of hashes shared with ``other``."
        if not isinstance(other, MinHash):
            raise TypeError("Must be a MinHash!")
        return self._methodcall(lib.kmerminhash_count_common, other._get_objptr(), downsample)

    def intersection_and_union_size(self, other):
        "(|A ∩ B|, |A ∪ B|)"
        if not isinstance(other, MinHash):
            raise TypeError("Must be a MinHash!")
        if not self.is_compatible(other):
            raise TypeError("incompatible MinHash objects")
        usize = ffi.new("uint64_t *")
        common = self._methodcall(lib.kmerminhash_intersection_union_size, other._get_objptr(), usize)
        return common, usize[0]

    def jaccard(self, other, downsample=False):
        "Jaccard similarity."
        if self.num != other.num:
            raise TypeError(f"must have same num: {self.num} != {other.num}")          # minhash.py:742-744
        return self._methodcall(lib.kmerminhash_similarity, other._get_objptr(), True, downsample)

    def similarity(self, other, ignore_abundance=False, downsample=False):
        "Angular similarity if both track abundance (and not ignored), else Jaccard (no num check here: minhash.py:787-806)."
        return self._methodcall(lib.kmerminhash_similarity, other._get_objptr(), ignore_abundance, downsample)

    def angular_similarity(self, other):
        if not (self.track_abundance and other.track_abundance):
            raise TypeError("Error: Angular (cosine) similarity requires both sketches to track hash abundance.")
        return self._methodcall(lib.kmerminhash_angular_similarity, other._get_objptr())

    def contained_by(self, other, downsample=False):
        "Bias-corrected containment of self in other (float math as in minhash.py:819-841)."
        if not (self.scaled and other.scaled):
            raise TypeError("Error: can only calculate containment for scaled MinHashes")
        denom = len(self)
        if not denom:
            return 0.0
        total_denom = float(denom * self.scaled)
        bias_factor = 1.0 - (1.0 - 1.0 / self.scaled) ** total_denom
        containment = self.count_common(other, downsample) / (denom * bias_factor)
        if containment >= 1:
            return 1.0
        if containment <= 0:
            return 0.0
        return containment

    def max_containment(self, other, downsample=False):
        "Containment relative to the smaller sketch (minhash.py:881-905)."
        if not (self.scaled and other.scaled):
            raise TypeError("Error: can only calculate containment for scaled MinHashes")
        min_denom = min((len(self), len(other)))
        if not min_denom:
            return 0.0
        total_denom = float(min_denom * self.scaled)
        bias_factor = 1.0 - (1.0 - 1.0 / self.scaled) ** total_denom
        c = self.count_common(other, downsample) / (min_denom * bias_factor)
        if c >= 1:
            return 1.0
        if c <= 0:
            return 0.0
        return c

    def avg_containment(self, other, *, downsample=False):
        "Mean of the two containments (minhash.py:946-959)."
        if not (self.scaled and other.scaled):
            raise TypeError("Error: can only calculate containment for scaled MinHashes")
        return (self.contained_by(other, downsample) + other.contained_by(self, downsample)) / 2

    # ------------------------------------------------------------------ set algebra
    def merge(self, other):
        if not isinstance(other, MinHash):
            raise TypeError("can only add MinHash objects to MinHash objects!")
        self._methodcall(lib.kmerminhash_merge, other._get_objptr())

    def __iadd__(self, other):
        self.merge(other)
        return self

    def __add__(self, other):
        if not isinstance(other, MinHash):
            raise TypeError("can only add MinHash objects to MinHash objects!")
        if self.num and other.num and self.num != other.num:
            raise TypeError(f"incompatible num values: self={self.num} other={other.num}")
        new_obj = self.to_mutable()
        new_obj += other
        return new_obj

    __or__ = __add__

    def intersection(self, other):
        "New sketch holding the common hashes (flat sketches only)."
        if not isinstance(other, MinHash):
            raise TypeError("can only intersect MinHash objects")
        if self.track_abundance or other.track_abundance:
            raise TypeError("can only intersect flat MinHash objects")
        return MinHash._from_objptr(self._methodcall(lib.kmerminhash_intersection, other._get_objptr()))

    __and__ = intersection

    def inflate(self, from_mh):
        "Flat self + abundances looked up in from_mh (hashes absent there are dropped)."
        if self.track_abundance or not from_mh.track_abundance:
            raise ValueError("inflate operates on a flat MinHash and takes a MinHash object with "
                             "track_abundance=True")
        orig = from_mh.hashes
        abund_mh = from_mh.copy_and_clear()
        abund_mh.set_abundances({h: orig.get(h, 0) for h in self.hashes})
        return abund_mh

    # ------------------------------------------------------------------ mutability
    def to_mutable(self):
        return self.__copy__()

    def to_frozen(self):
        new_mh = self.__copy__()
        new_mh.into_frozen()
        return new_mh

    def into_frozen(self):
        self.__class__ = FrozenMinHash

    # ------------------------------------------------------------------ abundance statistics
    @property
    def sum_abundances(self):
        return sum(self.hashes.values()) if self.track_abundance else None

    @property
    def mean_abundance(self):
        return np.mean(list(self.hashes.values())) if self.track_abundance else None

    @property
    def median_abundance(self):
        return np.median(list(self.hashes.values())) if self.track_abundance else None

    @property
    def std_abundance(self):
        return np.std(list(self.hashes.values())) if self.track_abundance else None

    @property
    def unique_dataset_hashes(self):
        if not self.scaled:
            raise TypeError("can only approximate unique_dataset_hashes for scaled MinHashes")
        return len(self) * self.scaled

    def size_is_accurate(self, relative_error=0.20, confidence=0.95):
        """True if len(self) * scaled is, with probability >= confidence, within relative_error
        of the true number of distinct k-mers (minhash.py:1129-1150)."""
        from .distance_utils import set_size_exact_prob
        if not self.scaled:
            raise TypeError("Error: can only estimate dataset size for scaled MinHashes")
        if not (0 <= relative_error <= 1) or not (0 <= confidence <= 1):
            raise ValueError("Error: relative error and confidence values must be between 0 and 1.")
        return set_size_exact_prob(self.unique_dataset_hashes, self.scaled, relative_error=relative_error) >= confidence

    def inflate(self, from_mh):
        """New sketch holding self's hashes with the abundances they have in ``from_mh``
        (hashes absent there are dropped; minhash.py:1071-1092)."""
        if self.track_abundance or not from_mh.track_abundance:
            raise ValueError("inflate operates on a flat MinHash and takes a MinHash object with track_abundance=True")
        orig = from_mh.hashes
        abund_mh = from_mh.copy_and_clear()
        abund_mh.downsample(scaled=self.scaled)
        abund_mh.set_abundances({h: orig.get(h, 0) for h in self.hashes})
        return abund_mh

    # ------------------------------------------------------------------ ANI (minhash.py:749-976)
    def _ani_operands(self, other, downsample):
        if not (self.scaled and other.scaled):
            raise TypeError("Error: can only calculate ANI for scaled MinHashes")
        a, b, scaled = self, other, self.scaled
        if downsample:
            scaled = max(a.scaled, b.scaled)
            a, b = a.downsample(scaled=scaled), b.downsample(scaled=scaled)
        return a, b, scaled

    def jaccard_ani(self, other, *, downsample=False, jaccard=None, prob_threshold=1e-3, err_threshold=1e-4):
        "ANI estimated from the Jaccard similarity of two scaled sketches."
        from .distance_utils import jaccard_to_distance
        a, b, scaled = self._ani_operands(other, downsample)
        if jaccard is None:
            jaccard = a.similarity(b, ignore_abundance=True)
        avg_n_kmers = round((len(a) + len(b)) / 2 * scaled)
        res = jaccard_to_distance(jaccard, a.ksize, scaled, n_unique_kmers=avg_n_kmers,
                                  prob_threshold=prob_threshold, err_threshold=err_threshold)
        if not self.size_is_accurate() or not other.size_is_accurate():
            res.size_is_inaccurate = True
        return res

    def containment_ani(self, other, *, downsample=False, containment=None, confidence=0.95, estimate_ci=False,
                        prob_threshold=1e-3):
        "ANI estimated from the containment of self in other."
        from .distance_utils import containment_to_distance
        a, b, scaled = self._ani_operands(other, downsample)
        if containment is None:
            containment = a.contained_by(b)
        res = containment_to_distance(containment, a.ksize, a.scaled, n_unique_kmers=len(a) * scaled,
                                      confidence=confidence, estimate_ci=estimate_ci, prob_threshold=prob_threshold)
        if not self.size_is_accurate() or not other.size_is_accurate():
            res.size_is_inaccurate = True
        return res

    def max_containment_ani(self, other, *, downsample=False, max_containment=None, confidence=0.95,
                            estimate_ci=False, prob_threshold=1e-3):
        "ANI estimated from the containment relative to the smaller sketch."
        from .distance_utils import containment_to_distance
        a, b, scaled = self._ani_operands(other, downsample)
        if max_containment is None:
            max_containment = a.max_containment(b)
        res = containment_to_distance(max_containment, a.ksize, scaled, n_unique_kmers=min(len(a), len(b)) * scaled,
                                      confidence=confidence, estimate_ci=estimate_ci, prob_threshold=prob_threshold)
        if not self.size_is_accurate() or not other.size_is_accurate():
            res.size_is_inaccurate = True
        return res

    def avg_containment_ani(self, other, *, downsample=False, prob_threshold=1e-3):
        "Mean of the two containment ANIs (None if either is not trustworthy)."
        if not (self.scaled and other.scaled):
            raise TypeError("Error: can only calculate ANI for scaled MinHashes")
        a1 = self.containment_ani(other, downsample=downsample, prob_threshold=prob_threshold).ani
        a2 = other.containment_ani(self, downsample=downsample, prob_threshold=prob_threshold).ani
        if a1 is None or a2 is None:
            return None
        return (a1 + a2) / 2


def _scalar_getter(c_function, doc):
    return property(lambda self: self._methodcall(c_function), doc=doc)


# plain scalar attributes: one C getter each (ffi/minhash.rs:303-378)
for _name, _cfn, _doc in (
        ("seed", lib.kmerminhash_seed, "murmurhash seed"),
        ("num", lib.kmerminhash_num, "bottom-k size (0 for scaled sketches)"),
        ("is_protein", lib.kmerminhash_is_protein, "protein k-mers"),
        ("dayhoff", lib.kmerminhash_dayhoff, "dayhoff-encoded protein k-mers"),
        ("hp", lib.kmerminhash_hp, "hydrophobic/polar-encoded protein k-mers"),
        ("max_hash", lib.kmerminhash_max_hash, "largest retained hash (deprecated alias of _max_hash)"),
        ("_max_hash", lib.kmerminhash_max_hash, "largest retained hash; 0 for num sketches")):
    setattr(MinHash, _name, _scalar_getter(_cfn, _doc))
del _name, _cfn, _doc


def _frozen(name):
    def method(self, *args, **kwargs):
        raise TypeError("FrozenMinHash does not support modification")
    method.__name__ = name
    return method


class FrozenMinHash(MinHash):
    "Read-only MinHash: every mutating method raises TypeError."

    add_sequence = _frozen("add_sequence")
    add_kmer = _frozen("add_kmer")
    add_many = _frozen("add_many")
    remove_many = _frozen("remove_many")
    add_hash = _frozen("add_hash")
    add_hash_with_abundance = _frozen("add_hash_with_abundance")
    clear = _frozen("clear")
    set_abundances = _frozen("set_abundances")
    add_protein = _frozen("add_protein")
    __iadd__ = _frozen("__iadd__")
    merge = _frozen("merge")

    def downsample(self, *, num=None, scaled=None):
        if num and self.num == num:
            return self
        if scaled and self.scaled == scaled:
            return self
        down = MinHash.downsample(self, num=num, scaled=scaled)
        down.into_frozen()
        return down

    def flatten(self):
        if not self.track_abundance:
            return self
        flat = MinHash.flatten(self)
        flat.into_frozen()
        return flat

    def to_mutable(self):
        mut = MinHash.__new__(MinHash)
        MinHash.__setstate__(mut, self.__getstate__())
        return mut

    def to_frozen(self):
        return self

    def into_frozen(self):
        pass

    def __setstate__(self, tup):
        MinHash.__setstate__(self, tup)
        self.into_frozen()

    def __copy__(self):
        return self

    copy = __copy__
