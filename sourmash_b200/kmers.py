"""The k-mers and records that carry a sketch's hashes (`sourmash sig kmers`), hashed and matched on the GPU.

The reference walks the records one at a time (src/sourmash/sig/__main__.py:1206-1256): a fresh sketch per record,
``add_sequence`` / ``add_protein``, ``intersection`` with the merged query, then ``kmers_and_hashes`` and a set lookup
per k-mer of every matching record.  ``match_records`` does all records of a ``sketch.RecordBatch`` in one library call
(``smb_kmer_match_records``): every window hashed and probed against the query on the device, the matches sorted into
file order.  K-mer strings are built on the host, for the matches only (``kmer_strings``).
"""
from dataclasses import dataclass

import numpy as np

from . import batch as B
from ._ffi import rustcall
from ._lowlevel import ffi, lib
from .minhash import _RC_TABLE


@dataclass
class KmerMatches:
    """Matches in file order (record, then the window's index in ``seq_to_hashes`` order), and per-record results.

    ``matched[r]``: ``seq_mh.intersection(query_mh)`` is not empty for record r.  ``has_invalid[r]``: a DNA window of
    record r holds a non-ACGT base (``add_sequence(seq, force=False)`` raises).  ``found``: the sorted query hashes of
    ``found_mh += seq_mh.intersection(query_mh)`` over the matched records (not skipped ones)."""
    records: np.ndarray
    ordinals: np.ndarray
    hashes: np.ndarray
    matched: np.ndarray
    has_invalid: np.ndarray
    found: np.ndarray


def _array(ptr, n, dtype):
    if not n:
        return np.zeros(0, dtype)
    return np.frombuffer(ffi.buffer(ptr, n * np.dtype(dtype).itemsize), dtype=dtype).copy()


def match_records(query_mh, records, *, is_protein=False, skip_invalid=False):
    """Match every window of every record of ``records`` (a ``sketch.RecordBatch``) against ``query_mh``.

    ``is_protein``: the records are residues (``add_protein``); otherwise DNA, translated in six frames for a
    protein-family sketch.  ``skip_invalid``: records with ``has_invalid`` add nothing to ``found`` (what
    ``sig kmers --check-sequence --force`` does with them).  Returns ``KmerMatches``."""
    hf = B._HASH_FUNCTIONS[query_mh.moltype.lower()]
    if is_protein and hf == 1:
        raise ValueError("cannot add protein sequence to DNA MinHash")
    ksize = query_mh.ksize * (1 if hf == 1 else 3)
    q = np.ascontiguousarray(query_mh._mins_array(), dtype=np.uint64)
    p = rustcall(lib.smb_kmer_match_records, records._ptr, ffi.cast("uint64_t *", q.ctypes.data), len(q), ksize, hf,
                 int(query_mh.seed), int(query_mh._max_hash), int(query_mh.num), bool(is_protein),
                 bool(skip_invalid))
    try:
        m = int(lib.smb_kmer_matches_len(p))
        n = len(records)
        keys = _array(lib.smb_kmer_matches_keys(p), m, np.uint64)
        return KmerMatches(records=(keys >> np.uint64(32)).astype(np.int64),
                           ordinals=(keys & np.uint64(0xffffffff)).astype(np.int64),
                           hashes=_array(lib.smb_kmer_matches_hashes(p), m, np.uint64),
                           matched=_array(lib.smb_kmer_matches_matched(p), n, np.uint8).astype(bool),
                           has_invalid=_array(lib.smb_kmer_matches_has_invalid(p), n, np.uint8).astype(bool),
                           found=_array(lib.smb_kmer_matches_found(p), int(lib.smb_kmer_matches_n_found(p)), np.uint64))
    finally:
        lib.smb_kmer_matches_free(p)


def kmer_strings(query_mh, sequence, ordinals, *, is_protein=False):
    """The k-mers of ``sequence`` (str) at the given ordinals, as ``kmers_and_hashes`` yields them: slices of the
    upper-cased sequence; for translated input the forward or reverse-complement slice of 3k bases."""
    seq = sequence.upper()
    k = query_mh.ksize
    if query_mh.moltype == "DNA" or is_protein:
        return [seq[o:o + k] for o in ordinals]
    span = 3 * k
    L = len(seq)
    nwin = [max((L - f) // 3 - k + 1, 0) if L >= f else 0 for f in range(3)]
    bases = [0, 2 * nwin[0], 2 * (nwin[0] + nwin[1])]
    rc = None
    out = []
    for o in ordinals:
        f = 2 if o >= bases[2] else 1 if o >= bases[1] else 0
        i = o - bases[f]
        reverse = i >= nwin[f]
        start = f + 3 * (i - nwin[f] if reverse else i)
        if not reverse:
            out.append(seq[start:start + span])
        else:
            if rc is None:
                rc = seq[::-1].translate(_RC_TABLE)
            out.append(rc[start:start + span])
    return out
