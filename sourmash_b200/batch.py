"""Batched GPU entry points: the Python face of Part 2 of include/sourmash_b200.h.

These replace the reference's per-record / per-pair Python loops
(command_sketch.py:662-789, compare.py:14-187, index/__init__.py:115-170,777-909) with one
C-ABI call per batch.  Arrays are numpy on the host side; ``SketchSet`` keeps the sketches
resident in HBM between calls.
"""
import numpy as np

from ._lowlevel import ffi, lib
from ._ffi import rustcall


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _ptr(a, ctype):
    return ffi.cast(ctype, a.ctypes.data) if a is not None and a.size else ffi.cast(ctype, 0)


def device_count():
    return int(lib.smb_device_count())


def device_probe_error():
    "What cudaGetDeviceCount said when no device was found ('' when the probe succeeded)."
    return ffi.string(lib.smb_device_probe_error()).decode(errors="replace")


def set_device(i):
    lib.smb_set_device(int(i))


def set_stream(cuda_stream_handle):
    """Run subsequent library work on this cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream)."""
    lib.smb_set_stream(ffi.cast("void *", int(cuda_stream_handle)))


def synchronize():
    rustcall(lib.smb_synchronize)


def kernel_launches():
    return int(lib.smb_kernel_launches())


def set_profiling(on):
    lib.smb_set_profiling(bool(on))


def last_kernel_ms(which):
    """CUDA-event duration of the last pairwise tile kernel (0) / hash pass (1); -1 if none."""
    return float(rustcall(lib.smb_last_kernel_ms, int(which)))


def last_compare_plan():
    "Planner decision of the last all-vs-all count: dict(algo, est_increments, est_elements, max_group)."
    out = ffi.new("double[4]")
    lib.smb_last_compare_plan(out)
    return {"algo": "join" if out[0] else "tile", "est_increments": out[1], "est_elements": out[2],
            "max_group": int(out[3])}


def max_hash_for_scaled(scaled):
    return int(lib.smb_max_hash_for_scaled(int(scaled)))


class PinnedArray:
    """numpy view of page-locked host memory (for end-to-end transfers)."""

    def __init__(self, shape, dtype):
        self.dtype = np.dtype(dtype)
        self.shape = tuple(int(x) for x in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        nbytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize
        self._ptr = rustcall(lib.smb_alloc_pinned, max(nbytes, 16))
        buf = ffi.buffer(self._ptr, max(nbytes, 16))
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape, dtype=np.int64))).reshape(self.shape)

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p is not None and lib is not None:
            self.array = None
            lib.smb_free_pinned(p)


def pinned_empty(shape, dtype):
    return PinnedArray(shape, dtype)


class SketchSet:
    """CSR set of sorted-unique u64 sketches resident on the GPU."""

    def __init__(self, ptr, keepalive=None):
        self._ptr = ptr
        self._keepalive = keepalive

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:                    # lib is None during interpreter shutdown
            lib.smb_sketchset_free(p)

    @classmethod
    def from_host(cls, hashes, offsets, abunds=None):
        hashes, offsets = _u64(hashes), _u64(offsets)
        ab = _u64(abunds) if abunds is not None else None
        n = len(offsets) - 1
        p = rustcall(lib.smb_sketchset_from_host, _ptr(hashes, "uint64_t *"), _ptr(offsets, "uint64_t *"),
                     n, _ptr(ab, "uint64_t *") if ab is not None else ffi.NULL)
        return cls(p)

    @classmethod
    def from_rows(cls, rows, abund_rows=None):
        offsets = np.zeros(len(rows) + 1, dtype=np.uint64)
        if len(rows):
            offsets[1:] = np.cumsum([len(r) for r in rows])
        hashes = np.concatenate([_u64(r) for r in rows]) if len(rows) else np.zeros(0, np.uint64)
        ab = None
        if abund_rows is not None:
            ab = np.concatenate([_u64(r) for r in abund_rows]) if len(rows) else np.zeros(0, np.uint64)
        return cls.from_host(hashes, offsets, ab)

    @classmethod
    def from_device(cls, d_hashes_ptr, d_offsets_ptr, h_offsets, keepalive=None):
        h_offsets = _u64(h_offsets)
        p = rustcall(lib.smb_sketchset_from_device, ffi.cast("uint64_t *", int(d_hashes_ptr)),
                     ffi.cast("uint64_t *", int(d_offsets_ptr)), _ptr(h_offsets, "uint64_t *"),
                     len(h_offsets) - 1)
        return cls(p, keepalive=keepalive)

    def __len__(self):
        return int(lib.smb_sketchset_len(self._ptr))

    @property
    def total_hashes(self):
        return int(lib.smb_sketchset_total_hashes(self._ptr))

    @property
    def has_abunds(self):
        return bool(lib.smb_sketchset_has_abunds(self._ptr))

    def offsets(self):
        out = np.zeros(len(self) + 1, dtype=np.uint64)
        lib.smb_sketchset_offsets(self._ptr, _ptr(out, "uint64_t *"))
        return out

    def sizes(self):
        return np.diff(self.offsets().astype(np.int64))

    def to_host(self, with_abunds=False):
        off = self.offsets()
        h = np.zeros(int(off[-1]), dtype=np.uint64)
        ab = np.zeros(int(off[-1]), dtype=np.uint64) if (with_abunds and self.has_abunds) else None
        rustcall(lib.smb_sketchset_to_host, self._ptr, _ptr(h, "uint64_t *"),
                 _ptr(ab, "uint64_t *") if ab is not None else ffi.NULL)
        return (h, off, ab) if with_abunds else (h, off)

    def rows(self):
        h, off = self.to_host()
        return [h[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]

    def build_index(self):
        """Build the inverted index (hash -> rows) of this resident set; search / prefetch / gather
        counts on it then cost work proportional to the query instead of a pass over the set.
        Returns the number of distinct hashes."""
        return int(rustcall(lib.smb_sketchset_build_index, self._ptr))

    def drop_index(self):
        rustcall(lib.smb_sketchset_drop_index, self._ptr)

    @property
    def has_index(self):
        return bool(lib.smb_sketchset_has_index(self._ptr))

    def downsample(self, max_hash):
        return SketchSet(rustcall(lib.smb_sketchset_downsample, self._ptr, int(max_hash)))

    def take_rows(self, rows):
        "The given rows (any order) as a new resident SketchSet."
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        return SketchSet(rustcall(lib.smb_sketchset_take_rows, self._ptr, _ptr(rows, "uint32_t *"), len(rows)))

    def copy_to_device(self, d_hashes_ptr, d_offsets_ptr=0):
        rustcall(lib.smb_sketchset_copy_to_device, self._ptr, ffi.cast("uint64_t *", int(d_hashes_ptr)),
                 ffi.cast("uint64_t *", int(d_offsets_ptr)))

    def device_pointers(self):
        return (int(ffi.cast("uintptr_t", lib.smb_sketchset_device_hashes(self._ptr))),
                int(ffi.cast("uintptr_t", lib.smb_sketchset_device_offsets(self._ptr))))


_HASH_FUNCTIONS = {"dna": 1, "protein": 2, "dayhoff": 3, "hp": 4}


def sketch_sequences(seqs, seq_offsets, ksizes, scaled=0, num=0, seed=42, track_abundance=False,
                     seq_to_sketch=None, n_sketches=None, moltype="DNA", input_is_protein=False):
    """Sketch a batch of records.  Returns (SketchSet, n_kmers); row = sketch * len(ksizes) + k_index.

    ``moltype`` "protein" / "dayhoff" / "hp" builds protein-family sketches (ksizes in residues):
    from residues when ``input_is_protein`` (sketch protein), else from DNA translated in six
    frames (sketch translate)."""
    if isinstance(seqs, (bytes, bytearray)):
        seqs = np.frombuffer(seqs, dtype=np.uint8)
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    seq_offsets = _u64(seq_offsets)
    ks = np.ascontiguousarray(ksizes, dtype=np.uint32)
    n_seqs = len(seq_offsets) - 1
    s2s = None
    if seq_to_sketch is not None:
        s2s = np.ascontiguousarray(seq_to_sketch, dtype=np.uint32)
        if n_sketches is None:
            n_sketches = int(s2s.max()) + 1 if len(s2s) else 0
    else:
        n_sketches = n_seqs
    nk = ffi.new("uint64_t *")
    hf = _HASH_FUNCTIONS[moltype.lower()]
    if hf != 1:
        ks = np.ascontiguousarray(ks * np.uint32(3))           # ABI ksize of protein-family sketches
        p = rustcall(lib.smb_sketch_sequences_aa, _ptr(seqs, "uint8_t *"), _ptr(seq_offsets, "uint64_t *"), n_seqs,
                     _ptr(s2s, "uint32_t *") if s2s is not None else ffi.NULL, n_sketches,
                     _ptr(ks, "uint32_t *"), len(ks), hf, bool(input_is_protein), int(scaled), int(num),
                     int(seed), bool(track_abundance), nk)
        return SketchSet(p), int(nk[0])
    if input_is_protein:
        raise ValueError("cannot add protein sequence to DNA MinHash")
    p = rustcall(lib.smb_sketch_sequences, _ptr(seqs, "uint8_t *"), _ptr(seq_offsets, "uint64_t *"), n_seqs,
                 _ptr(s2s, "uint32_t *") if s2s is not None else ffi.NULL, n_sketches,
                 _ptr(ks, "uint32_t *"), len(ks), int(scaled), int(num), int(seed), bool(track_abundance), nk)
    return SketchSet(p), int(nk[0])


def sketch_streams_device(d_bases_ptr, stream_offsets, stream_lens, ksizes, scaled=0, num=0, seed=42,
                          track_abundance=False):
    """Sketch streams that already live in HBM (device pointer as int)."""
    so, sl = _u64(stream_offsets), _u64(stream_lens)
    ks = np.ascontiguousarray(ksizes, dtype=np.uint32)
    nk = ffi.new("uint64_t *")
    p = rustcall(lib.smb_sketch_streams_dev, ffi.cast("uint8_t *", int(d_bases_ptr)), _ptr(so, "uint64_t *"),
                 _ptr(sl, "uint64_t *"), len(so), _ptr(ks, "uint32_t *"), len(ks), int(scaled), int(num),
                 int(seed), bool(track_abundance), nk)
    return SketchSet(p), int(nk[0])


def pairwise_common(a, b=None, num=0, want_usize=False):
    """(n_a, n_b) uint32 matrix of |A_i ∩ B_j| (b None: all-vs-all of a)."""
    na, nb = len(a), len(b) if b is not None else len(a)
    out = np.zeros((na, nb), dtype=np.uint32)
    us = np.zeros((na, nb), dtype=np.uint32) if (num and want_usize) else None
    rustcall(lib.smb_pairwise_common, a._ptr, b._ptr if b is not None else ffi.NULL, int(num),
             _ptr(out, "uint32_t *"), _ptr(us, "uint32_t *") if us is not None else ffi.NULL)
    return (out, us) if want_usize else out


def compare_jaccard(sset, num=0, out=None):
    """float64 (n, n) Jaccard matrix with ones on the diagonal (compare_serial's contract)."""
    n = len(sset)
    if out is None:
        out = np.empty((n, n), dtype=np.float64)
    assert out.dtype == np.float64 and out.shape == (n, n) and out.flags.c_contiguous
    rustcall(lib.smb_compare_jaccard, sset._ptr, int(num), _ptr(out, "double *"))
    return out


def compare_angular(sset, out=None):
    """float64 (n, n) angular-similarity matrix of a SketchSet that carries abundances."""
    n = len(sset)
    if out is None:
        out = np.empty((n, n), dtype=np.float64)
    rustcall(lib.smb_compare_angular, sset._ptr, _ptr(out, "double *"))
    return out


def compare_jaccard_device(sset, d_out_ptr, num=0):
    rustcall(lib.smb_compare_jaccard_dev, sset._ptr, int(num), ffi.cast("double *", int(d_out_ptr)))


def pairwise_counts_shard_device(sset, shard, n_shards, d_common_ptr):
    rustcall(lib.smb_pairwise_counts_shard_dev, sset._ptr, int(shard), int(n_shards),
             ffi.cast("uint32_t *", int(d_common_ptr)))


def compare_counts_shard_device(sset, shard, n_shards, d_counts_ptr, bits=32):
    "Partial counters of shard `shard` as whole rows (n*n counters of `bits` bits, device): they add up over the shards (see the header)."
    rustcall(lib.smb_compare_counts_shard_dev, sset._ptr, int(shard), int(n_shards), ffi.cast("void *", int(d_counts_ptr)), int(bits))


def finalize_counts_rows_device(sset, d_counts_rows_ptr, row_begin, row_end, d_out_ptr, bits=32):
    "Summed whole-row counters of rows [row_begin, row_end) -> float64 Jaccard rows (device memory)."
    rustcall(lib.smb_finalize_counts_rows_dev, sset._ptr, ffi.cast("void *", int(d_counts_rows_ptr)), int(bits), int(row_begin),
             int(row_end), ffi.cast("double *", int(d_out_ptr)))


def finalize_jaccard_rows_device(sset, d_common_ptr, row_begin, row_end, d_out_ptr):
    rustcall(lib.smb_finalize_jaccard_rows_dev, sset._ptr, ffi.cast("uint32_t *", int(d_common_ptr)),
             int(row_begin), int(row_end), ffi.cast("double *", int(d_out_ptr)))


def compare_jaccard_rows_device(sset, row_begin, row_end, d_out_ptr):
    "Rows [row_begin, row_end) of the all-vs-all Jaccard matrix into device memory (see the header)."
    rustcall(lib.smb_compare_jaccard_rows_dev, sset._ptr, int(row_begin), int(row_end),
             ffi.cast("double *", int(d_out_ptr)))


def one_vs_many(query, db):
    q = _u64(query)
    out = np.zeros(len(db), dtype=np.uint32)
    rustcall(lib.smb_one_vs_many, _ptr(q, "uint64_t *"), len(q), db._ptr, _ptr(out, "uint32_t *"))
    return out


def one_vs_many_device(d_query_ptr, n_query, db, d_counts_ptr):
    "|query ∩ row| for every row, query (sorted u64) and the u32 counters resident in device memory."
    rustcall(lib.smb_one_vs_many_dev, ffi.cast("uint64_t *", int(d_query_ptr)), int(n_query), db._ptr,
             ffi.cast("uint32_t *", int(d_counts_ptr)))


def query_covered(query, db, rows):
    """Boolean mask over ``query`` (sorted-unique u64, at the set's scaled): True where some row ``rows[i]`` of ``db``
    holds the hash.  ``query[mask]`` is the union of the rows' intersections with the query (prefetch's matched hashes),
    ``query[~mask]`` the rest.  The rows are probed in place on the device; a row may be listed twice."""
    q = _u64(query)
    r = np.asarray(rows, dtype=np.int64).ravel()
    if len(r) and (r.min() < 0 or r.max() > 0xFFFFFFFF):              # would wrap as uint32; the library checks the rest
        raise ValueError(f"row index {int(r[(r < 0) | (r > 0xFFFFFFFF)][0])} out of range for a set of {len(db)} rows")
    r = np.ascontiguousarray(r, dtype=np.uint32)
    out = np.zeros(len(q), dtype=np.uint8)
    rustcall(lib.smb_query_covered, _ptr(q, "uint64_t *"), len(q), db._ptr, _ptr(r, "uint32_t *"), len(r),
             _ptr(out, "uint8_t *"))
    return out.view(np.bool_)


def search_angular(q_hashes, q_abunds, sset, max_hash):
    """Angular similarity of one abundance query (sorted-unique ``q_hashes``, ``q_abunds``) with every row of ``sset``
    (which must carry abundances), over the hashes <= ``max_hash`` of both sides: a float64 ``(len(sset),)`` array,
    bit for bit what ``similarity(..., downsample=True)`` gives for each row when ``max_hash`` is the coarser side's
    (``2**64 - 1``: every hash)."""
    q, qa = _u64(q_hashes), _u64(q_abunds)
    if len(q) != len(qa):
        raise ValueError("query hashes and abundances differ in length")
    out = np.zeros(len(sset), dtype=np.float64)
    rustcall(lib.smb_search_angular, sset._ptr, _ptr(q, "uint64_t *"), _ptr(qa, "uint64_t *"), len(q), int(max_hash),
             _ptr(out, "double *"))
    return out


def _query_csr(queries):
    "(hashes, offsets) of a list of sorted-unique u64 queries"
    qs = [_u64(q) for q in queries]
    offs = np.zeros(len(qs) + 1, dtype=np.uint64)
    if qs:
        offs[1:] = np.cumsum([len(q) for q in qs])
    return (np.concatenate(qs) if qs else np.zeros(0, np.uint64)), offs


def many_vs_many(queries, db):
    """|query ∩ row| for every query (sorted-unique u64 arrays) and every row of ``db``: a (len(queries), len(db))
    uint32 array equal to ``np.stack([one_vs_many(q, db) for q in queries])``.  Groups of queries share one pass over
    the database on the device instead of one pass per query."""
    hashes, offs = _query_csr(queries)
    n = len(offs) - 1
    out = np.zeros((n, len(db)), dtype=np.uint32)
    rustcall(lib.smb_many_vs_many, _ptr(hashes, "uint64_t *"), _ptr(offs, "uint64_t *"), n, db._ptr,
             _ptr(out, "uint32_t *"))
    return out


def many_vs_many_device(d_hashes_ptr, offsets, db, d_counts_ptr):
    """many_vs_many with the queries' hashes and the (Q, len(db)) u32 counters in device memory; ``offsets`` (Q + 1,
    host) delimit the queries inside the hashes."""
    offs = np.ascontiguousarray(offsets, dtype=np.uint64)
    rustcall(lib.smb_many_vs_many_dev, ffi.cast("uint64_t *", int(d_hashes_ptr)), _ptr(offs, "uint64_t *"),
             len(offs) - 1, db._ptr, ffi.cast("uint32_t *", int(d_counts_ptr)))


COMBINE_OPS = {"union": 0, "all": 1, "first_only": 2}


def combine(sset, op, num=0):
    """Union ("union"), intersection ("all") or difference ("first_only": row 0 minus every other row) of all rows of
    ``sset`` in one device sort.  Returns ``(hashes, abunds)`` as uint64 arrays in hash order; ``abunds`` holds each
    hash's summed abundances for a union of a set with abundances, else None.  ``num`` > 0 keeps the union's first
    ``num`` hashes, as merging into a num sketch does."""
    code = COMBINE_OPS[op] if isinstance(op, str) else int(op)
    p = rustcall(lib.smb_sketchset_combine, sset._ptr, code, int(num))
    try:
        n = int(lib.smb_combined_len(p))
        h = np.frombuffer(ffi.buffer(lib.smb_combined_hashes(p), n * 8), dtype=np.uint64).copy() if n else \
            np.zeros(0, np.uint64)
        a = None
        if code == 0 and sset.has_abunds:
            a = np.frombuffer(ffi.buffer(lib.smb_combined_abunds(p), n * 8), dtype=np.uint64).copy() if n else \
                np.zeros(0, np.uint64)
        return h, a
    finally:
        lib.smb_combined_free(p)


LCA_NO_NODE = 0xFFFFFFFF


def lca_parse_hashvals(text):
    """The "hashval_to_idx" member of an LCA database's JSON text (bytes), parsed natively: ``(hashes, idx, span)``,
    one uint64 hash and one uint32 idx per listed idx in file order, and the byte span ``(begin, end)`` of the member's
    value (``(-1, -1)`` when the document has none).  Raises on malformed JSON inside the member."""
    buf = ffi.from_buffer(text)
    p = rustcall(lib.smb_lca_parse_hashvals, buf, len(text))
    try:
        n = int(lib.smb_lca_hashvals_len(p))
        h = np.frombuffer(ffi.buffer(lib.smb_lca_hashvals_hashes(p), n * 8), dtype=np.uint64).copy() if n else \
            np.zeros(0, np.uint64)
        ix = np.frombuffer(ffi.buffer(lib.smb_lca_hashvals_idx(p), n * 4), dtype=np.uint32).copy() if n else \
            np.zeros(0, np.uint32)
        b, e = ffi.new("int64_t *"), ffi.new("int64_t *")
        lib.smb_lca_hashvals_span(p, b, e)
        return h, ix, (int(b[0]), int(e[0]))
    finally:
        lib.smb_lca_hashvals_free(p)


class LcaTable:
    """The LCA node of every distinct database hash, resident on the GPU (``lca_table``)."""

    def __init__(self, ptr):
        self._ptr = ptr

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:
            lib.smb_lca_table_free(p)

    def __len__(self):
        return int(lib.smb_lca_table_len(self._ptr))

    def to_host(self):
        "(hashes ascending, lca nodes) as numpy arrays"
        n = len(self)
        h, lca = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        rustcall(lib.smb_lca_table_copy, self._ptr, _ptr(h, "uint64_t *"), _ptr(lca, "uint32_t *"))
        return h, lca


def lca_table(hashes, nodes, parent, depth, max_hash=2**64 - 1):
    """Fold the (hash, trie node) pairs of every database into one LCA node per distinct hash, on the device.  The trie
    is ``parent`` / ``depth`` (node 0 the root; ``parent[i] < i``); a node of ``LCA_NO_NODE`` contributes nothing, and
    hashes above ``max_hash`` are cut.  The node of a hash is the one the reference's tree walk gives for its lineages:
    the deepest when they lie on one root path, else the node where they branch."""
    h = _u64(hashes)
    nd = np.ascontiguousarray(nodes, dtype=np.uint32)
    par = np.ascontiguousarray(parent, dtype=np.uint32)
    dep = np.ascontiguousarray(depth, dtype=np.uint8)
    if len(h) != len(nd):
        raise ValueError("hashes and nodes differ in length")
    if len(par) != len(dep):
        raise ValueError("parent and depth differ in length")
    return LcaTable(rustcall(lib.smb_lca_table_build, _ptr(h, "uint64_t *"), _ptr(nd, "uint32_t *"), len(h),
                             _ptr(par, "uint32_t *"), _ptr(dep, "uint8_t *"), len(par), int(max_hash)))


def lca_counts(table, query_hashes, offsets=None, weights=None):
    """Every distinct (query, LCA node) of a batch of queries' hashes found in ``table``: ``(query, node, count,
    first)`` as numpy arrays ordered by (query, node).  ``count`` sums the weights of the hashes (1 each, or the
    query's abundances), ``first`` is the smallest position in the query of a hash with that node.  The queries are a
    CSR (``query_hashes``, ``offsets``, optional ``weights`` parallel to the hashes) or a resident ``SketchSet``, with
    ``weights=True`` to weight by its abundances."""
    if isinstance(query_hashes, SketchSet):
        sset, use = query_hashes, bool(weights)
    else:
        h, off = _u64(query_hashes), _u64(offsets)
        if len(off) == 0 or int(off[-1]) != len(h) or (weights is not None and len(weights) != len(h)):
            raise ValueError("query offsets must end at the number of hashes, and weights match the hashes")
        sset = SketchSet.from_host(h, off, weights)
        use = weights is not None
    p = rustcall(lib.smb_lca_counts, table._ptr, sset._ptr, use)
    try:
        n = int(lib.smb_lca_counts_len(p))

        def take(fn, dtype):
            return np.frombuffer(ffi.buffer(fn(p), n * np.dtype(dtype).itemsize), dtype=dtype).copy() if n else \
                np.zeros(0, dtype)
        return (take(lib.smb_lca_counts_query, np.uint32), take(lib.smb_lca_counts_node, np.uint32),
                take(lib.smb_lca_counts_count, np.uint64), take(lib.smb_lca_counts_first, np.uint64))
    finally:
        lib.smb_lca_counts_free(p)


class LcaIndex:
    """Every hash of a resident set grouped with the idx (rows) that hold it, on the GPU (``lca_index``): keys in the
    order LCA_Database.insert first saw them, each key's idx ascending."""

    def __init__(self, ptr):
        self._ptr = ptr

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:
            lib.smb_lca_index_free(p)

    def __len__(self):
        return int(lib.smb_lca_index_len(self._ptr))

    def pairs(self):
        return int(lib.smb_lca_index_pairs(self._ptr))

    def arrays(self):
        "(hashes in key order, offsets (len + 1), idx) as numpy arrays: key k's idx are idx[offsets[k]:offsets[k + 1]]"
        n, m = len(self), self.pairs()
        h, off, ix = np.zeros(n, np.uint64), np.zeros(n + 1, np.uint64), np.zeros(m, np.uint32)
        rustcall(lib.smb_lca_index_copy, self._ptr, _ptr(h, "uint64_t *"), _ptr(off, "uint64_t *"),
                 _ptr(ix, "uint32_t *"))
        return h, off, ix

    def _ranges(self, max_bytes):
        """memoryviews of one reused buffer, each holding one key range's text while the generator is not advanced;
        one call per range, and a second only for a key whose text alone is longer than max_bytes"""
        n, k, first = len(self), 0, True
        buf = bytearray(max(int(max_bytes), 2))
        size = ffi.new("uintptr_t *")
        while first or k < n:
            first = False
            size[0] = len(buf)
            nxt = rustcall(lib.smb_lca_index_text, self._ptr, k, int(max_bytes), ffi.from_buffer(buf), size)
            if int(size[0]) > len(buf):
                buf = bytearray(int(size[0]))
                size[0] = len(buf)
                nxt = rustcall(lib.smb_lca_index_text, self._ptr, k, int(max_bytes), ffi.from_buffer(buf), size)
            yield memoryview(buf)[:int(size[0])]
            k = int(nxt)

    def text_chunks(self, max_bytes=256 << 20):
        """The JSON text of "hashval_to_idx" (json.dump's form, braces included) as bytes, in ranges of whole keys of
        at most ``max_bytes`` each, braces counted (a key longer than that is one range alone)."""
        for view in self._ranges(max_bytes):
            yield bytes(view)

    def write_text(self, fh, max_bytes=256 << 20):
        "the text of text_chunks written to the binary file handle ``fh`` through one buffer; returns the bytes written"
        total = 0
        for view in self._ranges(max_bytes):
            fh.write(view)
            total += len(view)
        return total


def lca_index(sset):
    """Group every hash of the resident ``SketchSet`` (row r is idx r) with the rows holding it, on the device: the
    reference's LCA_Database.insert loop over the rows in order, with hashval_to_idx's keys in its first-insertion
    order.  Returns an ``LcaIndex``."""
    return LcaIndex(rustcall(lib.smb_lca_index_build, sset._ptr))


def gather(query, db, threshold=1, max_rounds=None):
    """Iterative min-set-cover; returns (match_ids, intersect_sizes) in pick order."""
    q = _u64(query)
    if max_rounds is None:
        max_rounds = len(db)
    ids = np.zeros(max(max_rounds, 1), dtype=np.uint32)
    sizes = np.zeros(max(max_rounds, 1), dtype=np.uint32)
    n = rustcall(lib.smb_gather, _ptr(q, "uint64_t *"), len(q), db._ptr, int(threshold),
                 _ptr(ids, "uint32_t *"), _ptr(sizes, "uint32_t *"), int(max_rounds))
    return ids[:n].copy(), sizes[:n].copy()


def multigather(queries, db, thresholds=None, min_counts=None, max_rounds=None, stats=None):
    """gather() of every query (sorted-unique u64 arrays) against the one resident ``db``, the rounds of all queries run
    together on the device.  ``thresholds`` / ``min_counts``: one per query (or one for all; default 1), as gather()'s
    threshold and the least overlap a row needs to take part at all.  Returns, per query, (rows, sizes, consumed_round):
    the picks as gather() returns them, and for every query hash the round that took it (UINT32_MAX: none).
    ``stats`` (a dict) receives the kernel launches of the batched rounds ("round_launches") and, per query, the
    overlap of every picked row with the whole query ("overlaps")."""
    hashes, offs = _query_csr(queries)
    n = len(offs) - 1

    def per_query(v):
        if v is None:
            return None
        a = np.broadcast_to(np.asarray(v, dtype=np.int64), (n,))
        return np.ascontiguousarray(np.clip(a, 0, 0xffffffff), dtype=np.uint32)
    thr, mc = per_query(thresholds), per_query(min_counts)
    if max_rounds is None:
        max_rounds = len(db)
    m = rustcall(lib.smb_multigather, _ptr(hashes, "uint64_t *"), _ptr(offs, "uint64_t *"), n, db._ptr,
                 _ptr(thr, "uint32_t *") if thr is not None else ffi.NULL,
                 _ptr(mc, "uint32_t *") if mc is not None else ffi.NULL, int(max_rounds))
    try:
        consumed = np.zeros(len(hashes), dtype=np.uint32)
        lib.smb_multigather_consumed(m, _ptr(consumed, "uint32_t *"))
        out = []
        for i in range(n):
            k = int(rustcall(lib.smb_multigather_rounds, m, i))
            rows, sizes, overlaps = (np.zeros(k, dtype=np.uint32) for _ in range(3))
            rustcall(lib.smb_multigather_picks, m, i, _ptr(rows, "uint32_t *"), _ptr(sizes, "uint32_t *"),
                     _ptr(overlaps, "uint32_t *"))
            out.append((rows, sizes, consumed[int(offs[i]):int(offs[i + 1])]))
            if stats is not None:
                stats.setdefault("overlaps", []).append(overlaps)
        if stats is not None:
            stats["round_launches"] = int(lib.smb_multigather_round_launches(m))
        return out
    finally:
        lib.smb_multigather_free(m)


class GatherSession:
    """Step-wise gather over one (local) database: begin / peek / intersect / apply
    (smb_gather_* of the C ABI).  ``gather()`` above is this loop run inside the library;
    ``distributed.ShardedDatabase.gather`` runs it across ranks."""

    def __init__(self, query, db, min_count=1):
        q = _u64(query)
        self._db = db
        self._cap = int(db.sizes().max()) if len(db) else 0
        self._ptr = rustcall(lib.smb_gather_begin_min, _ptr(q, "uint64_t *"), len(q), db._ptr, int(min_count))
        self.remaining = len(q)

    def __del__(self):
        p, self._ptr = getattr(self, "_ptr", None), None
        if p and lib is not None:
            lib.smb_gather_end(p)

    def peek(self):
        "(best_count, local_row)"
        c, r = ffi.new("uint32_t *"), ffi.new("uint32_t *")
        rustcall(lib.smb_gather_peek, self._ptr, c, r)
        return int(c[0]), int(r[0])

    def intersect(self, row):
        out = np.zeros(max(self._cap, 1), dtype=np.uint64)
        n = rustcall(lib.smb_gather_intersect, self._ptr, int(row), _ptr(out, "uint64_t *"))
        return out[:n].copy()

    def apply(self, intersect_hashes):
        h = _u64(intersect_hashes)
        self.remaining = int(rustcall(lib.smb_gather_apply, self._ptr, _ptr(h, "uint64_t *"), len(h)))
        return self.remaining
