"""In-memory index with GPU-batched search / prefetch / gather.

Mirrors the reference's ``Index`` protocol (src/sourmash/index/__init__.py:115-320) and its
``CounterGather`` helper (:735-909) for the linear (flat) case: the per-subject Python loop
of ``Index.find`` and the per-dataset loop of ``CounterGather.consume`` become single
one-vs-many kernel launches over a SketchSet kept in HBM.
"""
from collections import namedtuple, Counter

import numpy as np

from . import batch as B
from .manifest import CollectionManifest, _check_select_parameters
from .minhash import flatten_and_intersect_scaled
from .search import calc_threshold_from_bp, make_containment_query, make_jaccard_search_query
from .sigset import _INFO_DTYPE

IndexSearchResult = namedtuple("IndexSearchResult", "score, signature, location")
GatherResult = namedtuple("GatherResult", "match, intersect_size, containment, location")


def select_signature(ss, *, ksize=None, moltype=None, scaled=0, num=0, containment=False, abund=None,
                     picklist=None):
    "Does this signature match the requirements?  (index/__init__.py:349-395)"
    mh = ss.minhash
    if ksize and ksize != mh.ksize:
        return False
    if moltype and moltype != mh.moltype:
        return False
    if containment:
        if not scaled:
            raise ValueError("'containment' requires 'scaled' in Index.select'")
        if not mh.scaled:
            return False
    if scaled and mh.num:
        return False
    if num and (mh.scaled or num != mh.num):
        return False
    if abund and not mh.track_abundance:
        return False
    if picklist is not None and ss not in picklist:
        return False
    return True


_U64_MAX = 2**64 - 1
_HASH_FUNCTION = {"DNA": 1, "protein": 2, "dayhoff": 3, "hp": 4}


def _abi_scaled(max_hash):
    "KmerMinHash::scaled() of the library (sketch/minhash.rs:233-235): the scaled similarity(downsample=True) compares"
    if not max_hash:
        return 0
    v = float(2**64) / float(max_hash)
    return _U64_MAX if v >= float(2**64) else int(v)


def _angular_cut(q_max_hash, s_max_hash):
    """The max_hash both sketches are cut at by `similarity(other, downsample=True)` (sketch/minhash.rs:682-702), or None
    when that call fails the scaled check of angular_similarity.  Equal scaled: no cut (num sketches of any num too).
    Else the finer side is downsampled to the coarser one's scaled, and its max_hash must then equal the coarser one's."""
    sq, ss = _abi_scaled(q_max_hash), _abi_scaled(s_max_hash)
    if sq == ss:
        return _U64_MAX if q_max_hash == s_max_hash else None
    coarse_max_hash, fine_scaled = (q_max_hash, ss) if sq > ss else (s_max_hash, sq)
    if fine_scaled == 0:                                  # a num sketch is not downsampled: num vs scaled
        return None
    cut = B.max_hash_for_scaled(max(sq, ss))
    return cut if cut == coarse_max_hash else None


class LinearIndex:
    "A list of signatures searched on the GPU (reference: LinearIndex, index/__init__.py:380-470)."

    is_database = False
    manifest = None                   # Index protocol (index/__init__.py:65-68): None, or a manifest that makes select() cheap

    def __init__(self, _signatures=None, filename=None):
        self._signatures = list(_signatures) if _signatures else []
        self.filename = filename
        self._device = None          # (scaled -> (SketchSet, sizes)) cache
        self._abund_cols = None      # search_abund: metadata of the subjects ...
        self._abund_device = None    # ... and their groups with abundances on the device

    @property
    def location(self):
        return self.filename

    def signatures(self):
        return iter(self._signatures)

    def signatures_with_location(self):
        for ss in self.signatures():
            yield ss, self.location

    def __len__(self):
        return len(self._signatures)

    def __bool__(self):
        return bool(self._signatures)

    def insert(self, node):
        self._signatures.append(node)
        self._device = self._abund_cols = self._abund_device = None

    def save(self, path):
        from .signature import save_signatures_to_json
        with open(path, "w") as fp:
            save_signatures_to_json(self.signatures(), fp)

    @classmethod
    def load(cls, location, filename=None):
        "Signatures of one .sig / .sig.gz file (LinearIndex.load, index/__init__.py:438-446)."
        from .signature import load_signatures_from_json
        return cls(load_signatures_from_json(location, do_raise=True), filename=filename or location)

    def select(self, **kwargs):
        "New LinearIndex with the signatures matching the requirements (index/__init__.py:448-460)."
        _check_select_parameters(**kwargs)
        return LinearIndex([ss for ss in self._signatures if select_signature(ss, **kwargs)], self.location)

    def _subject(self, idx):
        return self._signatures[idx]

    # -- device cache ----------------------------------------------------------------------
    def _groups(self):
        """Subjects grouped by their own scaled (or num): {key: (indices, SketchSet)}; rows flat."""
        if self._device is None:
            groups = {}
            for idx, ss in enumerate(self._signatures):
                mh = ss.minhash
                key = ("scaled", mh.scaled) if mh.scaled else ("num", mh.num)
                groups.setdefault(key, []).append((idx, mh._mins_array()))
            self._device = {k: ([i for i, _ in v], B.SketchSet.from_rows([r for _, r in v]))
                            for k, v in groups.items()}
        return self._device

    def _subject_params(self):
        "(ksize, moltype, seed) of every subject, in index order"
        return [(ss.minhash.ksize, ss.minhash.moltype, ss.minhash.seed) for ss in self._signatures]

    def _first_incompatible(self, query_mh):
        "index of the first subject the query cannot be compared with (None: all compatible)"
        want = (query_mh.ksize, query_mh.moltype, query_mh.seed)
        for idx, got in enumerate(self._subject_params()):
            if got != want:
                return idx
        return None

    def build_device_index(self):
        """Build the inverted index (hash -> rows) of every resident group of this collection
        (batch.SketchSet.build_index): later search / prefetch / gather calls at the collection's own
        scaled probe it instead of streaming the rows.  Returns the number of distinct hashes."""
        return sum(sset.build_index() for _, sset in self._groups().values() if len(sset))

    # -- the 1 x N scoring loop ------------------------------------------------------------
    def find(self, search_fn, query, **kwargs):
        """Yield IndexSearchResult for subjects passing search_fn, in index order
        (Index.find, index/__init__.py:115-170)."""
        yield from self._find(search_fn, query)

    def _find(self, search_fn, query, counted=None, cache=None):
        """find(); ``counted`` maps a resident group's key to (query size, shared counts) already computed for this
        query by ``_many_counts`` (``cache``: its downsampled groups), the other groups are counted here."""
        search_fn.check_is_compatible(query)
        query_mh = query.minhash
        assert not query_mh.track_abundance
        # The reference scores subject by subject and `intersection_and_union_size` raises
        # TypeError("incompatible MinHash objects") at the first subject whose ksize / molecule / seed
        # differ from the query's (minhash.py:649-654): results of earlier subjects have been yielded by then.
        first_bad = self._first_incompatible(query_mh)
        scored = []
        for (kind, val), (indices, sset) in self._groups().items():
            if query_mh.scaled:
                if kind != "scaled":
                    raise ValueError("cannot compare scaled query against num sketches")
                s = max(query_mh.scaled, val)
                sub = self._downsampled(kind, val, sset, s, cache)
                if counted is not None and (kind, val) in counted:
                    n_query, shared = counted[(kind, val)]
                else:
                    q = query_mh.downsample(scaled=s) if s > query_mh.scaled else query_mh
                    qarr = q._mins_array()
                    n_query, shared = len(qarr), B.one_vs_many(qarr, sub)
                sizes = sub.sizes()
                total = n_query + sizes - shared
                qsize = np.full(len(indices), n_query)
            else:
                if kind != "num":
                    raise ValueError("cannot compare num query against scaled sketches")
                n = min(query_mh.num, val)
                rows = sset.rows()
                sub = B.SketchSet.from_rows([r[:n] for r in rows])
                qarr = query_mh._mins_array()[:n]
                cm, us = B.pairwise_common(B.SketchSet.from_rows([qarr]), sub, num=n, want_usize=True)
                shared, total = cm[0], us[0]
                sizes = sub.sizes()
                qsize = np.full(len(indices), len(qarr))
            for pos, idx in enumerate(indices):
                scored.append((idx, int(qsize[pos]), int(shared[pos]), int(sizes[pos]), int(total[pos])))
        scored.sort()
        for idx, qs, sh, ss_size, tot in scored:
            if first_bad is not None and idx >= first_bad:
                raise TypeError("incompatible MinHash objects")
            score = search_fn.score_fn(qs, sh, ss_size, tot)
            if search_fn.passes(score):
                subj = self._subject(idx)
                if search_fn.collect(score, subj):
                    yield IndexSearchResult(score, subj, self.location)

    def _downsampled(self, kind, val, sset, s, cache=None):
        "the resident group (kind, val) at scaled s >= val (cache: {(kind, val, s): SketchSet} shared across queries)"
        if s <= val:
            return sset
        if cache is None:
            return sset.downsample(B.max_hash_for_scaled(s))
        key = (kind, val, s)
        if key not in cache:
            cache[key] = sset.downsample(B.max_hash_for_scaled(s))
        return cache[key]

    def _many_counts(self, queries):
        """({query position: {group key: (query size, shared counts)}}, downsampled groups) for the queries the batched pass takes: flat
        scaled queries compatible with every subject, against the scaled groups.  Each (group, effective scaled
        s = max(query scaled, group scaled)) is one downsampled copy and one many_vs_many call.  Every other query
        and group is counted by _find itself, query by query, with its errors."""
        mhs = [q.minhash for q in queries]
        ok = [i for i, mh in enumerate(mhs) if mh.scaled and not mh.track_abundance
              and self._first_incompatible(mh) is None]
        out = {i: {} for i in ok}
        cache = {}
        for (kind, val), (_indices, sset) in self._groups().items():
            if kind != "scaled" or not ok:
                continue
            by_s = {}
            for i in ok:
                by_s.setdefault(max(mhs[i].scaled, val), []).append(i)
            for s, members in by_s.items():
                sub = self._downsampled(kind, val, sset, s, cache)
                qarrs = [(mhs[i].downsample(scaled=s) if s > mhs[i].scaled else mhs[i])._mins_array() for i in members]
                counts = B.many_vs_many(qarrs, sub)
                for i, qarr, row in zip(members, qarrs, counts):
                    out[i][(kind, val)] = (len(qarr), row)
        return out, cache

    def search_many(self, queries, *, threshold=None, do_containment=False, do_max_containment=False,
                    best_only=False, **kwargs):
        """search() of every query: element i equals ``self.search(queries[i], ...)``, the first query whose
        search would raise raises the same here.  Queries that share a resident group and an effective scaled are
        counted together, one pass over the group for many queries."""
        if not queries:
            return []
        if threshold is None:
            raise TypeError("'search' requires 'threshold'")
        counted, cache = self._many_counts(queries)
        out = []
        for i, query in enumerate(queries):
            search_obj = make_jaccard_search_query(do_containment=do_containment,
                                                   do_max_containment=do_max_containment,
                                                   best_only=best_only, threshold=float(threshold))
            matches = list(self._find(search_obj, query, counted.get(i), cache))
            matches.sort(key=lambda x: -x.score)
            out.append(matches)
        return out

    def prefetch_many(self, queries, threshold_bp, **kwargs):
        """prefetch() of every query: element i equals ``list(self.prefetch(queries[i], threshold_bp))``, the first
        query whose prefetch would raise raises the same here.  Counted as in search_many."""
        if not queries:
            return []
        if not self:
            raise ValueError("no signatures to search")
        counted, cache = self._many_counts(queries)
        return [list(self._find(make_containment_query(query.minhash, threshold_bp, best_only=False), query,
                                counted.get(i), cache))
                for i, query in enumerate(queries)]

    # -- search_abund: the subjects' metadata, their resident groups with abundances, the match objects ------------
    def _subject_ptrs(self, positions):
        """The library's view of the subjects at ``positions``: (signature pointers, sketch pointers, objects to keep
        alive).  A SourmashSignature is passed as it is; any other subject by its ``.minhash``, as the reference's loop
        only reads ``subject.minhash``."""
        from ._lowlevel import ffi
        from .signature import SourmashSignature
        sigs, mhs, keep = [], [], []
        for i in positions:
            o = self._signatures[i]
            if isinstance(o, SourmashSignature):
                sigs.append(o._get_objptr())
                mhs.append(ffi.NULL)
            else:
                mh = o.minhash
                keep.append(mh)
                sigs.append(ffi.NULL)
                mhs.append(mh._get_objptr())
        return ffi.new("SourmashSignature *[]", sigs), ffi.new("SourmashKmerMinHash *[]", mhs), keep

    def _abund_info(self):
        """ksize (as stored), hash_function, seed, max_hash and has_abund of every subject, in index order (one
        library call, no sketch copied; built once)"""
        if self._abund_cols is None:
            from ._ffi import rustcall
            from ._lowlevel import ffi, lib
            n = len(self._signatures)
            sigs, mhs, _keep = self._subject_ptrs(range(n))
            info = ffi.new("SmbSketchInfo[]", max(n, 1))
            rustcall(lib.smb_subjects_sketch_info, sigs, mhs, n, info)
            self._abund_cols = np.frombuffer(ffi.buffer(info, n * ffi.sizeof("SmbSketchInfo")), dtype=_INFO_DTYPE).copy()
        return self._abund_cols

    def _abund_sketchset(self, positions):
        "the subjects at ``positions`` as one resident set with abundances, gathered straight from the objects"
        from ._ffi import rustcall
        from ._lowlevel import lib
        sigs, mhs, _keep = self._subject_ptrs(positions)
        return B.SketchSet(rustcall(lib.smb_sketchset_from_subjects, sigs, mhs, len(positions), True))

    def _subjects(self, positions):
        "the subject objects at ``positions``"
        return [self._signatures[i] for i in positions]

    def _abund_groups(self):
        """Subjects grouped by their max_hash: {max_hash: (positions, SketchSet with abundances)}, one upload per group
        (built once, beside the flat ``_groups()``)."""
        if self._abund_device is None:
            groups = {}
            for pos, mx in enumerate(self._abund_info()["max_hash"].tolist()):
                groups.setdefault(mx, []).append(pos)
            self._abund_device = {mx: (np.array(pos), self._abund_sketchset(pos)) for mx, pos in groups.items()}
        return self._abund_device

    def search_abund(self, query, *, threshold=None, **kwargs):
        """Matches by angular similarity of abundance sketches, best first (Index.search_abund, index/__init__.py:172-200).

        The reference calls `query.similarity(subject, downsample=True)` subject by subject.  Here every resident group
        (one max_hash) is scored in one device pass (batch.search_angular), both sides cut at the max_hash that call
        downsamples to.  The first subject at which the reference's loop raises is found from the metadata, and raises
        the same exception before anything is scored; signature objects are built for the matches only."""
        query_mh = query.minhash
        if not query_mh.track_abundance:
            raise TypeError("'search_abund' requires query signature with abundance information")
        if threshold is None:
            raise TypeError("'search_abund' requires 'threshold'")
        threshold = float(threshold)
        info = self._abund_info()
        if not len(info):
            return []
        track, max_hash = info["has_abund"].astype(bool), info["max_hash"]
        mq = query_mh._max_hash
        cuts = {mx: _angular_cut(mq, mx) for mx in np.unique(max_hash).tolist()}
        # check_compatible (sketch/minhash.rs:886-912) on the stored columns: ksize as stored (3k for protein-family
        # sketches), hash function, seed; the max_hash condition is in `cuts`
        hf = _HASH_FUNCTION[query_mh.moltype]
        bad = ~track | (info["ksize"] != query_mh.ksize * (1 if hf == 1 else 3)) | (info["hash_function"] != hf)
        bad |= info["seed"] != np.uint64(query_mh.seed)
        bad |= np.isin(max_hash, np.array([mx for mx, c in cuts.items() if c is None], dtype=np.uint64))
        if bad.any():
            i = int(np.argmax(bad))
            if not track[i]:
                raise TypeError("'search_abund' requires subject signatures with abundance information")
            query.similarity(self._subjects([i])[0], downsample=True)   # raises the reference's exception for this subject
            raise AssertionError("subject %d was expected to be incompatible with the query" % i)
        qh, qa = query_mh._mins_array(), query_mh._abunds_array()
        scores = np.empty(len(info), dtype=np.float64)
        for mx, (pos, sset) in self._abund_groups().items():
            scores[pos] = B.search_angular(qh, qa, sset, cuts[mx])
        order = np.argsort(-scores, kind="stable")              # list.sort(key=-score) is stable: ties keep index order
        keep = order[scores[order] >= threshold].tolist()
        return [IndexSearchResult(float(scores[i]), subj, self.location)
                for i, subj in zip(keep, self._subjects(keep))]

    def search(self, query, *, threshold=None, do_containment=False, do_max_containment=False,
               best_only=False, **kwargs):
        "Sorted (best first) matches at or above threshold (Index.search, :202-239)."
        if threshold is None:
            raise TypeError("'search' requires 'threshold'")
        threshold = float(threshold)
        search_obj = make_jaccard_search_query(do_containment=do_containment,
                                               do_max_containment=do_max_containment,
                                               best_only=best_only, threshold=threshold)
        matches = list(self.find(search_obj, query, **kwargs))
        matches.sort(key=lambda x: -x.score)
        return matches

    def prefetch(self, query, threshold_bp, **kwargs):
        "All subjects overlapping the query by at least threshold_bp (Index.prefetch, :241-256)."
        if not self:
            raise ValueError("no signatures to search")
        search_fn = make_containment_query(query.minhash, threshold_bp, best_only=False)
        yield from self.find(search_fn, query, **kwargs)

    def counter_gather(self, query, threshold_bp, **kwargs):
        "CounterGather pre-loaded with every prefetch match (Index.counter_gather, :302-320)."
        counter = CounterGather(query)
        for result in self.prefetch(query, threshold_bp, **kwargs):
            counter.add(result.signature, location=result.location, require_overlap=False)
        return counter

    def best_containment(self, query, threshold_bp=None, **kwargs):
        results = self.prefetch(query, threshold_bp, best_only=True, **kwargs)
        results = sorted(results, key=lambda x: (-x.score, x.signature.md5sum()))
        return results[0] if results else None


class ZipFileLinearIndex(LinearIndex):
    """A read-only .zip collection of signatures (reference: ZipFileLinearIndex,
    index/__init__.py:529-733), selected through its manifest when it has one.

    The reference loads members lazily, one Python object per sketch per pass.  Here the whole
    collection is parsed once by the library (``sigset.SignatureSet``: members inflated and parsed
    on all host threads into one CSR) and searched from HBM; ``SourmashSignature`` objects are only
    built for the subjects a search returns, or when ``signatures()`` is iterated."""

    is_database = True

    def __init__(self, storage, *, selection_dict=None, traverse_yield_all=False, manifest=None,
                 use_manifest=True, _sigset=None):
        from .sigset import SignatureSet
        self.storage = storage
        self.selection_dict = selection_dict
        self.traverse_yield_all = traverse_yield_all
        self.use_manifest = use_manifest
        self.filename = storage.path
        self._device = None
        self._abund_device = None
        self._objects = {}
        self._sigset = _sigset if _sigset is not None else SignatureSet.from_files(
            [storage.path], use_manifest=use_manifest, traverse_yield_all=traverse_yield_all)
        ss = self._sigset
        self.manifest = None
        if use_manifest:
            self.manifest = manifest if manifest is not None else self._load_manifest()
        if self.manifest is not None:
            assert not self.selection_dict, self.selection_dict
            # `for filename in manifest.locations(): ... if ss in manifest` (index/__init__.py:644-657)
            locations, md5s = set(self.manifest.locations()), self.manifest._md5_set
            self._rows = np.array([i for i, (md5, loc) in enumerate(zip(ss.md5sums(), ss.locations()))
                                   if md5 in md5s and loc in locations], dtype=np.uint32)
        else:
            self._rows = self._select_rows(**(selection_dict or {}))

    def _load_manifest(self):
        from io import StringIO
        try:
            data = self.storage.load("SOURMASH-MANIFEST.csv")
        except (KeyError, FileNotFoundError):
            return None
        return CollectionManifest.load_from_csv(StringIO(data.decode("utf-8")))

    def _select_rows(self, *, ksize=None, moltype=None, scaled=0, num=0, containment=False, abund=None,
                     picklist=None):
        "select_signature over the metadata columns of the parsed collection."
        if picklist is not None:
            raise NotImplementedError("picklists are outside the GPU path")
        ss = self._sigset
        is_dna = ss.hash_function == 1
        keep = np.ones(len(ss), bool)
        if ksize:
            keep &= np.where(is_dna, ss.ksize, ss.ksize // 3) == ksize
        if moltype:
            keep &= ss.hash_function == {"DNA": 1, "protein": 2, "dayhoff": 3, "hp": 4}[moltype]
        if containment:
            if not scaled:
                raise ValueError("'containment' requires 'scaled' in Index.select'")
            keep &= ss.max_hash != 0
        if scaled:
            keep &= ss.num == 0
        if num:
            keep &= (ss.max_hash == 0) & (ss.num == num)
        if abund:
            keep &= ss.has_abund
        return np.nonzero(keep)[0].astype(np.uint32)

    @classmethod
    def load(cls, location, traverse_yield_all=False, use_manifest=True):
        import os

        from .sbt_storage import ZipStorage
        if not os.path.exists(location):
            raise FileNotFoundError(location)
        return cls(ZipStorage(location), traverse_yield_all=traverse_yield_all, use_manifest=use_manifest)

    @property
    def location(self):
        return self.storage.path

    def __len__(self):
        return len(self.manifest) if self.manifest is not None else len(self._rows)

    def __bool__(self):
        """Any matching signature?  Never len() (index/__init__.py:584-591).  The selected rows are known here without building
        a single object; a subclass without them (the reference's test fakes one) is asked for its first signature."""
        rows = getattr(self, "_rows", None)
        if rows is not None:
            return len(rows) > 0
        try:
            next(iter(self.signatures()))
        except StopIteration:
            return False
        return True

    def insert(self, signature):
        raise NotImplementedError

    def save(self, path):
        raise NotImplementedError

    def _subject(self, idx):
        if idx not in self._objects:
            self._objects[idx] = self._sigset.signatures(self._rows[idx:idx + 1])[0]
        return self._objects[idx]

    def signatures(self):
        missing = [i for i in range(len(self._rows)) if i not in self._objects]
        if missing:
            for i, obj in zip(missing, self._sigset.signatures(self._rows[missing])):
                self._objects[i] = obj
        for i in range(len(self._rows)):
            yield self._objects[i]

    def _signatures_with_internal(self):
        "(signature, member name) of everything in the file, selection ignored (index/__init__.py:620-637)."
        ss = self._sigset
        for i, obj in enumerate(ss.signatures()):
            yield obj, ss.location(i)

    def select(self, **kwargs):
        _check_select_parameters(**kwargs)
        if self.manifest is not None:
            return ZipFileLinearIndex(self.storage, traverse_yield_all=self.traverse_yield_all,
                                      manifest=self.manifest.select_to_manifest(**kwargs), use_manifest=True,
                                      _sigset=self._sigset)
        if self.selection_dict:
            d = dict(self.selection_dict)
            for k, v in kwargs.items():
                if k in d and d[k] is not None and d[k] != v:
                    raise ValueError(f"incompatible select on '{k}'")
                d[k] = v
            kwargs = d
        return ZipFileLinearIndex(self.storage, selection_dict=kwargs, traverse_yield_all=self.traverse_yield_all,
                                  manifest=None, use_manifest=False, _sigset=self._sigset)

    def _subject_params(self):
        "(ksize, moltype, seed) of the selected sketches from the parser's metadata columns (no objects built)"
        ss = self._sigset
        out = []
        for row in self._rows.tolist():
            mol = ss.moltype(row)
            k = int(ss.ksize[row])
            out.append((k if mol == "DNA" else k // 3, mol, int(ss.seed[row])))   # protein-family sketches store 3*k
        return out

    def _abund_info(self):
        ss = self._sigset
        info = np.zeros(len(self._rows), dtype=_INFO_DTYPE)
        for name in ("ksize", "hash_function", "seed", "max_hash", "has_abund"):
            info[name] = getattr(ss, name)[self._rows]
        return info

    def _abund_sketchset(self, positions):
        return self._sigset.to_sketchset(self._rows[positions], with_abunds=True)

    def _subjects(self, positions):
        "the signature objects at ``positions``, the ones not built yet in one call"
        missing = sorted({i for i in positions if i not in self._objects})
        if missing:
            for i, obj in zip(missing, self._sigset.signatures(self._rows[missing])):
                self._objects[i] = obj
        return [self._objects[i] for i in positions]

    def _groups(self):
        "Selected rows grouped by scaled (or num), each group one CSR upload straight from the parser's arrays."
        if self._device is None:
            ss, groups = self._sigset, {}
            scaled = ss.python_scaled()
            for pos, row in enumerate(self._rows.tolist()):
                key = ("scaled", int(scaled[row])) if ss.max_hash[row] else ("num", int(ss.num[row]))
                groups.setdefault(key, []).append(pos)
            self._device = {k: (pos, ss.to_sketchset(self._rows[pos])) for k, pos in groups.items()}
        return self._device


class CounterGather:
    """Tracks overlaps between a query and candidate matches for min-set-cover ``gather``
    (protocol of index/__init__.py:735-909; conformance: tests/test_index_protocol.py of the
    reference).  ``add`` records candidates, the first ``peek`` moves them to HBM, ``consume``
    decrements every counter with one one-vs-many launch."""

    def __init__(self, query):
        query_mh = query.minhash
        if not query_mh.scaled:
            raise ValueError("gather requires scaled signatures")
        self.orig_query_mh = query_mh.copy().flatten()
        self.scaled = query_mh.scaled
        self.siglist = {}
        self.locations = {}
        self.counter = Counter()     # md5 -> overlap, insertion ordered (ties: first added wins), a Counter like the reference's
        self.query_started = 0
        self._pending = []           # signatures added but not yet counted
        self._sset = None
        self._order = None

    def _count_pending(self):
        if not self._pending:
            return
        qarr = self.orig_query_mh._mins_array()
        rows = [ss.minhash._mins_array() for ss, _, _ in self._pending]
        counts = B.one_vs_many(qarr, B.SketchSet.from_rows(rows))
        pending, self._pending = self._pending, []
        for (ss, location, require_overlap), overlap in zip(pending, counts.tolist()):
            if overlap:
                md5 = ss.md5sum()
                self.counter[md5] = overlap
                self.siglist[md5] = ss
                self.locations[md5] = location
                self.downsample(ss.minhash.scaled)
            elif require_overlap:
                raise ValueError("no overlap between query and signature!?")

    def add(self, ss, *, location=None, require_overlap=True):
        "Register a candidate match (overlap counted on the GPU)."
        if self.query_started:
            raise ValueError("cannot add more signatures to counter after peek/consume")
        # count_common(query, match, downsample=True) of the reference checks compatibility first
        # (sketch/minhash.rs:539-547,886-912): same ksize / molecule / seed, both scaled
        mh, q = ss.minhash, self.orig_query_mh
        if mh.ksize != q.ksize:
            raise ValueError("different ksizes cannot be compared")
        if mh.moltype != q.moltype:
            raise ValueError("DNA/prot minhashes cannot be compared")
        if not mh.scaled:
            raise ValueError("mismatch in scaled; comparison fail")
        if mh.seed != q.seed:
            raise ValueError("mismatch in seed; comparison fail")
        self._pending.append((ss, location, require_overlap))
        if require_overlap:
            self._count_pending()          # the reference raises at add() time

    def downsample(self, scaled):
        if scaled > self.scaled:
            self.scaled = scaled
        return self.scaled

    def signatures(self):
        self._count_pending()
        yield from self.siglist.values()

    @property
    def union_found(self):
        self._count_pending()
        found_mh = self.orig_query_mh.copy_and_clear()
        for ss in self.siglist.values():
            found_mh.add_many(flatten_and_intersect_scaled(ss.minhash, self.orig_query_mh))
        return found_mh

    def _start(self):
        self._count_pending()
        self.query_started = 1
        if self._sset is None and self.siglist:
            self._order = list(self.siglist.keys())
            self._sset = B.SketchSet.from_rows([self.siglist[m].minhash._mins_array() for m in self._order])

    def peek(self, cur_query_mh, *, threshold_bp=0):
        "Best remaining match and its intersection with the current query; [] if none."
        self._start()
        if not self.counter:
            return []
        scaled = self.downsample(cur_query_mh.scaled)
        cur_query_mh = cur_query_mh.downsample(scaled=scaled)
        if not cur_query_mh:
            return []
        if cur_query_mh.contained_by(self.orig_query_mh, downsample=True) < 1:
            raise ValueError("current query not a subset of original query")
        try:
            threshold, n_threshold_hashes = calc_threshold_from_bp(threshold_bp, scaled, len(cur_query_mh))
        except ValueError:
            return []
        best = max(self.counter.values())
        dataset_id = next(k for k, v in self.counter.items() if v == best)   # first inserted wins ties
        if best < n_threshold_hashes:
            return []
        match = self.siglist[dataset_id]
        cont = cur_query_mh.contained_by(match.minhash, downsample=True)
        assert cont
        assert cont >= threshold
        match_mh = match.minhash.downsample(scaled=scaled).flatten()
        intersect_mh = cur_query_mh & match_mh
        return (IndexSearchResult(cont, match, self.locations[dataset_id]), intersect_mh)

    def consume(self, intersect_mh):
        "Subtract the hashes of the chosen match from every remaining counter."
        self._start()
        if not intersect_mh:
            return
        deltas = B.one_vs_many(intersect_mh._mins_array(), self._sset)
        for md5, d in zip(self._order, deltas.tolist()):
            if d and md5 in self.counter:
                self.counter[md5] -= d
                if self.counter[md5] == 0:
                    del self.counter[md5]


def gather(query, index, threshold_bp=0):
    """Iterative min-set-cover of ``query`` by the signatures of ``index`` (the loop of
    GatherDatabases.__next__, search.py:877-949).  Yields GatherResult in pick order."""
    counter = index.counter_gather(query, threshold_bp)
    cur = query.minhash.flatten().to_mutable()
    while True:
        result = counter.peek(cur, threshold_bp=threshold_bp)
        if not result:
            return
        sr, intersect_mh = result
        counter.consume(intersect_mh)
        yield GatherResult(sr.signature, len(intersect_mh), sr.score, sr.location)
        cur = cur.downsample(scaled=counter.scaled).to_mutable() if counter.scaled > cur.scaled else cur
        cur.remove_many(sr.signature.minhash.downsample(scaled=cur.scaled) if
                        sr.signature.minhash.scaled < cur.scaled else sr.signature.minhash)


def load_file_as_index(filename, yield_all_files=False, _use_manifest=True):
    """A collection of signatures by location -- the loaders of the reference's chain (save_load.py:46-66, 140-233) that are
    in scope: a directory -> LinearIndex over the *.sig / *.sig.gz files below it (every file with ``yield_all_files``),
    a .zip collection -> ZipFileLinearIndex, a .sig JSON file (plain or compressed) -> LinearIndex.  SBT, LCA and sqlite
    databases, standalone manifests and path lists are not handled.  Failure is the reference's ValueError."""
    import os
    err = ValueError(f"Error while reading signatures from '{filename}'.")
    if not os.path.exists(filename):
        raise err
    if os.path.isdir(filename):
        found = []
        for root, _dirs, files in sorted(os.walk(filename)):
            for name in sorted(files):
                if yield_all_files or name.endswith(".sig") or name.endswith(".sig.gz"):
                    path = os.path.join(root, name)
                    try:
                        found.extend(LinearIndex.load(path).signatures())
                    except Exception:
                        if not yield_all_files:            # forced traversal skips what does not parse
                            raise err
        return LinearIndex(found, filename)
    try:
        return LinearIndex.load(filename)
    except Exception:
        pass
    if filename.endswith(".zip"):
        try:
            return ZipFileLinearIndex.load(filename, traverse_yield_all=yield_all_files, use_manifest=_use_manifest)
        except Exception:
            pass
    raise err


def load_file_as_signatures(filename, *, select_moltype=None, ksize=None, picklist=None, yield_all_files=False, progress=None,
                            pattern=None, _use_manifest=True):
    """Iterator over the signatures at ``filename`` that match (sourmash_args.py:765-816).  Picklists and name patterns are
    out of scope: passing one raises."""
    if picklist is not None or pattern is not None:
        raise NotImplementedError("picklists / patterns are not supported by sourmash_b200.load_file_as_signatures")
    if progress:
        progress.notify(filename)
    db = load_file_as_index(filename, yield_all_files=yield_all_files, _use_manifest=_use_manifest)

    def gen():
        yield from db.select(moltype=select_moltype, ksize=ksize).signatures()
    return gen()
