"""All-vs-all comparison of signatures on the GPU.

Function-for-function replacement of sourmash/src/sourmash/compare.py (:14-358): the
reference walks ``itertools.combinations`` in Python and crosses the FFI three times per
pair; here a list of signatures becomes one CSR SketchSet in HBM and one batched call
produces the whole count matrix.  Float post-processing follows the reference's operation
order (similarity = common / max(1, union) on the device as an IEEE f64 divide; containment
bias factors computed with Python floats exactly like minhash.py:827-841).
"""
import sys

import numpy as np

from . import batch as B
from . import distance_utils as DU

_FALSE_NEG_WARNING = ("WARNING: Some of these sketches may have no hashes in common based on chance alone "
                      "(false negatives). Consider decreasing your scaled value to prevent this.")
_JACCARD_WARNING = ("WARNING: Jaccard estimation for at least one of these comparisons is likely inaccurate. "
                    "Could not estimate ANI for these comparisons.")


def notify(msg):
    print(msg, file=sys.stderr)


def _sizes_accurate_arrays(sizes, scaleds, relative_error=0.20, confidence=0.95):
    "size_is_accurate() for sketches given as (number of hashes, scaled) arrays."
    if not np.all(scaleds):
        raise TypeError("Error: can only calculate ANI for scaled MinHashes")
    out = np.zeros(len(sizes), dtype=bool)
    cache = {}
    for i, key in enumerate(zip((int(x) for x in sizes), (int(x) for x in scaleds))):
        if key not in cache:
            cache[key] = bool(DU.set_size_exact_prob(key[0] * key[1], key[1], relative_error=relative_error) >= confidence)
        out[i] = cache[key]
    return out


def _p_nothing_in_common(dist, n_unique_kmers, ksize, scaled):
    "get_exp_probability_nothing_common for arrays (distance_utils.py:247-270)."
    q = 1 - (1 - dist) ** ksize
    p = np.exp((n_unique_kmers - n_unique_kmers * q) * np.log(1.0 - 1.0 / float(scaled)))
    return np.where(dist == 1.0, 1.0, np.where(dist == 0.0, 0.0, p))


def _flat_minhashes(siglist):
    return [s.minhash if hasattr(s, "minhash") else s for s in siglist]


def _collect(siglist, *, downsample, need_scaled=False, with_abunds=False):
    """Validate compatibility like the per-pair calls would and return the sketches as host CSR:
    dict(hashes, offsets, abunds, num, scaled, sizes, has_abund, ksize).  The sketches of all
    objects come out of the library in one call (SignatureSet.from_objects); mixed lists fall back
    to one call per object."""
    from .sigset import SignatureSet
    objs = list(siglist)
    ss = SignatureSet.from_objects(objs)
    if ss is None:
        return _collect_per_object(objs, downsample=downsample, need_scaled=need_scaled, with_abunds=with_abunds)
    n = len(ss)
    pyscaled = ss.python_scaled()
    # the reference's per-pair checks, in its order, reported for the first offending sketch
    bad = (ss.ksize != ss.ksize[0]) | (ss.hash_function != ss.hash_function[0]) | (ss.seed != ss.seed[0]) | \
        (ss.num != ss.num[0])
    if bad.any():
        i = int(np.argmax(bad))
        if ss.ksize[i] != ss.ksize[0]:
            raise ValueError("different ksizes cannot be compared")
        if ss.hash_function[i] != ss.hash_function[0]:
            raise ValueError("DNA/prot minhashes cannot be compared")
        if ss.seed[i] != ss.seed[0]:
            raise ValueError("mismatch in seed; comparison fail")
        if (ss.num[0] == 0) != (ss.num[i] == 0):         # a scaled sketch against a num sketch: max_hash differs (minhash.rs:886-912)
            raise ValueError("mismatch in scaled; comparison fail")
        raise TypeError(f"incompatible num values: self={int(ss.num[0])} other={int(ss.num[i])}")
    if need_scaled and not pyscaled.all():
        raise TypeError("Error: can only calculate containment for scaled MinHashes")
    scaled = int(pyscaled.max())
    cut, raw = 0, None
    if len(np.unique(pyscaled)) > 1:
        if not downsample:
            raise ValueError("mismatch in scaled; comparison fail")
        cut = B.max_hash_for_scaled(scaled)
        raw = ss.csr_host(0, with_abunds=True)            # the sketches as given: pairs are compared at max(scaled_i, scaled_j)
    h, off, ab = ss.csr_host(cut, with_abunds=True)
    ksize = int(ss.ksize[0]) if int(ss.hash_function[0]) == 1 else int(ss.ksize[0]) // 3
    return {"hashes": h, "offsets": off, "abunds": ab if with_abunds else None, "num": int(ss.num[0]),
            "scaled": scaled, "sizes": np.diff(off.astype(np.int64)), "has_abund": ss.has_abund.copy(), "ksize": ksize,
            "orig_sizes": ss.n_mins.astype(np.int64), "orig_scaled": pyscaled, "raw": raw, "_keepalive": ss}


def _collect_per_object(objs, *, downsample, need_scaled, with_abunds):
    "Same contract through one FFI round trip per object (MinHash-like objects of other origins)."
    mhs = _flat_minhashes(objs)
    first = mhs[0]
    for mh in mhs[1:]:
        if mh.ksize != first.ksize:
            raise ValueError("different ksizes cannot be compared")
        if mh.moltype != first.moltype:
            raise ValueError("DNA/prot minhashes cannot be compared")
        if mh.seed != first.seed:
            raise ValueError("mismatch in seed; comparison fail")
        if bool(mh.num) != bool(first.num):
            raise ValueError("mismatch in scaled; comparison fail")
        if mh.num != first.num:
            raise TypeError(f"incompatible num values: self={first.num} other={mh.num}")
    if need_scaled and not all(mh.scaled for mh in mhs):
        raise TypeError("Error: can only calculate containment for scaled MinHashes")
    scaleds = {mh.scaled for mh in mhs}
    scaled = max(scaleds)
    has_ab = np.array([bool(mh.track_abundance) for mh in mhs])
    orig_sizes = np.array([len(mh) for mh in mhs], dtype=np.int64)
    orig_scaled = np.array([mh.scaled for mh in mhs], dtype=np.uint64)
    raw = None
    if len(scaleds) > 1:
        if not downsample:
            raise ValueError("mismatch in scaled; comparison fail")
        raw_rows = [mh._mins_array() for mh in mhs]
        raw_off = np.zeros(len(raw_rows) + 1, dtype=np.uint64)
        raw_off[1:] = np.cumsum([len(r) for r in raw_rows])
        raw = (np.concatenate(raw_rows), raw_off,
               np.concatenate([mh._abunds_array() if mh.track_abundance else np.ones(len(r), dtype=np.uint64)
                               for mh, r in zip(mhs, raw_rows)]))
        mhs = [mh.downsample(scaled=scaled) if mh.scaled != scaled else mh for mh in mhs]
    rows = [mh._mins_array() for mh in mhs]
    off = np.zeros(len(rows) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    h = np.concatenate(rows) if rows else np.zeros(0, np.uint64)
    ab = None
    if with_abunds:
        ab = np.concatenate([mh._abunds_array() if mh.track_abundance else np.ones(len(r), dtype=np.uint64)
                             for mh, r in zip(mhs, rows)]) if rows else np.zeros(0, np.uint64)
    return {"hashes": h, "offsets": off, "abunds": ab, "num": first.num, "scaled": scaled,
            "sizes": np.diff(off.astype(np.int64)), "has_abund": has_ab, "ksize": first.ksize,
            "orig_sizes": orig_sizes, "orig_scaled": orig_scaled, "raw": raw}


def _scaled_groups(c):
    """Sketches with different scaled values: one group per distinct value S -- the sketches with scaled <= S, cut at S
    (what downsample(scaled=S) keeps of a sorted row is a prefix).  Yields (S, rows of the group, their lengths at S,
    hashes, offsets, mask of the pairs whose coarser member has scaled S: the pairs the reference compares at S)."""
    h, off, _ab = c["raw"]
    scaleds = np.asarray(c["orig_scaled"]).astype(np.int64)
    for S in sorted(set(scaleds.tolist())):
        idx = np.nonzero(scaleds <= S)[0]
        if len(idx) < 2:
            continue
        cut = np.uint64(B.max_hash_for_scaled(S))
        lens = [int(np.searchsorted(h[int(off[i]):int(off[i + 1])], cut, side="right")) for i in idx]
        sub_off = np.zeros(len(idx) + 1, dtype=np.uint64)
        sub_off[1:] = np.cumsum(lens)
        sub_h = np.concatenate([h[int(off[i]):int(off[i]) + m] for i, m in zip(idx, lens)])
        here = (scaleds[idx][:, None] == S) | (scaleds[idx][None, :] == S)      # pairs decided at this scaled
        yield S, idx, lens, sub_h, sub_off, here


def _mixed_pair_tables(c, *, jaccard=False, angular=False):
    """Sketches with different scaled values and ``downsample=True``: the reference compares EVERY PAIR at
    max(scaled_i, scaled_j) -- `similarity(other, downsample=True)` / `count_common(other, True)` downsample
    the finer sketch of the pair (minhash.rs:539-547,682-702) -- not everything at the coarsest scaled of the
    list.  One batched call per distinct scaled value S over the sketches with scaled <= S, cut at S; the pairs
    whose coarser member has scaled S take their cells from that call.
    Returns dict(common=u32 (n,n), jaccard / angular = float64 (n,n) or None)."""
    h, off, ab = c["raw"]
    scaleds = np.asarray(c["orig_scaled"]).astype(np.int64)
    n = len(scaleds)
    out = {"common": np.zeros((n, n), dtype=np.uint32), "jaccard": np.ones((n, n)) if jaccard else None,
           "angular": np.ones((n, n)) if angular else None}
    for S, idx, lens, sub_h, sub_off, here in _scaled_groups(c):
        cells = np.ix_(idx, idx)

        def put(name, block):
            full = out[name][cells]
            full[here] = block[here]
            out[name][cells] = full
        sset = B.SketchSet.from_host(sub_h, sub_off)
        put("common", B.pairwise_common(sset))
        if jaccard:
            put("jaccard", B.compare_jaccard(sset))
        if angular:
            sub_ab = np.concatenate([ab[int(off[i]):int(off[i]) + m] for i, m in zip(idx, lens)])
            put("angular", B.compare_angular(B.SketchSet.from_host(sub_h, sub_off, sub_ab)))
    return out


def compare_all_pairs(siglist, ignore_abundance, *, downsample=False, n_jobs=None, return_ani=False):
    """Similarity matrix (n, n) float64, ones on the diagonal -- ``compare_all_pairs`` /
    ``compare_serial`` / ``compare_parallel`` of the reference (compare.py:14-64,241-358).
    ``n_jobs`` is accepted for signature compatibility; the GPU does the whole matrix."""
    n = len(siglist)
    if n == 0:
        return np.ones((0, 0))
    try:
        c = _collect(siglist, downsample=downsample, with_abunds=not ignore_abundance)
    except TypeError as exc:
        if return_ani or "incompatible num values" not in str(exc):
            raise
        # num sketches of different sizes (found by _collect without touching the objects one by one): the reference does
        # not refuse them, and what it computes depends on which side is `self` (the union is cut at self.num,
        # minhash.rs:596-617).  No batched form: its own loop, pair by pair through the ABI -- cells (i, j) and (j, i) both
        # take siglist[i].similarity(siglist[j]) for i < j (compare.py:36-54)
        mhs = _flat_minhashes(siglist)
        out = np.ones((n, n))
        for i in range(n):
            for j in range(i + 1, n):
                out[i][j] = out[j][i] = mhs[i].similarity(mhs[j], ignore_abundance=ignore_abundance, downsample=downsample)
        return out
    has_ab, num, scaled, sizes = c["has_abund"], c["num"], c["scaled"], c["sizes"]
    if c.get("raw") is not None:                         # different scaled values: every pair at its own max scaled
        if return_ani:
            ani, untrustworthy, false_neg = _mixed_ani(c, "jaccard")
            if untrustworthy:
                notify(_JACCARD_WARNING)
            if false_neg:
                notify(_FALSE_NEG_WARNING)
            return ani
        want_ang = not ignore_abundance and bool(has_ab.any())
        t = _mixed_pair_tables(c, jaccard=True, angular=want_ang)
        out = np.where(has_ab[:, None] & has_ab[None, :], t["angular"], t["jaccard"]) if want_ang else t["jaccard"]
        np.fill_diagonal(out, 1.0)
        return out
    if return_ani:
        accurate = _sizes_accurate_arrays(c["orig_sizes"], c["orig_scaled"])   # raises for num sketches, like jaccard_ani
    sset = B.SketchSet.from_host(c["hashes"], c["offsets"])
    jac = B.compare_jaccard(sset, num=num)
    if return_ani:
        # compare.py:36-54: ANI from Jaccard for every pair; untrustworthy estimates become 0
        ani, untrustworthy, false_neg = DU.jaccard_to_ani_matrix(jac, sizes, c["ksize"], scaled,
                                                                  size_accurate=accurate)
        if untrustworthy:
            notify(_JACCARD_WARNING)
        if false_neg:
            notify(_FALSE_NEG_WARNING)
        return ani
    if ignore_abundance or not has_ab.any():
        return jac
    # angular similarity where both sketches track abundance, Jaccard elsewhere (minhash.rs:682-702);
    # flat sketches carry abundance 1 in the abundance set (their cells are replaced by Jaccard)
    ang = B.compare_angular(B.SketchSet.from_host(c["hashes"], c["offsets"], c["abunds"]))
    both = has_ab[:, None] & has_ab[None, :]
    out = np.where(both, ang, jac)
    np.fill_diagonal(out, 1.0)
    return out


def compare_serial(siglist, ignore_abundance, *, downsample=False, return_ani=False):
    return compare_all_pairs(siglist, ignore_abundance, downsample=downsample, return_ani=return_ani)


def compare_parallel(siglist, ignore_abundance, downsample, n_jobs, return_ani=False):
    return compare_all_pairs(siglist, ignore_abundance, downsample=downsample, n_jobs=n_jobs, return_ani=return_ani)


def _bias_factors(sizes, scaled):
    """bias_factor(n) = 1 - (1 - 1/scaled) ** float(n * scaled), Python floats (minhash.py:830-833);
    `scaled` is one value or an array shaped like `sizes` (the scaled of the sketch whose method is called)."""
    sizes = np.asarray(sizes)
    scaleds = np.broadcast_to(np.asarray(scaled), sizes.shape)
    table = {}
    flat = np.empty(sizes.size, dtype=np.float64)
    for k, (n, sc) in enumerate(zip(sizes.ravel().tolist(), scaleds.ravel().tolist())):
        key = (int(n), int(sc))
        if key not in table:
            table[key] = 1.0 - (1.0 - 1.0 / key[1]) ** float(key[0] * key[1]) if key[0] else 1.0
        flat[k] = table[key]
    return flat.reshape(sizes.shape)


def _clamp01(m):
    m = np.where(m >= 1, 1.0, m)
    return np.where(m <= 0, 0.0, m)


class _MixedAni(Exception):
    "carries the finished ANI matrix of a list with different scaled values out of _containment_parts"


def _containment_parts(siglist, downsample, return_ani=False, kind="containment"):
    "(common counts as float64, sizes, scaled, ksize, size_is_accurate flags or None)"
    if not len(siglist):
        return None, np.zeros(0, np.int64), 0, 0, None
    c = _collect(siglist, downsample=downsample, need_scaled=True)
    if c.get("raw") is not None:
        # different scaled values: counts per pair at max(scaled_i, scaled_j) (count_common(other, downsample=True)),
        # while contained_by / max_containment keep len(self) and self.scaled of the sketches AS GIVEN in the
        # denominator (minhash.py:827-841,889-905); the ANI forms take everything from the downsampled pair (_mixed_ani)
        if return_ani:
            m, _untrustworthy, false_neg = _mixed_ani(c, kind)
            if false_neg:
                notify(_FALSE_NEG_WARNING)
            raise _MixedAni(m)
        common = _mixed_pair_tables(c)["common"].astype(np.float64)
        return common, c["orig_sizes"], np.asarray(c["orig_scaled"]).astype(np.int64), c["ksize"], None
    accurate = _sizes_accurate_arrays(c["orig_sizes"], c["orig_scaled"]) if return_ani else None
    sset = B.SketchSet.from_host(c["hashes"], c["offsets"])
    common = B.pairwise_common(sset).astype(np.float64)
    return common, c["sizes"], c["scaled"], c["ksize"], accurate


def compare_serial_containment(siglist, *, downsample=False, return_ani=False):
    """containments[i][j] = siglist[j].contained_by(siglist[i]) (compare.py:67-106); with
    ``return_ani`` the containment ANI of j in i (0.0 where it cannot be trusted)."""
    try:
        common, sizes, scaled, ksize, accurate = _containment_parts(siglist, downsample, return_ani)
    except _MixedAni as done:
        return done.args[0]
    n = len(sizes)
    if n == 0:
        return np.ones((0, 0))
    m, false_neg = _containment_block(common, sizes, scaled, ksize, accurate, return_ani)
    if false_neg:
        notify(_FALSE_NEG_WARNING)
    np.fill_diagonal(m, 1.0)
    return m


def _containment_block(common, sizes, scaled, ksize, accurate, return_ani, cells=None):
    "containment (or its ANI) of column sketch j in row sketch i from the common counts; (matrix, false-negative flag)"
    denom = sizes.astype(np.float64) * _bias_factors(sizes, scaled)       # per column j
    with np.errstate(divide="ignore", invalid="ignore"):
        m = common / denom[np.newaxis, :]
    m = _clamp01(m)
    m[:, sizes == 0] = 0.0
    if not return_ani:
        return m, False
    ani = DU.containment_to_ani_matrix(m, ksize, size_accurate_rows=accurate, size_accurate_cols=accurate)
    p = _p_nothing_in_common(1.0 - DU.containment_to_ani_matrix(m, ksize),
                             (sizes * scaled).astype(np.float64)[np.newaxis, :], ksize, scaled)
    np.fill_diagonal(p, 0.0)
    return ani, bool(((p > 1e-3) if cells is None else (p > 1e-3) & cells).any())


def _max_containment_block(common, sizes, scaled, ksize, accurate, return_ani, cells=None):
    "the same for max_containment with ONE scaled value: common / (min(|A|, |B|) * bias(min))"
    mins = np.minimum(sizes[:, None], sizes[None, :])
    flat = np.unique(mins.ravel())
    lut = dict(zip(flat.tolist(), _bias_factors(flat, scaled).tolist()))
    denom = mins.astype(np.float64) * np.vectorize(lut.get, otypes=[np.float64])(mins)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = common / denom
    m = _clamp01(m)
    m[mins == 0] = 0.0
    if not return_ani:
        return m, False
    ani = DU.containment_to_ani_matrix(m, ksize, size_accurate_rows=accurate, size_accurate_cols=accurate)
    p = _p_nothing_in_common(1.0 - DU.containment_to_ani_matrix(m, ksize), (mins * scaled).astype(np.float64), ksize, scaled)
    np.fill_diagonal(p, 0.0)
    return ani, bool(((p > 1e-3) if cells is None else (p > 1e-3) & cells).any())


def _mixed_ani(c, kind):
    """ANI matrices of sketches with different scaled values (``downsample=True``): jaccard_ani / containment_ani /
    max_containment_ani downsample BOTH sketches of a pair to max(scaled_i, scaled_j) and take every quantity -- the
    similarity, the sketch sizes, the scaled of the formulas -- from the downsampled pair (minhash.py:749-785,843-945);
    only size_is_accurate() is asked of the sketches as given (of the downsampled ones by avg_containment_ani, which the
    reference computes through FracMinHashComparison).  One batched call per distinct scaled value, the formulas
    of the one-scaled case on it, and every pair keeps the cell of its own scaled.
    Returns (matrix with a unit diagonal, jaccard-untrustworthy flag, false-negative flag)."""
    n = len(c["orig_scaled"])
    accurate = _sizes_accurate_arrays(c["orig_sizes"], c["orig_scaled"])
    out, untrustworthy, false_neg = np.ones((n, n)), False, False
    for S, idx, lens, sub_h, sub_off, here in _scaled_groups(c):
        sset = B.SketchSet.from_host(sub_h, sub_off)
        sizes, acc = np.asarray(lens, dtype=np.int64), accurate[idx]
        if kind == "jaccard":
            block, u, f = DU.jaccard_to_ani_matrix(B.compare_jaccard(sset), sizes, c["ksize"], S, size_accurate=acc, cells=here)
            untrustworthy |= u
        elif kind == "avg_containment":                     # mean of the two directed ANIs; accuracy of the downsampled pair
            acc = _sizes_accurate_arrays(sizes, np.full(len(sizes), S, dtype=np.int64))
            block, f = _containment_block(B.pairwise_common(sset).astype(np.float64), sizes, S, c["ksize"], acc, True, cells=here)
            block = np.where(acc[:, None] & acc[None, :], (block + block.T) / 2, 0.0)
        else:
            fn = _containment_block if kind == "containment" else _max_containment_block
            block, f = fn(B.pairwise_common(sset).astype(np.float64), sizes, S, c["ksize"], acc, True, cells=here)
        false_neg |= f
        cells = np.ix_(idx, idx)
        full = out[cells]
        full[here] = block[here]
        out[cells] = full
    np.fill_diagonal(out, 1.0)
    return out, untrustworthy, false_neg


def compare_serial_max_containment(siglist, *, downsample=False, return_ani=False):
    """max_containment matrix (compare.py:109-147): common / (min(|A|,|B|) * bias(min))."""
    try:
        common, sizes, scaled, ksize, accurate = _containment_parts(siglist, downsample, return_ani, kind="max_containment")
    except _MixedAni as done:
        return done.args[0]
    n = len(sizes)
    if n == 0:
        return np.ones((0, 0))
    mins = np.minimum(sizes[:, None], sizes[None, :])
    if np.ndim(scaled):
        # cell (i, j), i < j, is siglist[j].max_containment(siglist[i]): the bias uses the scaled of the sketch
        # with the HIGHER index (compare.py:131-140), mirrored into (j, i)
        hi = np.maximum(np.arange(n)[:, None], np.arange(n)[None, :])
        denom = mins.astype(np.float64) * _bias_factors(mins, np.asarray(scaled)[hi])
        with np.errstate(divide="ignore", invalid="ignore"):
            m = common / denom
        m = _clamp01(m)
        m[mins == 0] = 0.0
    else:
        m, false_neg = _max_containment_block(common, sizes, scaled, ksize, accurate, return_ani)
        if false_neg:
            notify(_FALSE_NEG_WARNING)
    np.fill_diagonal(m, 1.0)
    return m


def compare_serial_avg_containment(siglist, *, downsample=False, return_ani=False):
    """avg_containment matrix (compare.py:150-187): mean of the two directed containments; with
    ``return_ani`` the mean of the two containment ANIs, 0.0 if either cannot be trusted."""
    accurate = None
    if return_ani and len(siglist):
        c0 = _collect(siglist, downsample=True, need_scaled=True)           # (the ANI form downsamples whatever the flag says)
        if c0.get("raw") is not None:
            # different scaled values: the reference goes through FracMinHashComparison here (compare.py:150-187), which
            # downsamples the pair first and asks size_is_accurate() of the DOWNSAMPLED sketches (sketchcomparison.py:99-236)
            m, _untrustworthy, false_neg = _mixed_ani(c0, "avg_containment")
            if false_neg:
                notify(_FALSE_NEG_WARNING)
            return m
        accurate = _sizes_accurate_arrays(c0["orig_sizes"], c0["orig_scaled"])
    c = compare_serial_containment(siglist, downsample=downsample, return_ani=return_ani)
    m = (c + c.T) / 2
    if accurate is not None:
        m = np.where(accurate[:, None] & accurate[None, :], m, 0.0)
    np.fill_diagonal(m, 1.0)
    return m
