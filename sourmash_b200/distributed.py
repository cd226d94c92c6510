"""Multi-GPU plumbing (one process per GPU, torch.distributed; NCCL on GPUs, gloo in CPU tests).

The reference has no distributed path at all (SURVEY 2a); sharding follows SURVEY 8e:
  * sketching shards by genome, followed by ONE variable-length all-gather of the shards (`ShardGather`);
  * compare all-gathers the sketches, splits the HASH SPACE into key ranges -- rank r sorts, tags and counts
    only the hashes of range r, for whole rows -- sums the partial counters with one reduce-scatter by row block
    and finalises its block of rows (`CompareShard`);
  * search / gather shard the database by subject (`ShardedDatabase`).
Host-side logic (shard bounds, padded all-gather + compaction, offsets, tie breaks) is backend agnostic and is
what the gloo tests exercise; the compute calls need a GPU.
"""
import numpy as np


def shard_bounds(n, world):
    """Contiguous row blocks: rank r owns rows [b[r], b[r+1])."""
    return [n * r // world for r in range(world + 1)]


class ShardGather:
    """Variable-length all-gather of CSR shards (rank order == row order) with the bookkeeping done ONCE: the
    sizes of the shards are exchanged at construction (one small collective and one host read), after which
    `gather()` is a single all-gather of padded hash blocks plus `world` device-to-device slice copies -- no
    host synchronisation in the step.  Row lengths are known on the host when sketches exist (they are the CSR
    offsets), so the exchange belongs to setting the job up."""

    def __init__(self, torch, dist, n_local_hashes, local_sizes, device):
        self.torch, self.dist, self.device = torch, dist, device
        world = dist.get_world_size()
        sizes = np.asarray(local_sizes, dtype=np.int64)
        meta = torch.tensor([int(n_local_hashes), len(sizes)], dtype=torch.int64, device=device)
        metas = torch.empty(2 * world, dtype=torch.int64, device=device)
        dist.all_gather_into_tensor(metas, meta)
        metas = metas.cpu().numpy().reshape(world, 2)
        self.n_hashes, self.n_rows = metas[:, 0].copy(), metas[:, 1].copy()
        self.pad_h = max(int(self.n_hashes.max()), 1)
        pad_r = max(int(self.n_rows.max()), 1)
        mine = torch.zeros(pad_r, dtype=torch.int64, device=device)
        mine[: len(sizes)] = torch.from_numpy(sizes).to(device)
        all_s = torch.empty(world * pad_r, dtype=torch.int64, device=device)
        dist.all_gather_into_tensor(all_s, mine)
        all_s = all_s.cpu().numpy().reshape(world, pad_r)
        self.sizes = np.concatenate([all_s[r, : self.n_rows[r]] for r in range(world)]) if world else sizes
        self.offsets = np.zeros(len(self.sizes) + 1, dtype=np.uint64)
        self.offsets[1:] = np.cumsum(self.sizes)
        self.total = int(self.n_hashes.sum())
        self.d_offsets = torch.from_numpy(self.offsets.view(np.int64)).to(device)
        self.hashes = torch.empty(max(self.total, 1), dtype=torch.int64, device=device)
        starts = np.concatenate([[0], np.cumsum(self.n_hashes)])
        # Two ranks: every shard lands where it belongs in the gathered array -- the views of an all_gather with shards of
        # different sizes (NCCL: one grouped broadcast per rank straight into its view; no padding, no compaction copy).
        # That suits two ranks; with more, N broadcasts are no match for one all-gather of equal blocks through the
        # switch, so from four ranks on the shards travel as padded equal blocks and are compacted locally.
        self._views = [self.hashes[int(starts[r]):int(starts[r + 1])] for r in range(world)]
        self._uneven_ok = dist.get_backend() == "nccl" and world <= 2 and all(int(x) > 0 for x in self.n_hashes)
        if not self._uneven_ok:                           # >= 4 ranks / gloo (CPU tests) / an empty shard: padded blocks + compaction
            self._padded = torch.zeros(self.pad_h, dtype=torch.int64, device=device)
            self._all = torch.empty(world * self.pad_h, dtype=torch.int64, device=device)

    def gather(self, local_hashes):
        "all ranks' hashes, compacted, in `self.hashes[:total]` (int64 view of the u64 hashes)"
        world = len(self.n_hashes)
        if self._uneven_ok:
            self.dist.all_gather(self._views, local_hashes)
            return self.hashes[: self.total]
        pad = self.pad_h
        self._padded[: local_hashes.numel()] = local_hashes
        self.dist.all_gather_into_tensor(self._all, self._padded)
        pos = 0
        for r in range(world):
            nh = int(self.n_hashes[r])
            self.hashes[pos:pos + nh] = self._all[r * pad: r * pad + nh]
            pos += nh
        return self.hashes[: self.total]


def allgather_csr(torch, dist, local_hashes, local_sizes, device):
    """One-shot form of ShardGather: returns (hashes int64 tensor [total], sizes int64 numpy [n_rows_total])."""
    sizes = local_sizes.cpu().numpy() if hasattr(local_sizes, "cpu") else np.asarray(local_sizes)
    g = ShardGather(torch, dist, local_hashes.numel(), sizes, device)
    return g.gather(local_hashes), g.sizes


def allgather_sketchset(torch, dist, B, sset, cache=None):
    """All-gather a per-rank SketchSet into a full SketchSet on every rank.  `cache` (a dict the caller keeps) holds
    the ShardGather of a step that repeats with the same shard sizes."""
    device = torch.device("cuda", torch.cuda.current_device())
    off = sset.offsets()
    sizes = np.diff(off.astype(np.int64))
    key = (int(off[-1]), len(sizes))
    g = cache.get("g") if cache is not None and cache.get("key") == key and np.array_equal(cache.get("sizes"), sizes) else None
    if g is None:
        g = ShardGather(torch, dist, int(off[-1]), sizes, device)
        if cache is not None:
            cache.update(g=g, key=key, sizes=sizes, local=torch.empty(max(int(off[-1]), 1), dtype=torch.int64, device=device))
    local = cache["local"] if cache is not None else torch.empty(max(int(off[-1]), 1), dtype=torch.int64, device=device)
    sset.copy_to_device(local.data_ptr())
    hashes = g.gather(local[: int(off[-1])])
    return B.SketchSet.from_device(hashes.data_ptr(), g.d_offsets.data_ptr(), g.offsets, keepalive=(hashes, g.d_offsets, g))


class CompareShard:
    """One rank's part of an N-GPU all-vs-all compare.

    step(): (1) all-gather of the sketch shards (as if every rank had sketched its own genomes); (2) this rank's
    KEY RANGE of the hash space: sort, tags and whole-row counting of the hashes in range `rank` only
    (smb_compare_counts_shard_dev) -- every stage shrinks with 1 / world; (3) one reduce-scatter of the partial
    counters by row block (the only exchange of results: (world - 1) / world of n^2 * 2 bytes per rank with 16-bit
    counters, * 4 with 32-bit ones);
    (4) float64 Jaccard rows of this rank's block.  gloo has no reduce-scatter: all-reduce + slice there."""

    def __init__(self, torch, dist, B, hashes, offsets, rank, world):
        self.torch, self.dist, self.B, self.rank, self.world = torch, dist, B, rank, world
        n = len(offsets) - 1
        self.n = n
        self.bounds = shard_bounds(n, world)
        lo, hi = self.bounds[rank], self.bounds[rank + 1]
        self.device = torch.device("cuda", torch.cuda.current_device())
        local = hashes[int(offsets[lo]):int(offsets[hi])].view(np.int64)
        sizes = np.diff(offsets.astype(np.int64))[lo:hi]
        self.pin_h = torch.from_numpy(local.copy()).pin_memory()
        self.d_local = self.pin_h.to(self.device)
        self.gatherer = ShardGather(torch, dist, len(local), sizes, self.device)
        self.per = max(b1 - b0 for b0, b1 in zip(self.bounds[:-1], self.bounds[1:]))      # rows per reduce-scatter block
        self.even = all(b1 - b0 == self.per for b0, b1 in zip(self.bounds[:-1], self.bounds[1:]))
        rows_padded = self.per * world if self.even else n
        # 16-bit counters when every sketch is shorter than 65 536 hashes (a count never exceeds the shorter row): half
        # the bytes through NVLink.  The reduce-scatter adds them two at a time as int32 -- sums stay below 65 536, so
        # nothing carries from one counter into its neighbour.
        self.bits = 16 if (n % 2 == 0 and int(self.gatherer.sizes.max() if len(self.gatherer.sizes) else 0) < 65536) else 32
        cdtype = torch.int16 if self.bits == 16 else torch.int32
        self.d_partial = torch.zeros((rows_padded, n), dtype=cdtype, device=self.device)
        self.d_counts = torch.zeros((self.per, n), dtype=cdtype, device=self.device)
        self.d_out = torch.empty((hi - lo, n), dtype=torch.float64, device=self.device)
        self.pin_out = torch.empty((hi - lo, n), dtype=torch.float64).pin_memory()
        self.h2d_bytes = int(local.nbytes + sizes.nbytes)
        self.d2h_bytes = int((hi - lo) * n * 8)

    def step(self, e2e):
        torch, dist, B = self.torch, self.dist, self.B
        if e2e:
            self.d_local.copy_(self.pin_h, non_blocking=True)
        g = self.gatherer
        hashes = g.gather(self.d_local)
        sset = B.SketchSet.from_device(hashes.data_ptr(), g.d_offsets.data_ptr(), g.offsets, keepalive=(hashes, g.d_offsets))
        lo, hi = self.bounds[self.rank], self.bounds[self.rank + 1]
        B.compare_counts_shard_device(sset, self.rank, self.world, self.d_partial.data_ptr(), bits=self.bits)
        wide = (lambda t: t.view(torch.int32)) if self.bits == 16 else (lambda t: t)
        if self.even and dist.get_backend() == "nccl":
            dist.reduce_scatter_tensor(wide(self.d_counts), wide(self.d_partial))
            counts = self.d_counts
        else:                                               # uneven blocks / gloo: sum everything, keep this rank's rows
            dist.all_reduce(wide(self.d_partial))
            counts = self.d_partial[lo:hi].contiguous()
        B.finalize_counts_rows_device(sset, counts.data_ptr(), lo, hi, self.d_out.data_ptr(), bits=self.bits)
        if e2e:
            self.pin_out.copy_(self.d_out, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return float(self.pin_out[0, 1 if self.n > 1 else 0])
        return None


class ShardedDatabase:
    """A sketch database sharded by subject over the ranks (SURVEY §8e): every rank keeps its
    block of rows in HBM; a query is replicated.

    * ``search_counts(query)``: local one-vs-many, then one all-gather of the u32 counts.
    * ``gather(query, threshold)``: the CounterGather rounds with two tiny collectives per
      round -- all-gather of (best count, global row), broadcast of the winner's intersection.
    Works with any backend for the collectives (NCCL on GPUs; tensors for gloo live on the CPU).
    """

    def __init__(self, torch, dist, B, local_rows_sset, n_rows_total, row_begin):
        self.torch, self.dist, self.B = torch, dist, B
        self.sset, self.n_total, self.row_begin = local_rows_sset, n_rows_total, row_begin
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" \
            else torch.device("cpu")

    def build_index(self):
        "Inverted index of this rank's block of rows (batch.SketchSet.build_index): counts and gather rounds probe it."
        return self.sset.build_index() if len(self.sset) else 0

    def _shard_sizes(self):
        "rows per rank (one small collective, cached: the sharding of a resident database does not change)"
        if getattr(self, "_sizes", None) is None:
            torch, dist = self.torch, self.dist
            mine = torch.tensor([len(self.sset), int(self.sset.sizes().max()) if len(self.sset) else 0],
                                dtype=torch.int64, device=self.device)
            allv = torch.empty(2 * self.world, dtype=torch.int64, device=self.device)
            dist.all_gather_into_tensor(allv, mine)
            allv = allv.cpu().numpy().reshape(self.world, 2)
            self._sizes, self._max_row = allv[:, 0].copy(), int(allv[:, 1].max())
        return self._sizes

    def search_counts(self, query):
        "|query ∩ S_j| for every row of the whole database, on every rank (host arrays in and out)."
        torch, dist = self.torch, self.dist
        all_sizes = self._shard_sizes()
        local = self.B.one_vs_many(query, self.sset).astype(np.int32)
        pad = torch.zeros(max(int(all_sizes.max()), 1), dtype=torch.int32, device=self.device)
        pad[: len(local)] = torch.from_numpy(local).to(self.device)
        out = torch.empty(self.world * pad.numel(), dtype=torch.int32, device=self.device)
        dist.all_gather_into_tensor(out, pad)
        out = out.cpu().numpy().reshape(self.world, -1)
        return np.concatenate([out[r, : all_sizes[r]] for r in range(self.world)]).astype(np.uint32)

    def search_counts_device(self, d_query, d_local_counts, d_all_counts=None):
        """The same with the query (int64 view of the sorted u64 hashes) and the counters resident on the device: the
        local pass writes `d_local_counts` (int32 [local rows]); with `d_all_counts` (int32 [world * max local rows])
        one all-gather of equally sized blocks follows (shards of shard_bounds() differ by at most one row; a rank with
        fewer rows leaves its last slot unused).  No host round trip."""
        self.B.one_vs_many_device(d_query.data_ptr(), d_query.numel(), self.sset, d_local_counts.data_ptr())
        if d_all_counts is not None:
            self.dist.all_gather_into_tensor(d_all_counts, d_local_counts)
        return d_all_counts

    REPLICATE_LIMIT = 1 << 26            # hashes: candidate rows are replicated when together they are smaller than this

    def gather(self, query, threshold=1, max_rounds=None):
        """Returns (global match rows, intersect sizes) in pick order -- identical on every rank.

        The expensive part of gather is the prefetch pass over the database, and that is what the shards divide.  The
        rounds only ever touch the rows whose overlap reached the threshold (CounterGather holds prefetch matches only,
        index/__init__.py:302-320) -- typically a few hundred genomes -- so those rows are all-gathered once (their
        global ids, lengths and hashes) and every rank runs the rounds on its own copy: identical picks everywhere, no
        collective inside the loop.  Only when the candidates are a large part of the database does the loop stay
        sharded (`gather_sharded_rounds`: one collective per round)."""
        torch, dist = self.torch, self.dist
        threshold = max(int(threshold), 1)
        counts = self.B.one_vs_many(query, self.sset) if len(self.sset) else np.zeros(0, np.uint32)
        cand = np.nonzero(counts >= threshold)[0].astype(np.uint32)
        sizes = np.asarray(self.sset.sizes(), dtype=np.int64)[cand] if len(cand) else np.zeros(0, np.int64)
        meta = torch.tensor([len(cand), int(sizes.sum())], dtype=torch.int64, device=self.device)
        metas = torch.empty(2 * self.world, dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(metas, meta)
        metas = metas.cpu().numpy().reshape(self.world, 2)
        if int(metas[:, 1].sum()) > self.REPLICATE_LIMIT:
            return self.gather_sharded_rounds(query, threshold, max_rounds)
        if int(metas[:, 0].sum()) == 0:
            return np.zeros(0, np.uint32), np.zeros(0, np.uint32)
        # one padded all-gather: [global ids | lengths | hashes] of this rank's candidates
        pad_r, pad_h = max(int(metas[:, 0].max()), 1), max(int(metas[:, 1].max()), 1)
        rec = np.zeros(2 * pad_r + pad_h, dtype=np.int64)
        rec[: len(cand)] = cand.astype(np.int64) + self.row_begin
        rec[pad_r: pad_r + len(cand)] = sizes
        if len(cand):
            hh, _ = self.sset.take_rows(cand).to_host()
            rec[2 * pad_r: 2 * pad_r + len(hh)] = np.asarray(hh, dtype=np.uint64).view(np.int64)
        mine = torch.from_numpy(rec).to(self.device)
        allv = torch.empty(self.world * len(rec), dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(allv, mine)
        allv = allv.cpu().numpy().reshape(self.world, len(rec))
        ids, lens, parts = [], [], []
        for r in range(self.world):                       # rank order == global row order (contiguous shards)
            nr, nh = int(metas[r, 0]), int(metas[r, 1])
            ids.append(allv[r, :nr])
            lens.append(allv[r, pad_r: pad_r + nr])
            parts.append(allv[r, 2 * pad_r: 2 * pad_r + nh])
        ids, lens = np.concatenate(ids), np.concatenate(lens)
        off = np.zeros(len(ids) + 1, dtype=np.uint64)
        off[1:] = np.cumsum(lens)
        cset = self.B.SketchSet.from_host(np.concatenate(parts).view(np.uint64), off)
        picks, isect = self.B.gather(query, cset, threshold=threshold, max_rounds=max_rounds)
        return ids[np.asarray(picks, dtype=np.int64)].astype(np.uint32), np.asarray(isect, dtype=np.uint32)

    def gather_sharded_rounds(self, query, threshold=1, max_rounds=None):
        """The rounds with the counters left sharded (used when the candidates are too many to replicate).
        One collective per round: every rank contributes a fixed-size record (best count, global row, the row's
        intersection with the remaining query); the host of every rank reads the records once, picks the winner
        (largest count, lowest global row on ties == first inserted in the reference's Counter) and applies the
        winner's intersection to its own counters."""
        torch, dist = self.torch, self.dist
        threshold = max(int(threshold), 1)
        self._shard_sizes()
        rec_len = 3 + max(self._max_row, 1)
        session = self.B.GatherSession(query, self.sset, threshold)
        ids, sizes = [], []
        max_rounds = self.n_total if max_rounds is None else max_rounds
        rec = torch.zeros(rec_len, dtype=torch.int64, device=self.device)
        all_rec = torch.empty(self.world * rec_len, dtype=torch.int64, device=self.device)
        while len(ids) < max_rounds:
            cnt, row = session.peek() if len(self.sset) else (0, 0)
            host_rec = np.zeros(rec_len, dtype=np.int64)
            host_rec[0], host_rec[1] = cnt, self.row_begin + row
            if cnt >= threshold:
                isect = np.asarray(session.intersect(row), dtype=np.uint64)
                host_rec[2] = len(isect)
                host_rec[3:3 + len(isect)] = isect.view(np.int64)
            rec.copy_(torch.from_numpy(host_rec))
            dist.all_gather_into_tensor(all_rec, rec)
            recs = all_rec.cpu().numpy().reshape(self.world, rec_len)
            best = int(recs[:, 0].max())
            if best < threshold:
                break
            cand = np.nonzero(recs[:, 0] == best)[0]
            owner = int(cand[np.argmin(recs[cand, 1])])
            grow, n_isect = int(recs[owner, 1]), int(recs[owner, 2])
            isect = recs[owner, 3:3 + n_isect].copy().view(np.uint64)
            ids.append(grow)
            sizes.append(n_isect)
            if session.apply(isect) == 0:
                break
        return np.array(ids, dtype=np.uint32), np.array(sizes, dtype=np.uint32)
