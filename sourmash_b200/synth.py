"""Deterministic synthetic workloads (SURVEY §8d configs), shared by tests and bench.py."""
import numpy as np

MAX_HASH_1000 = 18446744073709552


def synth_genome(length, seed, n_every=0, lower=False):
    """Uniform ACGT bytes from PCG64(seed) (config 2); optional N every n_every bases."""
    rng = np.random.Generator(np.random.PCG64(seed))
    codes = rng.integers(0, 4, size=length, dtype=np.uint8)
    lut = np.frombuffer(b"acgt" if lower else b"ACGT", dtype=np.uint8)
    seq = lut[codes]
    if n_every:
        seq = seq.copy()
        seq[n_every - 1::n_every] = ord("N")
    return seq


def synth_sketches(n, mean=5000, sd=500, lo=3000, hi=7000, n_families=100, pool=6000,
                   max_hash=MAX_HASH_1000, seed=0):
    """Config 3: n sketches in families sharing a hash pool.  Returns (hashes, offsets) CSR."""
    rng0 = np.random.Generator(np.random.PCG64(12345 + seed))
    sizes = np.clip(rng0.normal(mean, sd, size=n).round().astype(np.int64), lo, hi)
    pools = []
    for f in range(n_families):
        r = np.random.Generator(np.random.PCG64(2000 + f + 1000003 * seed))
        pools.append(np.unique(r.integers(1, max_hash, size=pool, dtype=np.uint64, endpoint=True)))
    rows = []
    for i in range(n):
        r = np.random.Generator(np.random.PCG64(3000 + i + 1000003 * seed))
        p = pools[i % n_families]
        frac = r.uniform(0.5, 0.95)
        take = min(int(frac * len(p)), int(sizes[i]))
        shared = r.choice(p, size=take, replace=False)
        extra = r.integers(1, max_hash, size=max(int(sizes[i]) - take, 0), dtype=np.uint64, endpoint=True)
        rows.append(np.unique(np.concatenate([shared, extra])))
    offsets = np.zeros(n + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(r) for r in rows])
    return np.concatenate(rows), offsets


def rows_of(hashes, offsets):
    return [hashes[int(offsets[i]):int(offsets[i + 1])] for i in range(len(offsets) - 1)]


# ---------------------------------------------------------------------------------------------------------
# configs[3] / configs[4]: large databases of uniform random sketches with a few rows planted from a query
# (SURVEY 8d).  1.5e9 hashes cannot be drawn and sorted row by row on the host in reasonable time, so a block
# of rows is produced on the GPU with torch when a device is at hand (one flat draw, two stable sorts); the
# numpy twin serves small sizes (CPU tests).  The two do not produce the same numbers -- every consumer takes
# the rows it was given as the truth -- but each is deterministic in its seeds, block by block, so that a
# rank of a multi-GPU run can build exactly its own rows of the same database.
# ---------------------------------------------------------------------------------------------------------
def database_plan(n_rows, seed, planted_frac=0.0, mean=5000, sd=500, lo=3000, hi=7000):
    """(sizes int64[n_rows], frac float64[n_rows]): row lengths ~ N(mean, sd) clipped; `planted_frac` of the rows
    draw 20-80 % of their hashes from the query (frac > 0), the others none."""
    rng = np.random.Generator(np.random.PCG64(seed))
    sizes = np.clip(rng.normal(mean, sd, size=n_rows).round().astype(np.int64), lo, hi)
    planted = rng.random(n_rows) < planted_frac
    frac = rng.uniform(0.2, 0.8, size=n_rows) * planted
    return sizes, frac


def _planted_indices(rng, k, nq):
    "k distinct ascending indices into a query of nq hashes"
    return np.sort(rng.integers(0, nq - k, size=k)) + np.arange(k)


def database_block(sizes, frac, query, row_begin, row_end, seed, max_hash=MAX_HASH_1000, overrides=None, torch=None,
                   device=None):
    """Rows [row_begin, row_end) of the database as one flat sorted-unique-per-row array, in the order of the rows.
    Returns a numpy uint64 array, or -- with `torch` and a CUDA `device` -- an int64 tensor on the device.
    `overrides` maps a row to the exact content it must have (its length must equal sizes[row])."""
    sz = sizes[row_begin:row_end]
    off = np.zeros(len(sz) + 1, dtype=np.int64)
    off[1:] = np.cumsum(sz)
    total = int(off[-1])
    rng = np.random.Generator(np.random.PCG64([seed, row_begin]))
    pos, qidx = [], []
    for i in np.nonzero(frac[row_begin:row_end] > 0)[0]:
        k = int(frac[row_begin + i] * sz[i])
        if k:
            pos.append(off[i] + np.arange(k))
            qidx.append(_planted_indices(rng, k, len(query)))
    pos = np.concatenate(pos) if pos else np.zeros(0, np.int64)
    qidx = np.concatenate(qidx) if qidx else np.zeros(0, np.int64)
    mine = {r: v for r, v in (overrides or {}).items() if row_begin <= r < row_end}
    if torch is None:
        vals = rng.integers(1, max_hash, size=total, dtype=np.uint64, endpoint=True)
        vals[pos] = np.asarray(query, dtype=np.uint64)[qidx]
        for i in range(len(sz)):
            vals[off[i]:off[i + 1]] = np.sort(vals[off[i]:off[i + 1]])
        for r, v in mine.items():
            assert len(v) == sz[r - row_begin]
            vals[off[r - row_begin]:off[r - row_begin + 1]] = v
        bad = (vals[1:] == vals[:-1])
        bad[off[1:-1] - 1] = False                               # the last element of a row vs the first of the next
        assert not bad.any(), "a synthetic row drew the same hash twice; change the seed"
        return vals
    gen = torch.Generator(device=device)
    gen.manual_seed(int(seed) * 1000003 + int(row_begin))
    vals = torch.randint(1, int(max_hash) + 1, (total,), dtype=torch.int64, device=device, generator=gen)
    if len(pos):
        qd = query if torch.is_tensor(query) else torch.from_numpy(np.asarray(query, dtype=np.uint64).view(np.int64)).to(device)
        vals[torch.from_numpy(pos).to(device)] = qd[torch.from_numpy(qidx).to(device)]
    rowid = torch.repeat_interleave(torch.arange(len(sz), dtype=torch.int32, device=device),
                                    torch.from_numpy(sz).to(device))
    vals, order = torch.sort(vals)                               # hashes are < 2^63: int64 order == u64 order
    rowid = rowid[order]
    del order
    rowid, order = torch.sort(rowid, stable=True)
    vals = vals[order]
    del order, rowid
    for r, v in mine.items():
        assert len(v) == sz[r - row_begin]
        vals[off[r - row_begin]:off[r - row_begin + 1]] = torch.from_numpy(np.asarray(v, dtype=np.uint64).view(np.int64)).to(device)
    dup = vals[1:] == vals[:-1]
    dup[torch.from_numpy(off[1:-1] - 1).to(device)] = False
    assert not bool(dup.any()), "a synthetic row drew the same hash twice; change the seed"
    return vals


def search_query(n_query=10_000_000, seed=4000, max_hash=MAX_HASH_1000):
    "configs[3]: 1e7 hashes uniform in [1, max_hash], sorted-unique"
    rng = np.random.Generator(np.random.PCG64(seed))
    return np.unique(rng.integers(1, max_hash, size=n_query, dtype=np.uint64, endpoint=True))


def gather_workload(n_db, seed=5000, n_clusters=20, members=10, pool=6000, noise=20_000, max_hash=MAX_HASH_1000):
    """configs[4]: a metagenome query of ~1e5 hashes and the planted rows of the database: `n_clusters` x `members`
    genomes, the members of a cluster sharing 70-95 % of a pool (so that picking one shrinks the others' overlap).
    Returns (query, sizes, frac (all zero), overrides {row: hashes})."""
    rng = np.random.Generator(np.random.PCG64(seed))
    sizes, frac = database_plan(n_db, seed + 1)
    rows_at = rng.choice(n_db, size=n_clusters * members, replace=False)
    overrides, parts = {}, []
    for c in range(n_clusters):
        p = np.unique(rng.integers(1, max_hash, size=pool, dtype=np.uint64, endpoint=True))
        for m in range(members):
            row = int(rows_at[c * members + m])
            take = rng.choice(p, size=int(rng.uniform(0.7, 0.95) * len(p)), replace=False)
            own = rng.integers(1, max_hash, size=max(int(sizes[row]) - len(take), 0), dtype=np.uint64, endpoint=True)
            v = np.unique(np.concatenate([take, own]))
            sizes[row] = len(v)
            overrides[row] = v
            parts.append(v[rng.random(len(v)) < 0.6])
    parts.append(rng.integers(1, max_hash, size=noise, dtype=np.uint64, endpoint=True))
    return np.unique(np.concatenate(parts)), sizes, frac * 0.0, overrides


def multigather_workload(n_db, n_queries, seed=5000):
    """configs[4] for many samples: the queries of gather_workload under n_queries seeds and ONE database of n_db rows
    holding the planted rows of all of them (a row planted by two queries keeps the content the later one gave it).
    Returns (queries, sizes, frac (all zero), overrides {row: hashes}) for database_block."""
    sizes, frac = database_plan(n_db, seed + 1)
    queries, overrides = [], {}
    for i in range(n_queries):
        q, _, _, planted = gather_workload(n_db, seed=seed + 7919 * i)
        queries.append(q)
        for row, v in planted.items():
            overrides[row] = v
            sizes[row] = len(v)
    return queries, sizes, frac * 0.0, overrides
