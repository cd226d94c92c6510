// tile_kernels.cuh -- the pair-by-pair intersection kernels (pairwise_tile_split_kernel and its u64 predecessor),
// their argument block and the planner that sizes the shared-memory tables.  In a header so that
// tests/host_emul/simt_emul.cu can run the kernels themselves on the CPU (tests/host_emul/simt.h) against the
// oracle; compare_kernels.cu includes it for the product and keeps the launchers.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "split_table.cuh"

namespace smb {

static constexpr int TILE_THREADS_MAX = 1024;
static constexpr int MAX_DYN_SMEM = 227 * 1024;

// Bucket = key >> shift with buckets 0 .. (max_key >> shift): the directory covers exactly the
// occupied key range, and shift is the finest one whose directory still fits next to the keys.
// Prefer more tables per CTA (fewer passes over the streamed rows) as long as the buckets stay
// sparse (<= ~0.45 keys per bucket at the largest row), because denser buckets mean the
// deferred long-bucket scan runs in nearly every batch.
inline PairwisePlan plan_pairwise_impl(uint64_t max_len_a, uint64_t max_key, int cols_override) {
    PairwisePlan p{};
    uint64_t cap = (max_len_a + 1 + 3) & ~3ULL;          // +1: room even if a row is empty
    if (cap < 64) cap = 64;
    const size_t key_bytes = (cap + 2) * 8;
    auto config = [&](int ta, int& shift, uint64_t& nb) -> bool {
        const size_t per_table = (size_t)MAX_DYN_SMEM / ta;
        if (per_table < key_bytes + 64) return false;
        const uint64_t max_entries = std::min<uint64_t>((per_table - key_bytes) / 2 - 2, 60000);
        shift = 0;
        while (shift < 63 && (max_key >> shift) >= max_entries) ++shift;   // (no +1: max_key may be 2^64-1)
        nb = (max_key >> shift) + 1;
        return nb <= max_entries;
    };
    int best_ta = 0, best_shift = 0;
    uint64_t best_nb = 0;
    for (int ta = 4; ta >= 1; --ta) {
        int sh; uint64_t nb;
        if (!config(ta, sh, nb)) continue;
        if (best_ta == 0) { best_ta = ta; best_shift = sh; best_nb = nb; }      // densest acceptable fallback
        if ((double)cap / (double)nb <= 0.45 || sh == 0) { best_ta = ta; best_shift = sh; best_nb = nb; break; }
        best_ta = ta; best_shift = sh; best_nb = nb;                             // keep the sparsest seen so far
    }
    if (best_ta == 0) { p.tables_per_cta = 0; return p; }                        // row too large for smem
    p.tables_per_cta = best_ta; p.shift = best_shift; p.nb = (int)best_nb; p.cap = (int)cap;
    p.smem_bytes = (size_t)best_ta * (key_bytes + (best_nb + 2) * 2);
    p.cols_per_cta = cols_override > 0 ? cols_override : 512;
    return p;
}

struct TileArgs {
    const u64* hA; const u64* offA; int nA;
    const u64* hB; const u64* offB; int nB;
    u32* out; size_t ldo;
    int shift, nb, cap, cols_per_cta, symmetric;
    int tile_offset, tile_stride;       // row tile = blockIdx.x * tile_stride + tile_offset
    int tile_count;                     // >= 0: launch at most this many tiles
};

// Directory entries are u16.  When every table row has < 16384 keys (OCC), the top two bits
// carry min(bucket occupancy, 3) so the probe knows, without touching the keys, whether more
// than two keys share the bucket; otherwise the entry is the plain start index and the
// "more keys" test is k1 < q.
template <int TA, bool OCC>
__device__ __forceinline__ void probe_fast(u64 q, u32 b, const u64* const (&keys)[TA],
                                           const u16* const (&dirs)[TA], u32 (&cnt)[TA], u32 valid,
                                           u32& pend, int ubit) {
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        const u32 ent = dirs[t][b];
        const u32 st = OCC ? (ent & 0x3fffu) : ent;
        const u64* kp = keys[t] + st;
        const u64 k0 = kp[0], k1 = kp[1];
        const u32 m = (k0 == q) | (k1 == q);
        cnt[t] += m & valid;
        const bool more = OCC ? (ent >= 0xC000u) : (k1 < q);
        if (more && valid) pend |= 1u << (ubit * TA + t);      // predicated OR, no branch
    }
}

// rare: a bucket holds more than two keys below/at q -- continue the scan past the two
// keys the fast path already compared
template <int TA, bool OCC>
__device__ __forceinline__ void probe_rest(u64 q, u32 b, int t, const u64* const (&keys)[TA],
                                           const u16* const (&dirs)[TA], u32 (&cnt)[TA]) {
    const u32 ent = dirs[t][b];
    const u32 st = OCC ? (ent & 0x3fffu) : ent;
    const u64* pp = keys[t] + st + 2;
    u64 kk;
    while ((kk = *pp) < q) ++pp;
    cnt[t] += (kk == q);
}

template <int TA, int U, bool OCC>
__global__ void __launch_bounds__(TILE_THREADS_MAX, 1) pairwise_tile_kernel(TileArgs a) {
    SMB_DYN_SHARED(unsigned char, smem_raw);
    const int i0 = (blockIdx.x * a.tile_stride + a.tile_offset) * TA;
    int jbeg = blockIdx.y * a.cols_per_cta;
    int jend = min(jbeg + a.cols_per_cta, a.nB);
    if (a.symmetric) jbeg = max(jbeg, i0 + 1);
    if (jbeg >= jend) return;

    const u32 shift = (u32)a.shift;
    const int nb = a.nb;                      // buckets 0 .. nb-1; dir has nb+1 entries
    const int tid = threadIdx.x;
    const int nthreads = blockDim.x;
    const int kstride = a.cap + 2;
    const int dstride = nb + 2;
    u64* keys_base = reinterpret_cast<u64*>(smem_raw);
    u16* dirs_base = reinterpret_cast<u16*>(smem_raw + (size_t)TA * kstride * 8);

    SMB_SHARED int s_n[TA];
    SMB_SHARED int s_hasmax[TA];

    // ---- load table rows (coalesced), strip a trailing UINT64_MAX key, add sentinels
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        int i = i0 + t;
        u64 beg = 0; int n = 0; int hm = 0;
        if (i < a.nA) {
            beg = a.offA[i];
            n = (int)(a.offA[i + 1] - beg);
            if (n > 0 && ld_nc_u64(a.hA + beg + n - 1) == SMB_U64_MAX) { --n; hm = 1; }
        }
        u64* kt = keys_base + (size_t)t * kstride;
        for (int p = tid; p < n; p += nthreads) kt[p] = ld_nc_u64(a.hA + beg + p);
        if (tid < 2) kt[n + tid] = SMB_U64_MAX;
        if (tid == 0) { s_n[t] = n; s_hasmax[t] = hm; }
        // directory default: "no key at or after this bucket" (= n); overwritten below up to the
        // bucket of the row's last key
        u16* dt = dirs_base + (size_t)t * dstride;
        for (int b = tid; b <= nb; b += nthreads) dt[b] = (u16)n;
    }
    __syncthreads();
    // ---- build directories: dir[b] = #keys with bucket < b, b in [0, nb]
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        const u64* kt = keys_base + (size_t)t * kstride;
        u16* dt = dirs_base + (size_t)t * dstride;
        int n = s_n[t];
        for (int p = tid; p < n; p += nthreads) {
            int bp = (int)(kt[p] >> shift);
            int bprev = p == 0 ? -1 : (int)(kt[p - 1] >> shift);
            for (int b = bprev + 1; b <= bp; ++b) dt[b] = (u16)p;
        }
    }
    __syncthreads();
    if (OCC) {          // fold min(occupancy, 3) into the top two bits
#pragma unroll
        for (int t = 0; t < TA; ++t) {
            u16* dt = dirs_base + (size_t)t * dstride;
            for (int b = tid; b < nb; b += nthreads) {
                u32 st = dt[b] & 0x3fffu, en = dt[b + 1] & 0x3fffu;
                u32 occ = en - st;
                dt[b] = (u16)(st | ((occ > 3u ? 3u : occ) << 14));
            }
        }
        __syncthreads();
    }

    const u64* keys[TA];
    const u16* dirs[TA];
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        keys[t] = keys_base + (size_t)t * kstride;
        dirs[t] = dirs_base + (size_t)t * dstride;
    }

    // ---- stream columns: one warp per streamed row
    const int warp = tid >> 5, lane = tid & 31;
    const int NWARPS = nthreads >> 5;
    for (int j = jbeg + warp; j < jend; j += NWARPS) {
        const u64 bbeg = a.offB[j];
        int nbj = (int)(a.offB[j + 1] - bbeg);
        int bmax = 0;
        if (nbj > 0 && ld_nc_u64(a.hB + bbeg + nbj - 1) == SMB_U64_MAX) { --nbj; bmax = 1; }
        const u64* row = a.hB + bbeg;
        u32 cnt[TA];
#pragma unroll
        for (int t = 0; t < TA; ++t) cnt[t] = 0;

        int base = 0;
        const int full = nbj - (nbj % (32 * U));
        u64 q[U];
        if (full > 0) {
#pragma unroll
            for (int u = 0; u < U; ++u) q[u] = ld_nc_u64(row + u * 32 + lane);
        }
        for (; base < full; base += 32 * U) {
            u64 cur[U];
#pragma unroll
            for (int u = 0; u < U; ++u) cur[u] = q[u];
            if (base + 32 * U < full) {       // prefetch next batch before probing this one
#pragma unroll
                for (int u = 0; u < U; ++u) q[u] = ld_nc_u64(row + base + 32 * U + u * 32 + lane);
            }
            u32 pend = 0;
#pragma unroll
            for (int u = 0; u < U; ++u)
                probe_fast<TA, OCC>(cur[u], (u32)(cur[u] >> shift), keys, dirs, cnt, 1u, pend, u);
            if (pend) {
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int t = 0; t < TA; ++t)
                        if (pend & (1u << (u * TA + t)))
                            probe_rest<TA, OCC>(cur[u], (u32)(cur[u] >> shift), t, keys, dirs, cnt);
            }
        }
        for (; base < nbj; base += 32) {      // ragged tail
            int e = base + lane;
            u32 valid = e < nbj;
            u64 qq = valid ? ld_nc_u64(row + e) : 0ULL;
            u32 pend = 0;
            probe_fast<TA, OCC>(qq, (u32)(qq >> shift), keys, dirs, cnt, valid, pend, 0);
            if (pend) {
#pragma unroll
                for (int t = 0; t < TA; ++t)
                    if (pend & (1u << t)) probe_rest<TA, OCC>(qq, (u32)(qq >> shift), t, keys, dirs, cnt);
            }
        }
#pragma unroll
        for (int t = 0; t < TA; ++t) {
            u32 c = __reduce_add_sync(0xffffffffu, cnt[t]);
            int i = i0 + t;
            if (lane == 0 && i < a.nA && (!a.symmetric || j > i))
                a.out[(size_t)i * a.ldo + j] = c + (u32)(s_hasmax[t] & bmax);
        }
    }
}

// ------------------------------------------------------------------------------------
// Split-word variant of the tile kernel (rows < 32760 keys, i.e. everything that fits).  The v1 kernel above is bound
// by the SM's shared-memory wavefront rate, two LDS.64 per probe being the bulk.
// Here the table keeps the low and high 32-bit halves of the keys in separate arrays: the
// fast path touches only the low words (two LDS.32, ~1/2 the wavefronts) and remembers, per
// probe, where a low word matched; the high words are read only for those probes, inside a
// warp-uniform branch that unrelated pairs never enter.  Exact: a low-word match is always
// verified against the high word (both slots if both low words match).
// ------------------------------------------------------------------------------------
template <int TA, int U>
__global__ void __launch_bounds__(TILE_THREADS_MAX, 1) pairwise_tile_split_kernel(TileArgs a) {
    SMB_DYN_SHARED(unsigned char, smem_raw);
    const int i0 = (blockIdx.x * a.tile_stride + a.tile_offset) * TA;
    int jbeg = blockIdx.y * a.cols_per_cta;
    int jend = min(jbeg + a.cols_per_cta, a.nB);
    if (a.symmetric) jbeg = max(jbeg, i0 + 1);
    if (jbeg >= jend) return;

    const u32 shift = (u32)a.shift;
    const int nb = a.nb;
    const int tid = threadIdx.x;
    const int nthreads = blockDim.x;
    const int kstride = a.cap + 2;                       // same footprint as the u64 layout
    const int dstride = nb + 2;
    u32* lo_base = reinterpret_cast<u32*>(smem_raw);
    u32* hi_base = lo_base + (size_t)TA * kstride;
    u16* dirs_base = reinterpret_cast<u16*>(smem_raw + (size_t)TA * kstride * 8);

    SMB_SHARED int s_n[TA];
    SMB_SHARED int s_hasmax[TA];

    // ---- build the tables (split_table.cuh: the same three phases run on the host in the tests)
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        int i = i0 + t;
        u64 beg = 0; int n = 0; int hm = 0;
        if (i < a.nA) {
            beg = a.offA[i];
            n = (int)(a.offA[i + 1] - beg);
            if (n > 0 && ld_nc_u64(a.hA + beg + n - 1) == SMB_U64_MAX) { --n; hm = 1; }
        }
        if (tid == 0) { s_n[t] = n; s_hasmax[t] = hm; }
        split_table_load(lo_base + (size_t)t * kstride, hi_base + (size_t)t * kstride,
                         dirs_base + (size_t)t * dstride, a.hA + beg, n, nb, tid, nthreads);
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < TA; ++t)
        split_table_heads(lo_base + (size_t)t * kstride, hi_base + (size_t)t * kstride,
                          dirs_base + (size_t)t * dstride, s_n[t], shift, tid, nthreads);
    __syncthreads();
#pragma unroll
    for (int t = 0; t < TA; ++t) split_table_flags(dirs_base + (size_t)t * dstride, nb, tid, nthreads);
    __syncthreads();

    SplitTable tab[TA];
#pragma unroll
    for (int t = 0; t < TA; ++t) {
        tab[t].lo = lo_base + (size_t)t * kstride;
        tab[t].hi = hi_base + (size_t)t * kstride;
        tab[t].dir = dirs_base + (size_t)t * dstride;
    }

    const int warp = tid >> 5, lane = tid & 31;
    const int NWARPS = nthreads >> 5;
    for (int j = jbeg + warp; j < jend; j += NWARPS) {
        const u64 bbeg = a.offB[j];
        int nbj = (int)(a.offB[j + 1] - bbeg);
        int bmax = 0;
        if (nbj > 0 && ld_nc_u64(a.hB + bbeg + nbj - 1) == SMB_U64_MAX) { --nbj; bmax = 1; }
        const u64* row = a.hB + bbeg;
        u32 cnt[TA];
#pragma unroll
        for (int t = 0; t < TA; ++t) cnt[t] = 0;

        int base = 0;
        const int full = nbj - (nbj % (32 * U));
        u64 q[U];
        if (full > 0) {
#pragma unroll
            for (int u = 0; u < U; ++u) q[u] = ld_nc_u64(row + u * 32 + lane);
        }
        for (; base < full; base += 32 * U) {
            u64 cur[U];
#pragma unroll
            for (int u = 0; u < U; ++u) cur[u] = q[u];
            if (base + 32 * U < full) {
#pragma unroll
                for (int u = 0; u < U; ++u) q[u] = ld_nc_u64(row + base + 32 * U + u * 32 + lane);
            }
            // fast path: directory entry + two low words per probe; one predicate and one OR
            // accumulator per element for the whole batch, nothing else is kept
            bool hit = false;
            u32 ov[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                ov[u] = 0;
#pragma unroll
                for (int t = 0; t < TA; ++t) hit |= split_probe_low(tab[t], cur[u], shift, ov[u]);
            }
            if (__any_sync(0xffffffffu, hit)) {                       // related rows only
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int t = 0; t < TA; ++t) cnt[t] += split_probe_verify(tab[t], cur[u], shift);
            }
            u32 ovany = 0;
#pragma unroll
            for (int u = 0; u < U; ++u) ovany |= ov[u];
            if (ovany & 1u) {                                          // rare: a crowded bucket was hit
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (ov[u] & 1u) {
#pragma unroll
                        for (int t = 0; t < TA; ++t) cnt[t] += split_probe_rest(tab[t], cur[u], shift);
                    }
            }
        }
        for (; base < nbj; base += 32) {      // ragged tail
            int e = base + lane;
            if (e < nbj) {
                u64 qq = ld_nc_u64(row + e);
#pragma unroll
                for (int t = 0; t < TA; ++t)
                    cnt[t] += split_probe_verify(tab[t], qq, shift) + split_probe_rest(tab[t], qq, shift);
            }
        }
#pragma unroll
        for (int t = 0; t < TA; ++t) {
            u32 c = __reduce_add_sync(0xffffffffu, cnt[t]);
            int i = i0 + t;
            if (lane == 0 && i < a.nA && (!a.symmetric || j > i))
                a.out[(size_t)i * a.ldo + j] = c + (u32)(s_hasmax[t] & bmax);
        }
    }
}

}  // namespace smb
