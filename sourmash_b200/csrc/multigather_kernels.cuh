// multigather_kernels.cuh -- gather rounds of many queries against one resident database, one launch per step for all
// queries together (smb_multigather, capi.cu).  Included from compare_kernels.cu, which keeps the launchers.
//
// The single-query device loop (search_kernels.cuh: counter_update_argmax_pick_kernel, intersect_alive_pick_kernel and
// a tile launch over the candidates) keeps one SM busy in three of its four launches.  Here every per-query array is
// segmented -- query q owns q_hashes[q_begin[q] .. q_end[q]), candidates cand_rows[cand_off[q] ..), its counters and
// deltas at the same positions, picks at pick_off[q] .., an intersection slice at isect_off[q] .. -- and a round is
//   1. multi_counter_update_argmax_pick_kernel   one CTA per query
//   2. multi_intersect_alive_pick_kernel         one CTA per query
//   3. multi_decrement_kernel                    CTAs mapped to (query, chunk of candidates) through cta_start[]
// whatever the number of queries.  A finished query turns its CTAs into no-ops; `live` counts the unfinished ones and is
// the only value the host reads while the rounds run.
#pragma once
#include "common.cuh"
#include "split_table.cuh"

namespace smb {

#ifndef SMB_MULTI_GATHER_ARGS_DEFINED
#define SMB_MULTI_GATHER_ARGS_DEFINED
struct MultiGatherArgs {
    const uint64_t* q_hashes;                              // sorted-unique query hashes ...
    const uint64_t* q_begin;   const uint64_t* q_end;      // [Q] ... of every query
    const uint32_t* cand_rows; const uint64_t* cand_off;   // [Q+1] candidate rows (database ids, ascending)
    uint32_t* counts;          uint32_t* delta;            // per candidate
    const uint64_t* pick_off;  uint32_t* pick_rows; uint32_t* pick_sizes;   // [Q+1]; capacity = the query's round cap
    uint32_t* state;                                       // [2Q]: rounds picked, done
    uint32_t* live;                                        // unfinished queries
    const uint32_t* threshold;                             // [Q], >= 1
    uint32_t* consumed;                                    // beside q_hashes: round that took the hash, UINT32_MAX while alive
    uint64_t* isect;           const uint64_t* isect_off;  // [Q+1] this round's intersection of every query
    uint32_t* isect_n;                                     // [Q]
    const uint64_t* db_hashes; const uint64_t* db_off;
    const uint32_t* cta_start;                             // [Q+1] first decrement CTA of every query
    int n_queries, cols_per_cta, shift, nb, kstride;
};
#endif

// counters -= delta (the delta is consumed: zeroed for the next round), argmax with the lowest candidate position winning
// ties (Counter.most_common()[0]; candidates are in database order), append the winner or finish the query.
__global__ void __launch_bounds__(1024) multi_counter_update_argmax_pick_kernel(MultiGatherArgs a) {
    SMB_SHARED unsigned long long sb[32];
    const int qi = blockIdx.x;
    if (a.state[2 * qi + 1]) return;
    const u64 c0 = a.cand_off[qi];
    const int n = (int)(a.cand_off[qi + 1] - c0);
    u32* __restrict__ counters = a.counts + c0;
    u32* __restrict__ delta = a.delta + c0;
    unsigned long long best = 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        u32 v = counters[j];
        const u32 d = delta[j];
        if (d) { v = d > v ? 0u : v - d; counters[j] = v; delta[j] = 0; }
        const unsigned long long key = ((unsigned long long)v << 32) | (unsigned long long)(0xffffffffu - (u32)j);
        best = key > best ? key : best;
    }
    for (int d = 16; d; d >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
        best = o > best ? o : best;
    }
    if (lane_id() == 0) sb[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
        best = threadIdx.x < (blockDim.x >> 5) ? sb[threadIdx.x] : 0ULL;
        for (int d = 16; d; d >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
            best = o > best ? o : best;
        }
        if (threadIdx.x == 0) {
            const u32 value = (u32)(best >> 32), pos = 0xffffffffu - (u32)(best & 0xffffffffu);
            const u32 r = a.state[2 * qi];
            const u64 p0 = a.pick_off[qi];
            if (value == 0 || value < a.threshold[qi] || r >= (u32)(a.pick_off[qi + 1] - p0)) {
                a.state[2 * qi + 1] = 1;
                atomicAdd(a.live, 0xffffffffu);                  // -1
            } else {
                a.pick_rows[p0 + r] = a.cand_rows[c0 + pos];
                a.pick_sizes[p0 + r] = 0;
                a.state[2 * qi] = r + 1;
            }
        }
    }
}

// intersect_alive_pick_kernel on the query's segment: the hashes of the picked row that are in the query and still alive,
// in row order, into the query's intersection slice; they are consumed on the spot (consumed[pos] = this round).  Eight
// binary searches in flight per thread, ordered compaction across the CTA.
__global__ void __launch_bounds__(1024) multi_intersect_alive_pick_kernel(MultiGatherArgs a) {
    constexpr int K = 8;
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u32 carry;
    const int qi = blockIdx.x;
    const u32 picked = a.state[2 * qi];
    if (a.state[2 * qi + 1] || picked == 0) {
        if (threadIdx.x == 0) a.isect_n[qi] = 0;
        return;
    }
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const u32 round = picked - 1;
    const u32 r = a.pick_rows[a.pick_off[qi] + round];
    const u64* __restrict__ row = a.db_hashes + a.db_off[r];
    const u64 rn = a.db_off[r + 1] - a.db_off[r];
    const u64* __restrict__ q = a.q_hashes + a.q_begin[qi];
    const u64 nq = a.q_end[qi] - a.q_begin[qi];
    u32* __restrict__ consumed = a.consumed + a.q_begin[qi];
    u64* __restrict__ out = a.isect + a.isect_off[qi];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    int steps = 0;
    while ((1ull << steps) < nq + 1) ++steps;
    for (u64 base = 0; base < rn; base += (u64)blockDim.x * K) {
        u64 x[K], lo[K];
        bool in[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const u64 e = base + (u64)threadIdx.x * K + k;
            in[k] = e < rn;
            x[k] = in[k] ? row[e] : 0;
            lo[k] = 0;
        }
        for (int b = steps - 1; b >= 0; --b) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const u64 probe = lo[k] + (1ull << b);
                if (probe <= nq && ld_nc_u64(q + probe - 1) < x[k]) lo[k] = probe;
            }
        }
        u32 keep = 0;
#pragma unroll
        for (int k = 0; k < K; ++k)
            if (in[k] && lo[k] < nq && ld_nc_u64(q + lo[k]) == x[k] && consumed[lo[k]] == 0xffffffffu) {
                keep |= 1u << k;
                consumed[lo[k]] = round;
            }
        u32 mine = (u32)__popc(keep), incl = mine;
        for (int d = 1; d < 32; d <<= 1) {
            const u32 o = __shfl_sync(0xffffffffu, incl, lane >= d ? lane - d : lane);
            if (lane >= d) incl += o;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        u32 before = 0;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        u32 pos_out = carry + before + incl - mine;
#pragma unroll
        for (int k = 0; k < K; ++k)
            if ((keep >> k) & 1u) out[pos_out++] = x[k];
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 t = 0;
            for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) t += warp_tot[w2];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        a.isect_n[qi] = carry;
        a.pick_sizes[a.pick_off[qi] + round] = carry;
    }
}

// delta[j] = |isect_q ∩ row(cand_q[j])| for the chunk of candidates of this CTA: the query's intersection becomes the
// shared-memory split table (split_table.cuh) and the candidate rows stream through it, one warp per row -- the probe of
// pairwise_tile_split_kernel with one table.  An empty intersection (finished query) makes the CTA a no-op.
__global__ void __launch_bounds__(512) multi_decrement_kernel(MultiGatherArgs a) {
    constexpr int U = 4;
    SMB_DYN_SHARED(unsigned char, smem_raw);
    SMB_SHARED int s_n;
    SMB_SHARED int s_hasmax;
    const u32 b = blockIdx.x;
    int lo_q = 0, hi_q = a.n_queries;                       // largest qi with cta_start[qi] <= b
    while (hi_q - lo_q > 1) {
        const int mid = (lo_q + hi_q) >> 1;
        if (a.cta_start[mid] <= b) lo_q = mid; else hi_q = mid;
    }
    const int qi = lo_q;
    const u32 n_isect = a.isect_n[qi];
    if (n_isect == 0) return;
    const u64 c0 = a.cand_off[qi];
    const int n_cand = (int)(a.cand_off[qi + 1] - c0);
    const int jbeg = (int)(b - a.cta_start[qi]) * a.cols_per_cta;
    const int jend = min(jbeg + a.cols_per_cta, n_cand);
    if (jbeg >= jend) return;
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const u32 shift = (u32)a.shift;
    u32* lo_w = reinterpret_cast<u32*>(smem_raw);
    u32* hi_w = lo_w + a.kstride;
    u16* dir = reinterpret_cast<u16*>(smem_raw + (size_t)a.kstride * 8);
    const u64* keys = a.isect + a.isect_off[qi];
    int n = (int)n_isect, hm = 0;
    if (ld_nc_u64(keys + n - 1) == SMB_U64_MAX) { --n; hm = 1; }
    if (tid == 0) { s_n = n; s_hasmax = hm; }
    split_table_load(lo_w, hi_w, dir, keys, n, a.nb, tid, nthreads);
    __syncthreads();
    split_table_heads(lo_w, hi_w, dir, s_n, shift, tid, nthreads);
    __syncthreads();
    split_table_flags(dir, a.nb, tid, nthreads);
    __syncthreads();
    SplitTable tab;
    tab.lo = lo_w; tab.hi = hi_w; tab.dir = dir;
    const int warp = tid >> 5, lane = tid & 31, NWARPS = nthreads >> 5;
    for (int j = jbeg + warp; j < jend; j += NWARPS) {
        const u32 r = a.cand_rows[c0 + j];
        const u64 bbeg = a.db_off[r];
        int nbj = (int)(a.db_off[r + 1] - bbeg);
        int bmax = 0;
        if (nbj > 0 && ld_nc_u64(a.db_hashes + bbeg + nbj - 1) == SMB_U64_MAX) { --nbj; bmax = 1; }
        const u64* row = a.db_hashes + bbeg;
        u32 cnt = 0;
        int base = 0;
        const int full = nbj - (nbj % (32 * U));
        u64 nxt[U];
        if (full > 0) {
#pragma unroll
            for (int u = 0; u < U; ++u) nxt[u] = ld_nc_u64(row + u * 32 + lane);
        }
        for (; base < full; base += 32 * U) {
            u64 cur[U];
#pragma unroll
            for (int u = 0; u < U; ++u) cur[u] = nxt[u];
            if (base + 32 * U < full) {
#pragma unroll
                for (int u = 0; u < U; ++u) nxt[u] = ld_nc_u64(row + base + 32 * U + u * 32 + lane);
            }
            bool hit = false;
            u32 ov = 0;
#pragma unroll
            for (int u = 0; u < U; ++u) hit |= split_probe_low(tab, cur[u], shift, ov);
            if (__any_sync(0xffffffffu, hit)) {
#pragma unroll
                for (int u = 0; u < U; ++u) cnt += split_probe_verify(tab, cur[u], shift);
            }
            if (ov & 1u) {
#pragma unroll
                for (int u = 0; u < U; ++u) cnt += split_probe_rest(tab, cur[u], shift);
            }
        }
        for (; base < nbj; base += 32) {
            const int e = base + lane;
            if (e < nbj) {
                const u64 x = ld_nc_u64(row + e);
                cnt += split_probe_verify(tab, x, shift) + split_probe_rest(tab, x, shift);
            }
        }
        const u32 c = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) a.delta[c0 + j] = c + (u32)(s_hasmax & bmax);
    }
}

}  // namespace smb
