// search_kernels.cuh -- the kernels behind search / prefetch / gather (compare_kernels.cu launches them): the
// bucket directory and occupancy bitmap over a large query, the one-vs-many pass against them, and the
// per-round steps of the gather session (live intersection, consumed flags, counter update + argmax, row set
// operations).  In a header so that tests/host_emul/simt_emul.cu can run the kernels themselves on the CPU
// (tests/host_emul/simt.h) -- a whole gather loop included -- against the oracle.
#pragma once
#include "common.cuh"

namespace smb {

__device__ __forceinline__ bool row_contains(const u64* __restrict__ r, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        u64 mid = (lo + hi) >> 1;
        u64 v = ld_nc_u64(r + mid);
        if (v < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && ld_nc_u64(r + lo) == x;
}

static constexpr u32 DIR_UNSET = 0xffffffffu;

__global__ void __launch_bounds__(256) global_dir_fill_kernel(u32* __restrict__ dir, u64 n_entries, u32 v) {
    for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_entries; b += (u64)gridDim.x * blockDim.x)
        dir[b] = v;
}

__global__ void __launch_bounds__(256) global_dir_heads_kernel(const u64* __restrict__ q, u64 nq, u32 shift,
                                                              u32* __restrict__ dir) {
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < nq; p += (u64)gridDim.x * blockDim.x) {
        const u64 bp = q[p] >> shift;
        const long long bprev = p == 0 ? -1 : (long long)(q[p - 1] >> shift);
        if ((long long)bp == bprev) continue;
        long long lo = (long long)bp - 32;                      // short gaps: fill directly
        if (lo < bprev + 1) lo = bprev + 1;
        for (long long b = lo; b <= (long long)bp; ++b) dir[b] = (u32)p;
    }
}

__global__ void __launch_bounds__(256) global_dir_resolve_kernel(const u64* __restrict__ q, u64 nq, u32 shift,
                                                                u64 nb, u32* __restrict__ dir) {
    for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b <= nb; b += (u64)gridDim.x * blockDim.x) {
        if (dir[b] != DIR_UNSET) continue;
        u64 lo = 0, hi = nq;                                    // first key with bucket >= b
        while (lo < hi) { u64 mid = (lo + hi) >> 1; if ((q[mid] >> shift) < b) lo = mid + 1; else hi = mid; }
        dir[b] = (u32)lo;
    }
}

// occupancy bitmap over the query: bit (key >> bm_shift) set iff some query key maps there.  It
// is 8-16x smaller than directory + keys, stays in L2, and rejects most probes of a subject
// element before the directory / key lines (DRAM for a 1e7-hash query) are touched.
__global__ void __launch_bounds__(256) build_query_bitmap_kernel(const u64* __restrict__ q, u64 nq,
                                                                u32 sh, int fine_log2,
                                                                u32* __restrict__ bitmap) {
    // bitmap is 2^fine_log2 times finer than the directory
    const u32 bm_shift = sh >= (u32)fine_log2 ? sh - (u32)fine_log2 : 0u;
    // q is sorted, so the keys of one 32-bit bitmap word are a contiguous run: the first key of
    // a run ORs the whole run together and stores the word -- no atomics, one writer per word.
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < nq; p += (u64)gridDim.x * blockDim.x) {
        const u64 bit = q[p] >> bm_shift;
        const u64 word = bit >> 5;
        if (p > 0 && ((q[p - 1] >> bm_shift) >> 5) == word) continue;
        u32 acc = 1u << (bit & 31);
        for (u64 r = p + 1; r < nq; ++r) {
            const u64 b2 = q[r] >> bm_shift;
            if ((b2 >> 5) != word) break;
            acc |= 1u << (b2 & 31);
        }
        bitmap[word] = acc;
    }
}

__global__ void __launch_bounds__(256) one_vs_many_global_kernel(
    const u64* __restrict__ q, u64 nq, const u32* __restrict__ dir, u32 shift, u64 nbk,
    const u32* __restrict__ bitmap, int fine_log2, const u64* __restrict__ hB,
    const u64* __restrict__ offB, int nB, u32* __restrict__ out) {
    const u32 bm_shift = shift >= (u32)fine_log2 ? shift - (u32)fine_log2 : 0u;
    const int lane = lane_id();
    const int wstride = gridDim.x * (blockDim.x >> 5);
    constexpr int U = 4;
    for (int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < nB; j += wstride) {
        const u64* row = hB + offB[j];
        const u64 n = offB[j + 1] - offB[j];
        u32 c = 0;
        for (u64 base = 0; base < n; base += 32 * U) {
            u64 x[U];
            u32 word[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                       // U independent loads in flight
                const u64 e = base + (u64)u * 32 + lane;
                x[u] = e < n ? ld_nc_u64(row + e) : SMB_U64_MAX;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                // beyond the query's key range nothing can match; lanes past the row's end are padding -- tested by
                // index, not by value: a query that holds UINT64_MAX (scaled = 1) covers the padding key too
                const bool in_range = base + (u64)u * 32 + lane < n && (x[u] >> shift) < nbk;
                word[u] = 0u;
                if (in_range) {
                    if (bitmap) {
                        const u64 bit = x[u] >> bm_shift;
                        word[u] = (__ldg(bitmap + (bit >> 5)) >> (bit & 31)) & 1u;
                    } else {
                        word[u] = 1u;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (word[u]) {                                   // ~4 % of the elements get here
                    const u64 b = x[u] >> shift;
                    u64 p = dir[b];
                    const u64 pe = dir[b + 1];
                    for (; p < pe; ++p) {
                        const u64 k = ld_nc_u64(q + p);
                        if (k >= x[u]) { c += (k == x[u]); break; }
                    }
                }
            }
        }
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) out[j] = c;
    }
}

// covered[p] = 1 for every query key q[p] held by one of the listed rows (prefetch's matched / unmatched query hashes).
// One warp per listed row, read in place from the CSR; every element probes the bitmap and directory exactly as
// one_vs_many_global_kernel does.  Writers of one byte all store 1, so no atomics; a row listed twice is harmless.
__global__ void __launch_bounds__(256) query_cover_kernel(
    const u64* __restrict__ q, u64 nq, const u32* __restrict__ dir, u32 shift, u64 nbk,
    const u32* __restrict__ bitmap, int fine_log2, const u64* __restrict__ hB,
    const u64* __restrict__ offB, const u32* __restrict__ rows, u64 n_rows, u8* __restrict__ covered) {
    const u32 bm_shift = shift >= (u32)fine_log2 ? shift - (u32)fine_log2 : 0u;
    const int lane = lane_id();
    const u64 wstride = (u64)gridDim.x * (blockDim.x >> 5);
    constexpr int U = 4;
    for (u64 j = (u64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_rows; j += wstride) {
        const u32 r = rows[j];
        const u64* row = hB + offB[r];
        const u64 n = offB[r + 1] - offB[r];
        for (u64 base = 0; base < n; base += 32 * U) {
            u64 x[U];
            u32 word[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const u64 e = base + (u64)u * 32 + lane;
                x[u] = e < n ? ld_nc_u64(row + e) : SMB_U64_MAX;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                // padding lanes by index, not by value: a query holding UINT64_MAX (scaled = 1) covers the padding key
                const bool in_range = base + (u64)u * 32 + lane < n && (x[u] >> shift) < nbk;
                word[u] = 0u;
                if (in_range) {
                    const u64 bit = x[u] >> bm_shift;
                    word[u] = (__ldg(bitmap + (bit >> 5)) >> (bit & 31)) & 1u;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (word[u]) {
                    const u64 b = x[u] >> shift;
                    u64 p = dir[b];
                    const u64 pe = dir[b + 1];
                    for (; p < pe; ++p) {
                        const u64 k = ld_nc_u64(q + p);
                        if (k >= x[u]) { if (k == x[u]) covered[p] = 1; break; }
                    }
                }
            }
        }
    }
}

template <bool KEEP_COMMON>
__global__ void __launch_bounds__(1024) setop_rows_kernel(const u64* __restrict__ a, u64 na,
                                                         const u64* __restrict__ b, u64 nb,
                                                         u64* __restrict__ out,
                                                         u32* __restrict__ d_n) {
    // stable compaction of a's elements that are (KEEP_COMMON ? in : not in) b.
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u32 carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    for (u64 base = 0; base < na; base += blockDim.x) {
        u64 e = base + threadIdx.x;
        bool valid = e < na;
        u64 x = valid ? a[e] : 0;
        bool in_b = valid && row_contains(b, nb, x);
        bool keep = valid && (KEEP_COMMON ? in_b : !in_b);
        u32 bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        u32 before = 0;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        u32 pos = carry + before + __popc(bal & ((1u << lane) - 1u));
        if (keep) out[pos] = x;
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 t = 0;
            for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) t += warp_tot[w2];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *d_n = carry;
}

// gather keeps its query fixed and flags consumed hashes instead of re-materialising the
// remaining query every round: intersect = row elements present in q and still alive.
__device__ __forceinline__ long long row_find(const u64* __restrict__ r, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        u64 mid = (lo + hi) >> 1;
        if (ld_nc_u64(r + mid) < x) lo = mid + 1; else hi = mid;
    }
    return (lo < n && ld_nc_u64(r + lo) == x) ? (long long)lo : -1;
}

__global__ void __launch_bounds__(1024) intersect_alive_kernel(const u64* __restrict__ q, u64 nq,
                                                              const u8* __restrict__ alive,
                                                              const u64* __restrict__ row, u64 rn,
                                                              u64* __restrict__ out, u32* __restrict__ d_n) {
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u32 carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    for (u64 base = 0; base < rn; base += blockDim.x) {
        u64 e = base + threadIdx.x;
        bool keep = false;
        u64 x = 0;
        if (e < rn) {
            x = row[e];
            long long pos = row_find(q, nq, x);
            keep = pos >= 0 && alive[pos];
        }
        u32 bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        u32 before = 0;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        u32 pos_out = carry + before + __popc(bal & ((1u << lane) - 1u));
        if (keep) out[pos_out] = x;
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 t = 0;
            for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) t += warp_tot[w2];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *d_n = carry;
}

__global__ void __launch_bounds__(256) mark_dead_kernel(const u64* __restrict__ q, u64 nq, u8* __restrict__ alive,
                                                       const u64* __restrict__ gone, u64 n) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (u64)gridDim.x * blockDim.x) {
        long long pos = row_find(q, nq, gone[e]);
        if (pos >= 0) alive[pos] = 0;
    }
}

__global__ void make_row_offsets_kernel(const u32* __restrict__ d_n, u64* __restrict__ off2) {
    off2[0] = 0;
    off2[1] = *d_n;
}

__global__ void __launch_bounds__(256) mark_dead_n_kernel(const u64* __restrict__ q, u64 nq, u8* __restrict__ alive,
                                                         const u64* __restrict__ gone, const u32* __restrict__ d_n) {
    const u64 n = *d_n;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (u64)gridDim.x * blockDim.x) {
        long long pos = row_find(q, nq, gone[e]);
        if (pos >= 0) alive[pos] = 0;
    }
}

// counters[j] -= delta[j] (delta nullable), then argmax with lowest-index tie break
// (Counter.most_common()[0] on insertion-ordered dict: src/sourmash/index/__init__.py:841).
__global__ void __launch_bounds__(1024) counter_update_argmax_kernel(
    u32* __restrict__ counters, const u32* __restrict__ delta, int n,
    unsigned long long* __restrict__ d_best) {
    // key = (value << 32) | (0xffffffff - index): max key == max value, then min index
    unsigned long long best = 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        u32 v = counters[j];
        if (delta) { u32 d = delta[j]; v = d > v ? 0u : v - d; counters[j] = v; }
        unsigned long long key = ((unsigned long long)v << 32) | (unsigned long long)(0xffffffffu - (u32)j);
        best = key > best ? key : best;
    }
    for (int d = 16; d; d >>= 1) {
        unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
        best = o > best ? o : best;
    }
    SMB_SHARED unsigned long long sb[32];
    if (lane_id() == 0) sb[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
        best = threadIdx.x < (blockDim.x >> 5) ? sb[threadIdx.x] : 0ULL;
        for (int d = 16; d; d >>= 1) {
            unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
            best = o > best ? o : best;
        }
        if (threadIdx.x == 0) {
            d_best[0] = best >> 32;                                   // value
            d_best[1] = 0xffffffffu - (u32)(best & 0xffffffffu);      // index
        }
    }
}


// ---- gather rounds driven from the device (smb_gather, candidate rows that fit the shared-memory table) ----------------
// The host loop above reads the winner of every round back (24 bytes + a stream synchronisation) to pick the row pointer.
// Here the row is picked ON the device: the argmax kernel appends (row, count) to a pick list and raises `done` when the
// best remaining overlap falls below the threshold; the intersect kernel takes its row from that pick; a finished loop
// turns every later kernel into a no-op (the intersection has length 0).  The host enqueues rounds in batches and looks
// at `state` once per batch.   state[0] = rounds picked, state[1] = done flag.
#ifndef SMB_GATHER_PICKS_DEFINED
#define SMB_GATHER_PICKS_DEFINED
struct GatherPicks {
    uint32_t* rows;       // [max_rounds] picked row per round
    uint32_t* sizes;      // [max_rounds] |row ∩ remaining query| per round
    uint32_t* state;      // [2]
    uint32_t threshold, max_rounds;
};
#endif

__global__ void __launch_bounds__(1024) counter_update_argmax_pick_kernel(u32* __restrict__ counters, const u32* __restrict__ delta,
                                                                         int n, GatherPicks g) {
    SMB_SHARED unsigned long long sb[32];
    const bool done = g.state[1] != 0;
    unsigned long long best = 0;
    if (!done) {
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            u32 v = counters[j];
            const u32 d = delta[j];
            v = d > v ? 0u : v - d;
            counters[j] = v;
            const unsigned long long key = ((unsigned long long)v << 32) | (unsigned long long)(0xffffffffu - (u32)j);
            best = key > best ? key : best;
        }
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
        if (threadIdx.x == 0 && !done) {
            const u32 value = (u32)(best >> 32), row = 0xffffffffu - (u32)(best & 0xffffffffu);
            const u32 r = g.state[0];
            if (value < g.threshold || value == 0 || r >= g.max_rounds) g.state[1] = 1;
            else { g.rows[r] = row; g.sizes[r] = 0; g.state[0] = r + 1; }
        }
    }
}

// intersect_alive_kernel for the row the last pick names (nothing, and *d_n = 0, once the loop is done).  One CTA (the
// output must stay in row order); every thread takes EIGHT consecutive elements per pass and runs their binary
// searches in lock step -- a fixed number of branch-free halving steps -- so that eight loads are in flight per thread
// instead of one: the kernel is a chain of ~17 dependent L2 loads per element and nothing else.
// The kept hashes are consumed on the spot (alive[pos] = 0: the job of mark_dead_n_kernel in the host-driven loop) -- the
// one-vs-many pass that follows reads the intersection, not the flags.
__global__ void __launch_bounds__(1024) intersect_alive_pick_kernel(const u64* __restrict__ q, u64 nq, u8* __restrict__ alive,
                                                                   const u64* __restrict__ hashes, const u64* __restrict__ off,
                                                                   GatherPicks g, u64* __restrict__ out, u32* __restrict__ d_n) {
    constexpr int K = 8;                                   // 8 192 elements per pass: a genome-sized row in one
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u32 carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const bool done = g.state[1] != 0 || g.state[0] == 0;
    const u32 round = done ? 0u : g.state[0] - 1;
    const u32 r = done ? 0u : g.rows[round];
    const u64* __restrict__ row = hashes + off[r];
    const u64 rn = done ? 0 : off[r + 1] - off[r];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    int steps = 0;                                         // halving steps that cover nq positions
    while ((1ull << steps) < nq + 1) ++steps;
    for (u64 base = 0; base < rn; base += (u64)blockDim.x * K) {
        u64 x[K], lo[K];
        bool in[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const u64 e = base + (u64)threadIdx.x * K + k;
            in[k] = e < rn;
            x[k] = in[k] ? row[e] : 0;
            lo[k] = 0;                                     // number of query keys < x, found from the top bit down
        }
        for (int b = steps - 1; b >= 0; --b) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const u64 probe = lo[k] + (1ull << b);     // q[probe - 1] < x  <=>  at least `probe` keys are smaller
                if (probe <= nq && ld_nc_u64(q + probe - 1) < x[k]) lo[k] = probe;
            }
        }
        u32 keep = 0;
#pragma unroll
        for (int k = 0; k < K; ++k)
            if (in[k] && lo[k] < nq && ld_nc_u64(q + lo[k]) == x[k] && alive[lo[k]]) { keep |= 1u << k; alive[lo[k]] = 0; }
        // ordered compaction: counts of the threads in front (warp prefix, then the warps in front)
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
        *d_n = carry;
        if (!done) g.sizes[round] = carry;
    }
}

}  // namespace smb
