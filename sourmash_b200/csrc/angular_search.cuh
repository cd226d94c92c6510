// angular_search.cuh -- the angular similarity of one abundance query against every row of a resident set that carries
// abundances (compare_kernels.cu launches it).  Replaces the per-subject loop of Index.search_abund
// (src/sourmash/index/__init__.py:172-200): one `similarity(..., downsample=True)` per subject, i.e. one upload, one
// single-CTA launch of angular_terms_kernel and one stream synchronisation per subject.
//
// For every row the kernel accumulates two of the terms of KmerMinHash::angular_similarity (minhash.rs:635-680), over
// the elements <= max_hash only (the downsampling of similarity(..., downsample=True), without a downsampled copy):
//   prod[row] = sum over shared hashes of q_abund * s_abund,   bsq[row] = sum of s_abund^2.
// Both are u64 sums that wrap, as the reference's release build does; wrapping addition is associative, so the atomics
// and any order of summation give the reference's value exactly.  The host adds the query's own sum of squares and
// finalizes the score with libm (the device acos is not libm's to the last ulp).
//
// Work mapping.  A row is cut into chunks of ANGULAR_CHUNK elements (chunk_start: prefix of the chunks of every row);
// a warp takes one chunk at a time and adds its two sums to the row's counters with one u64 atomic each, so a
// metagenome-sized row is spread over many warps instead of serialising one.  The grid is persistent: each CTA builds
// its probe table once.
//
// Probe (the query's keys, cut at max_hash, sorted-unique; the abundances stay in global memory and are read on a hit
// only).  UINT64_MAX cannot sit in the split table (it is the sentinel): it is answered from q_max_abund.  Keys above
// q_top are skipped by a compare.  Small queries: a shared-memory split table per CTA (split_table.cuh,
// split_probe_find).  Larger queries: the global bucket directory + L2 occupancy bitmap of the one-vs-many search
// (search_kernels.cuh, built by launch_build_global_dir / launch_build_query_bitmap).
#pragma once
#include "common.cuh"
#include "split_table.cuh"
#include "kernels.h"

namespace smb {

static constexpr int ANGULAR_THREADS = 512;

__host__ __device__ __forceinline__ size_t angular_split_smem(u64 nq, u64 nb) {
    return (size_t)(nq + 2) * 8 + (size_t)(nb + 2) * 2;
}

// position of x in the query of the global directory, -1 when absent (x < UINT64_MAX, x <= q_top)
__device__ __forceinline__ long long global_probe_find(const AngularSearchArgs& a, u64 x) {
    const u32 bm_shift = a.shift >= (u32)a.fine_log2 ? a.shift - (u32)a.fine_log2 : 0u;
    const u64 bit = x >> bm_shift;
    if (!((__ldg(a.bitmap + (bit >> 5)) >> (bit & 31)) & 1u)) return -1;
    const u64 b = x >> a.shift;
    for (u64 p = a.gdir[b], pe = a.gdir[b + 1]; p < pe; ++p) {
        const u64 k = ld_nc_u64(a.q + p);
        if (k >= x) return k == x ? (long long)p : -1;
    }
    return -1;
}

// q_abund * s_abund when x is a query key (0 otherwise)
__device__ __forceinline__ u64 angular_hit(const AngularSearchArgs& a, const SplitTable& t, u64 x, u64 sa) {
    if (x == SMB_U64_MAX) return a.q_has_max ? a.q_max_abund * sa : 0ull;
    if (a.nq == 0 || x > a.q_top) return 0ull;                  // (x >> shift) < nb from here on
    const long long p = a.split ? (long long)split_probe_find(t, x, a.shift) : global_probe_find(a, x);
    return p >= 0 ? ld_nc_u64(a.qa + p) * sa : 0ull;
}

__device__ __forceinline__ int angular_find_row(const u64* __restrict__ chunk_start, int n_rows, u64 c) {
    int lo = 0, hi = n_rows;                           // last row with chunk_start <= c
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (chunk_start[mid] <= c) lo = mid; else hi = mid; }
    return lo;
}

__global__ void __launch_bounds__(ANGULAR_THREADS, 2) angular_search_kernel(AngularSearchArgs a) {
    SMB_DYN_SHARED(unsigned char, smem_raw);
    const int tid = threadIdx.x;
    u32* lo_w = reinterpret_cast<u32*>(smem_raw);
    const int kstride = a.split ? (int)a.nq + 2 : 0;
    u32* hi_w = lo_w + kstride;
    u16* dir = reinterpret_cast<u16*>(smem_raw + (size_t)kstride * 8);
    SplitTable tab;
    tab.lo = lo_w; tab.hi = hi_w; tab.dir = dir;
    if (a.split) {
        split_table_load(lo_w, hi_w, dir, a.q, (int)a.nq, (int)a.nb, tid, ANGULAR_THREADS);
        __syncthreads();
        split_table_heads(lo_w, hi_w, dir, (int)a.nq, a.shift, tid, ANGULAR_THREADS);
        __syncthreads();
        split_table_flags(dir, (int)a.nb, tid, ANGULAR_THREADS);
        __syncthreads();
    }
    constexpr int U = 4;
    const int lane = lane_id();
    const u64 wstride = (u64)gridDim.x * (ANGULAR_THREADS / 32);
    for (u64 c = (u64)blockIdx.x * (ANGULAR_THREADS / 32) + (tid >> 5); c < a.n_chunks; c += wstride) {
        const int r = angular_find_row(a.chunk_start, a.n_rows, c);
        const u64 row_beg = a.off[r], row_end = a.off[r + 1];
        const u64 beg = row_beg + (c - a.chunk_start[r]) * (u64)ANGULAR_CHUNK;
        const u64 end = beg + ANGULAR_CHUNK < row_end ? beg + ANGULAR_CHUNK : row_end;
        u64 prod = 0, bsq = 0;
        for (u64 base = beg; base < end; base += 32 * U) {
            u64 x[U];
            bool in[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                   // U independent loads in flight
                const u64 e = base + (u64)u * 32 + lane;
                x[u] = e < end ? ld_nc_u64(a.h + e) : 0ull;
                in[u] = e < end && x[u] <= a.max_hash;
            }
            u64 sa[U];
#pragma unroll
            for (int u = 0; u < U; ++u) sa[u] = in[u] ? ld_nc_u64(a.ab + base + (u64)u * 32 + lane) : 0ull;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (!in[u]) continue;
                bsq += sa[u] * sa[u];
                prod += angular_hit(a, tab, x[u], sa[u]);
            }
            // rows ascend: once no lane is at or below max_hash, neither is the rest of the chunk
            if (!__any_sync(0xffffffffu, in[U - 1])) break;
        }
        for (int d = 16; d; d >>= 1) {
            prod += __shfl_xor_sync(0xffffffffu, prod, d);
            bsq += __shfl_xor_sync(0xffffffffu, bsq, d);
        }
        if (lane == 0) {
            if (prod) atomicAdd(a.prod + r, (unsigned long long)prod);
            if (bsq) atomicAdd(a.bsq + r, (unsigned long long)bsq);
        }
    }
}

}  // namespace smb
