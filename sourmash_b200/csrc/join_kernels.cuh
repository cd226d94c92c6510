// join_kernels.cuh -- kernels of the plain inverted join (compare_kernels.cu launches them): the all-vs-all
// count matrix by sorting the (hash, row) pairs of a key range and issuing one global reduction per pair of
// rows that share a hash.  It is the fallback of the stripe layout (join_stripe.cuh: matrices whose row of
// counters does not fit shared memory) and the form that shards by key range.  In a header so that
// tests/host_emul/simt_emul.cu runs the kernels on the CPU against the oracle.
#pragma once
#include "common.cuh"
#include "join_walk.cuh"

namespace smb {

__global__ void __launch_bounds__(256) join_row_range_kernel(const u64* __restrict__ h, const u64* __restrict__ off,
                                                            int n_rows, u64 key_lo, u64 key_hi, int bounded_hi,
                                                            u64* __restrict__ beg, u64* __restrict__ cnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    if (r == n_rows) { cnt[r] = 0; return; }              // extra slot: the scan then yields the total
    const u64* row = h + off[r];
    const u64 len = off[r + 1] - off[r];
    u64 lo = 0, hi = len;
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (row[mid] < key_lo) lo = mid + 1; else hi = mid; }
    const u64 b = lo;
    u64 e = len;
    if (bounded_hi) {
        lo = b; hi = len;
        while (lo < hi) { u64 mid = (lo + hi) >> 1; if (row[mid] < key_hi) lo = mid + 1; else hi = mid; }
        e = lo;
    }
    beg[r] = b;
    cnt[r] = e - b;
}

__global__ void __launch_bounds__(256) join_gather_kernel(const u64* __restrict__ h, const u64* __restrict__ off,
                                                         const u64* __restrict__ beg, const u64* __restrict__ dst_off,
                                                         int n_rows, u64* __restrict__ keys, u32* __restrict__ ids) {
    for (int r = blockIdx.x; r < n_rows; r += gridDim.x) {
        const u64 src = off[r] + beg[r], d0 = dst_off[r], n = dst_off[r + 1] - d0;
        for (u64 i = threadIdx.x; i < n; i += blockDim.x) { keys[d0 + i] = h[src + i]; ids[d0 + i] = (u32)r; }
    }
}

// out[0] += sum over groups of C(m,2); out[1] = max m
__global__ void __launch_bounds__(256) join_estimate_kernel(const u64* __restrict__ keys, u64 T,
                                                           unsigned long long* __restrict__ out) {
    unsigned long long pairs = 0, mmax = 0;
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < T; p += (u64)gridDim.x * blockDim.x) {
        const u64 m = join_group_size_at_head(keys, T, p);
        pairs += m * (m - (m ? 1 : 0)) / 2;
        mmax = m > mmax ? m : mmax;
    }
    for (int d = 16; d; d >>= 1) {
        pairs += __shfl_xor_sync(0xffffffffu, pairs, d);
        unsigned long long o = __shfl_xor_sync(0xffffffffu, mmax, d);
        mmax = o > mmax ? o : mmax;
    }
    if (lane_id() == 0) { if (pairs) atomicAdd(out, pairs); if (mmax) atomicMax(out + 1, mmax); }
}

// Every element pairs with the later elements of its group: ids ascend inside a group, so
// (ids[p], ids[b]) is an upper-triangle cell.  Increments are fire-and-forget reductions (RED)
// resolved in L2, and their rate is what bounds the kernel (1.44e9 reductions on the 10 000-sketch
// matrix); rewrites that attack everything else -- evict-first stream loads + evict-last reductions,
// walking the groups from a shared-memory tile instead of dependent L2 loads -- left the time
// unchanged.  Going faster needs fewer reductions (accumulating in shared-memory tiles of the
// matrix): the stripe layout of DESIGN.md section 4.5, the default.
__global__ void __launch_bounds__(256) join_count_kernel(const u64* __restrict__ keys, const u32* __restrict__ ids,
                                                        u64 T, u32* __restrict__ common, size_t ld) {
    const u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= T) return;
    join_walk(keys, ids, T, p, [&](u32 a, u32 b) { atomicAdd(common + (size_t)a * ld + b, 1u); });
}

}  // namespace smb
