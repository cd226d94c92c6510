// range_kernels.cuh -- the streaming one-vs-many pass for a query too large for shared memory: the inner loop
// of Index.find / prefetch / the first gather round against a metagenome-sized query
// (src/sourmash/index/__init__.py:115-170, count_common of src/core/src/sketch/minhash.rs:539-558 per subject).
// compare_kernels.cu launches these kernels, tests/host_emul/simt_emul.cu runs them on the CPU against the oracle.
//
// Problem: |Q ∩ S_j| for every row S_j of a resident database (300 000 rows x ~5 000 sorted u64 = 12 GB) and a
// query of 10^7 hashes.  Every database element must be read once (the HBM roofline) and tested for membership
// in Q.  A membership filter for 10^7 keys does not fit shared memory, so the KEY SPACE is cut into P equal
// ranges and the database is kept in a second, RANGE-MAJOR order (built once per resident set, like an index):
//   rm[ part p ] = the elements of range p of row 0, of row 1, ..., of row n-1, back to back
//   slice[p * n + r] = position in rm where row r's elements of range p start     (u32, one table)
// CTA p builds a two-probe Bloom bitmap of the query keys of ITS range in shared memory (~7 500 keys in 512 Kbit:
// 0.1 % false positives), then streams part p front to back -- fully coalesced, every lane busy, 8 loads in flight
// per thread -- and probes the bitmap.  The rare hits (true matches + false positives) go to a per-warp queue and
// are settled in bulk: exact binary search in the query's slice, then the row is found from `slice` and its counter
// incremented.  Algorithmic bytes: 8 (|Q| + sum |S_j|), each read once.
//
// The same pass counts a GROUP of G queries at once (many_vs_many): their keys, concatenated and sorted by a stable
// pair sort with the query id as the value, form one key stream with a parallel array of ids (ascending inside a run
// of equal keys).  The bitmap is built from the stream's slice as before -- a key held by several queries sets the
// same two bits again -- and a settled match adds 1 to counter (query, row) of every query in the key's run: the
// database is read once for the whole group instead of once per query.
#pragma once
#include "common.cuh"
#include "range_search.cuh"

namespace smb {

static constexpr int RM_THREADS = 512;                // 2 CTAs per SM (registers: two batches of loads live per thread), 64 KB bitmap each
static constexpr int RM_BITMAP_LOG2 = 19;             // 512 Kbit = 64 KB
static constexpr int RM_QUEUE = 128;                  // candidates per warp
static constexpr int RM_UNROLL = 8;                   // 8-byte loads in flight per thread
static constexpr u32 RM_HASH2_32 = 0x9E3779B1u;       // second probe: multiplicative hash of the low word of (x - lo)

// range of key x for ranges of `width` keys (x <= max_key, so the result is < P by construction of width)
__host__ __device__ __forceinline__ u32 rm_range_of(u64 x, u64 width) { return (u32)(x / width); }

// bounds[p * n + r] = index inside row r of its first element with range >= p  (p = 0 .. P): one warp per row walks
// the row once; where the range id steps from a to b the bounds a+1 .. b are the current index
__global__ void __launch_bounds__(256) rm_bounds_kernel(const u64* __restrict__ h, const u64* __restrict__ off, int n,
                                                       u64 width, int P, u32* __restrict__ bounds) {
    const u32 lane = lane_id();
    const int warp0 = (int)(((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int n_warps = (int)(((u64)gridDim.x * blockDim.x) >> 5);
    for (int r = warp0; r < n; r += n_warps) {
        const u64* __restrict__ row = h + off[r];
        const u64 len = off[r + 1] - off[r];
        long long carry = -1;                             // range of the element in front of the chunk
        for (u64 i0 = 0; i0 <= len; i0 += 32) {           // index len is a virtual element of range P (closes every bound)
            const u64 i = i0 + lane;
            long long pid = -2;                           // lanes behind the virtual element: nothing to do
            if (i < len) pid = (long long)rm_range_of(row[i], width);
            else if (i == len) pid = P;
            long long prev = __shfl_sync(0xffffffffu, pid, lane ? lane - 1 : 0);
            if (lane == 0) prev = carry;
            if (pid >= 0)
                for (long long p = prev + 1; p <= pid; ++p) bounds[(size_t)p * n + r] = (u32)i;
            carry = __shfl_sync(0xffffffffu, pid, 31);
        }
    }
}

// cnt[p * n + r] = number of elements of row r in range p (cub::DeviceScan::ExclusiveSum turns it into `slice`)
__global__ void __launch_bounds__(256) rm_counts_kernel(const u32* __restrict__ bounds, int n, int P, u32* __restrict__ cnt) {
    const u64 total = (u64)n * (u64)P;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= total; i += (u64)gridDim.x * blockDim.x)
        cnt[i] = i < total ? bounds[i + n] - bounds[i] : 0u;    // one extra slot: the scan leaves the total there
}

// one thread per (range, row) slice: a few elements, read where the row lies, written back to back
__global__ void __launch_bounds__(256) rm_scatter_kernel(const u64* __restrict__ h, const u64* __restrict__ off,
                                                        const u32* __restrict__ bounds, const u32* __restrict__ slice,
                                                        int n, int P, u64* __restrict__ rm) {
    const u64 total = (u64)n * (u64)P;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        const int r = (int)(i % (u64)n);
        const u32 b0 = bounds[i], b1 = bounds[i + n];
        const u64* __restrict__ src = h + off[r] + b0;
        u64* __restrict__ dst = rm + slice[i];
        for (u32 k = 0; k < b1 - b0; ++k) dst[k] = src[k];
    }
}

static constexpr int RM_COARSE_LOG2 = 6;              // every 64th row's slice start is repeated in a small table

// coarse[p * nc + k] = slice[p * n + min(k << RM_COARSE_LOG2, n)], k = 0 .. nc - 1 (nc = (n >> RM_COARSE_LOG2) + 2): the row
// attribution of a match searches this table (19 KB per part, cache resident) and then one 64-row window of `slice`
// instead of all of a part's 1.2 MB of it
__global__ void __launch_bounds__(256) rm_coarse_kernel(const u32* __restrict__ slice, int n, int P, int nc, u32* __restrict__ coarse) {
    const u64 total = (u64)P * (u64)nc;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        const u64 p = i / (u64)nc, k = i - p * (u64)nc;
        const u64 r = (k << RM_COARSE_LOG2) < (u64)n ? (k << RM_COARSE_LOG2) : (u64)n;
        coarse[i] = slice[p * (u64)n + r];
    }
}

struct RangeMajorArgs {
    const u64* q; u64 nq;                 // the query, sorted (a group of queries: their merged key stream, see qid)
    const u64* rm;                        // range-major database
    const u32* slice;                     // [P * n + 1]
    const u32* coarse; int nc;            // [P * nc]
    int n, P;
    u64 width;
    u32 bm_log2;                          // bits of the bitmap = 2^bm_log2 (RM_BITMAP_LOG2; tests use tiny bitmaps: false positives)
    u32 bm_shift;                         // (x - lo) >> bm_shift < 2^bm_log2
    u32* out;                             // zeroed by the caller: [n] counters, or [G x n] (query-major) with qid
    const u32* qid;                       // null: one query; else the query of every key of q (a G-query group)
};

__device__ __forceinline__ u32 rm_bit1(u64 d, u32 bm_shift) { return (u32)(d >> bm_shift); }
__device__ __forceinline__ u32 rm_bit2(u64 d, u32 bm_log2) { return ((u32)d * RM_HASH2_32) >> (32u - bm_log2); }

// settle the queued candidates of one warp: exact test against the query slice, then row attribution
__device__ __forceinline__ void rm_drain(const RangeMajorArgs& a, const u32* __restrict__ queue, u32 count, u64 qlo, u64 qhi,
                                         const u32* __restrict__ slice_p, const u32* __restrict__ coarse_p, u32 lane) {
    for (u32 i = lane; i < count; i += 32) {
        const u32 pos = queue[i];
        const u64 x = a.rm[pos];
        u64 lo = qlo, hi = qhi;
        while (lo < hi) { const u64 mid = (lo + hi) >> 1; if (a.q[mid] < x) lo = mid + 1; else hi = mid; }
        if (lo >= qhi || a.q[lo] != x) continue;          // a false positive of the bitmap
        // last row whose slice starts at or in front of pos: first the 64-row window (coarse table), then inside it
        int l = 0, r = a.nc;
        while (r - l > 1) { const int mid = (l + r) >> 1; if (coarse_p[mid] <= pos) l = mid; else r = mid; }
        l <<= RM_COARSE_LOG2;
        r = l + (1 << RM_COARSE_LOG2) < a.n ? l + (1 << RM_COARSE_LOG2) : a.n;
        while (r - l > 1) { const int mid = (l + r) >> 1; if (slice_p[mid] <= pos) l = mid; else r = mid; }
        // every query that holds x: the run of equal keys from lo (one query: the run is this key, the counter out[l])
        u64 j = lo;
        do atomicAdd(a.out + (a.qid ? (u64)a.qid[j] * (u64)a.n : 0ull) + l, 1u);
        while (a.qid && ++j < qhi && a.q[j] == x);
    }
}

// ids[k] = g for the keys k of query g of a group (qoff: its G + 1 offsets into the concatenated keys, from 0);
// stat[0] = the largest key (the sort's significant bits), stat[1] > 0 iff a query is not sorted and unique
__global__ void __launch_bounds__(256) rm_query_ids_kernel(const u64* __restrict__ q, const u64* __restrict__ qoff, int G,
                                                          u32* __restrict__ ids, unsigned long long* __restrict__ stat) {
    for (int g = blockIdx.x; g < G; g += gridDim.x) {
        const u64 b = qoff[g], e = qoff[g + 1];
        u32 bad = 0;
        for (u64 k = b + threadIdx.x; k < e; k += blockDim.x) {
            if (ids) ids[k] = (u32)g;
            bad |= k > b && q[k] <= q[k - 1];
        }
        if (bad) atomicAdd(stat + 1, 1ull);
        if (threadIdx.x == 0 && e > b) atomicMax(stat, (unsigned long long)q[e - 1]);
    }
}

// one CTA per key range
__global__ void __launch_bounds__(RM_THREADS, 2) one_vs_many_range_major_kernel(RangeMajorArgs a) {
    SMB_DYN_SHARED(u32, rm_smem);                          // [2^bm_log2 / 32] bitmap words, then the warps' queues
    SMB_SHARED u64 s_q[2];
    u32* bitmap = rm_smem;
    const u32 BM_WORDS = a.bm_log2 > 5 ? 1u << (a.bm_log2 - 5) : 1u;
    const int p = blockIdx.x;
    const u64 lo = (u64)p * a.width;
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    u32* queue = rm_smem + BM_WORDS + warp * RM_QUEUE;
    if (threadIdx.x == 0) {
        // query keys of this range: lo <= k, k - lo < width (monotone predicate, no overflow)
        const u64 qlo = range_lower_bound(a.q, a.nq, lo);
        u64 l = qlo, hgh = a.nq;
        while (l < hgh) { const u64 mid = (l + hgh) >> 1; if (a.q[mid] - lo < a.width) l = mid + 1; else hgh = mid; }
        s_q[0] = qlo; s_q[1] = l;
    }
    for (u32 i = threadIdx.x; i < BM_WORDS; i += blockDim.x) bitmap[i] = 0;
    __syncthreads();
    const u64 qlo = s_q[0], qhi = s_q[1];
    if (qlo == qhi) return;                                // no query key in this range: nothing can match
    for (u64 i = qlo + threadIdx.x; i < qhi; i += blockDim.x) {
        const u64 d = a.q[i] - lo;
        const u32 b1 = rm_bit1(d, a.bm_shift), b2 = rm_bit2(d, a.bm_log2);
        atomicOr(bitmap + (b1 >> 5), 1u << (b1 & 31));
        atomicOr(bitmap + (b2 >> 5), 1u << (b2 & 31));
    }
    __syncthreads();
    const u32* __restrict__ slice_p = a.slice + (size_t)p * a.n;
    const u32* __restrict__ coarse_p = a.coarse + (size_t)p * a.nc;
    const u64 begin = slice_p[0], end = slice_p[a.n];      // slice[(p + 1) * n] = start of the next part (or the total)
    u32 qn = 0;                                            // candidates in this warp's queue (warp-uniform)
    const u32 sh2 = 32u - a.bm_log2;

    // Both probes of one element, branch-free: bit 1 from the top bits of (x - lo), bit 2 from a multiplicative hash of
    // its low word (hash bits: independent of the top bits)
    auto probe = [&](u64 x) -> u32 {
        const u64 d = x - lo;
        const u32 b1 = (u32)(d >> a.bm_shift);
        const u32 b2 = ((u32)d * RM_HASH2_32) >> sh2;
        return (bitmap[b1 >> 5] >> (b1 & 31)) & (bitmap[b2 >> 5] >> (b2 & 31)) & 1u;
    };
    // rare path: queue the hits of one batch (bit u of hm = the lane's element at position pos0 + stride * u),
    // draining when the queue is full
    auto push = [&](u32 hm, u64 pos0, u32 stride) {
#pragma unroll
        for (int u = 0; u < RM_UNROLL; ++u) {
            const bool hit = (hm >> u) & 1u;
            const u32 m = __ballot_sync(0xffffffffu, hit);
            if (m == 0) continue;
            if (qn + (u32)__popc(m) > (u32)RM_QUEUE) {
                __syncwarp();
                rm_drain(a, queue, qn, qlo, qhi, slice_p, coarse_p, lane);
                __syncwarp();
                qn = 0;
            }
            if (hit) queue[qn + __popc(m & ((1u << lane) - 1u))] = (u32)(pos0 + (u64)stride * u);
            qn += (u32)__popc(m);
        }
    };
    // a batch of up to 32 * RM_UNROLL elements with bounds tests (the ragged head and tail of the part)
    auto checked = [&](u64 s0, u64 s1) {
        u32 hm = 0;
#pragma unroll
        for (int u = 0; u < RM_UNROLL; ++u) {
            const u64 i = s0 + (u64)u * 32 + lane;
            if (i < s1) hm |= probe(ld_stream_u64(a.rm + i)) << u;
        }
        if (__any_sync(0xffffffffu, hm != 0)) push(hm, s0 + lane, 32);
    };

    // main loop: 16-byte loads (positions are even), RM_UNROLL elements per lane per batch, and the NEXT batch's loads
    // are issued before the current batch is probed -- the kernel lives on bytes in flight
    constexpr int V = RM_UNROLL / 2;                       // 16-byte loads per lane per batch
    const u64 abeg = (begin + 1) & ~1ull;
    const u64 batch = 32ull * RM_UNROLL;
    const u64 n_batches = end > abeg ? (end - abeg) / batch : 0;
    const u32 n_warps = blockDim.x >> 5;
    if (warp == 0 && abeg > begin && begin < end) checked(begin, abeg);               // one element in front of the aligned start
    if (warp == n_warps - 1 && abeg + n_batches * batch < end) checked(abeg + n_batches * batch, end);
    const ulonglong2* __restrict__ src = reinterpret_cast<const ulonglong2*>(a.rm + abeg) + lane;
    ulonglong2 cur[V], nxt[V];
    u64 k = warp;
    if (k < n_batches) {
#pragma unroll
        for (int v = 0; v < V; ++v) cur[v] = ld_stream_u64x2(src + (k * V + v) * 32);
    }
    for (; k < n_batches; k += n_warps) {
        const u64 kn = k + n_warps;
        if (kn < n_batches) {
#pragma unroll
            for (int v = 0; v < V; ++v) nxt[v] = ld_stream_u64x2(src + (kn * V + v) * 32);
        }
        u32 hm = 0;
#pragma unroll
        for (int v = 0; v < V; ++v) hm |= (probe(cur[v].x) << (2 * v)) | (probe(cur[v].y) << (2 * v + 1));
        if (__any_sync(0xffffffffu, hm != 0)) {
            // element (v, half) of the lane sits at abeg + k * batch + v * 64 + 2 * lane + half: bit u = 2 v + half
#pragma unroll
            for (int u = 0; u < RM_UNROLL; ++u) {
                const bool hit = (hm >> u) & 1u;
                const u32 m = __ballot_sync(0xffffffffu, hit);
                if (m == 0) continue;
                if (qn + (u32)__popc(m) > (u32)RM_QUEUE) {
                    __syncwarp();
                    rm_drain(a, queue, qn, qlo, qhi, slice_p, coarse_p, lane);
                    __syncwarp();
                    qn = 0;
                }
                if (hit) queue[qn + __popc(m & ((1u << lane) - 1u))] = (u32)(abeg + k * batch + (u64)(u >> 1) * 64 + 2 * lane + (u & 1));
                qn += (u32)__popc(m);
            }
        }
#pragma unroll
        for (int v = 0; v < V; ++v) cur[v] = nxt[v];
    }
    __syncwarp();
    rm_drain(a, queue, qn, qlo, qhi, slice_p, coarse_p, lane);
}

}  // namespace smb
