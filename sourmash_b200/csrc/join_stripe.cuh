// join_stripe.cuh -- the stripe layout of the inverted join: the all-vs-all count matrix of `compare` with
// no count matrix in HBM and no global atomics (compare_kernels.cu launches these kernels; in a header so
// that tests/host_emul/simt_emul.cu runs the kernels themselves on the CPU against the oracle).
//
// What it computes: |A_i ∩ A_j| for every pair of rows, then jaccard = common / max(1, union) as float64 --
// intersection_size + jaccard of the reference (src/core/src/sketch/minhash.rs:593-631,1765-1807) for the
// n(n-1)/2 pairs that compare_serial walks one by one (src/sourmash/compare.py:36-54).
//
// Idea: |A_i ∩ A_j| = number of hashes held by both rows.  Sort the hashes of the whole set once; equal
// hashes become one contiguous *group* of the sorted stream, rows ascending inside it.  A CTA owns R complete
// rows of the RESULT as u32 counters in shared memory (a "stripe", R x n); for every hash of its rows it looks
// up the hash's group and bumps stripe[row][other row] for the other members with shared-memory atomics; the
// finished stripe is turned into float64 Jaccard values and written once.  Work is proportional to the
// number of (shared hash, pair) incidences -- unrelated pairs cost nothing.
//
// The sorted stream is stored as
//   tags[q] = row of sorted element q, top bit set on the first element of a group   (u16 if n < 32768: the
//             whole stream of a 10 000 x 5 000 set is then 100 MB instead of 200 MB; each CTA reads it front to back)
//   pos[e]  = sorted position of CSR element e
// and is built with FOUR radix passes instead of seven: the sort key is the top 32 significant bits of the
// hash, the remaining low bits travel in the 64-bit payload in front of the element index
// (payload = low bits << 32 | e).  Elements with equal 32-bit keys form a run, kept in CSR order by the
// stable sort; nearly every run is one group.  The rare runs that mix different hashes (expected
// distinct^2 / 2^33) are recognised by a payload that is smaller than its predecessor's and redone in order
// by one warp each -- ascending payloads = ascending (low bits, element) = groups contiguous, rows ascending.
// Because the key is a prefix of the hash, the stream is in hash order and every row walks it front to back.
#pragma once
#include "common.cuh"

namespace smb {

static constexpr int STRIPE_EBLK_LOG2 = 11;           // element blocks of the row lookup table: 25 000 entries for 5e7 elements, so
                                                      // the table and the row offsets it leads to stay in L1 (the tag kernel's
                                                      // chain of dependent loads payload -> block table -> row offsets hits L1)
static constexpr int STRIPE_MAX_WINDOWS = 2048;       // pos[] windows of the position pass (shared counters of the tag kernel)
static constexpr int STRIPE_MAX_ROWS = 32;            // rows per CTA (upper bound)
static constexpr int STRIPE_HEADER = 544;             // bytes in front of the counters: s_beg[32] + s_end[32] + control words, 16-aligned
static constexpr int STRIPE_TAG_PAD = 128;            // head flags stored behind the end of the tag stream

template <typename TagT> struct StripeTag;
template <> struct StripeTag<u16> { static constexpr u32 HEAD = 0x8000u; };
template <> struct StripeTag<u32> { static constexpr u32 HEAD = 0x80000000u; };

// row that owns CSR element e: largest r with off[r] <= e (rows may be empty)
__host__ __device__ __forceinline__ u32 stripe_row_of(const u64* __restrict__ off, int n, u64 e) {
    int lo = 0, hi = n;                                   // invariant: off[lo] <= e < off[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= e) lo = mid; else hi = mid;
    }
    return (u32)lo;
}

// the finalize step of compare (finalize_rows_kernel): ones on the diagonal, common / max(1, union)
__host__ __device__ __forceinline__ double stripe_jaccard(u32 common, u64 size_i, u64 size_j, bool diagonal) {
    if (diagonal) return 1.0;
    const u64 un = size_i + size_j - common;
    return (double)common / (double)(un > 1 ? un : 1);
}

// Column of a stripe that holds the counter of row j.  Inside every whole block of 32 columns the low five bits are
// XORed with the block index: rows a fixed stride apart (related genomes listed at regular distances -- the benchmark's
// families are rows f, f + 100, f + 200, ...: 8 banks for 25 lanes, 5 wavefronts per ATOMS) spread over all banks.
// The tags of the stream carry this column, so the count kernel pays nothing; its output stage reads counter
// stripe_col(j) for column j (a permutation inside each block: conflict-free).  `swz` = number of columns in whole
// blocks (the last partial block stays as it is), 0 = no swizzle.
__host__ __device__ __forceinline__ u32 stripe_col(u32 j, u32 swz) { return j < swz ? j ^ ((j >> 5) & 31u) : j; }

// rows per CTA for a stripe of `ncols` u32 counters per row in `smem_bytes` of shared memory
__host__ __device__ __forceinline__ int stripe_rows_per_block(size_t smem_bytes, int ncols) {
    if (smem_bytes <= (size_t)STRIPE_HEADER || ncols <= 0) return 0;
    const size_t r = (smem_bytes - STRIPE_HEADER) / ((size_t)ncols * sizeof(u32));
    return (int)(r > (size_t)STRIPE_MAX_ROWS ? (size_t)STRIPE_MAX_ROWS : r);
}

// number of low hash bits that do not fit the 32-bit sort key (0 when every key fits)
__host__ __device__ __forceinline__ int stripe_low_bits(u64 max_key) {
    int bits = 1;
    while (bits < 64 && (max_key >> bits)) ++bits;
    return bits > 32 ? bits - 32 : 0;
}

// ---- stream construction ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) stripe_keys_kernel(const u64* __restrict__ h, u64 T, int low_bits,
                                                         u32* __restrict__ key32, u64* __restrict__ payload) {
    const u64 low_mask = low_bits ? ((1ull << low_bits) - 1ull) : 0ull;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < T; e += (u64)gridDim.x * blockDim.x) {
        const u64 x = h[e];
        key32[e] = (u32)(x >> low_bits);
        payload[e] = ((x & low_mask) << 32) | e;
    }
}

// eblk[b] = row that owns element b << STRIPE_EBLK_LOG2
__global__ void __launch_bounds__(256) stripe_eblk_kernel(const u64* __restrict__ off, int n, u64 T, u32* __restrict__ eblk) {
    const u64 nblk = (T >> STRIPE_EBLK_LOG2) + 1;
    for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += (u64)gridDim.x * blockDim.x) {
        const u64 e = b << STRIPE_EBLK_LOG2;
        eblk[b] = e < T ? stripe_row_of(off, n, e) : (u32)(n > 0 ? n - 1 : 0);
    }
}

__global__ void __launch_bounds__(256) stripe_sizes_kernel(const u64* __restrict__ off, int n, u32* __restrict__ sizes) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) sizes[r] = (u32)(off[r + 1] - off[r]);
}

// Runs (equal 32-bit keys) whose payloads do not ascend hold more than one hash, interleaved.  The tag kernel
// below sees every (predecessor, element) pair of the stream anyway: the thread that meets the FIRST descent of a
// run appends the run's head to a worklist (the list can hold every element, so it never overflows), and
// stripe_fix_kernel redoes the tags and positions of the listed runs -- one warp per run: the payloads are
// ranked against each other (they are distinct: they end in the element index) and written in order to `tmp`
// (the sort's input buffer, which held the position buckets and is free again once stripe_pos_window_kernel has
// run; a run uses the slots of its own stream positions), then the run's tags and positions are derived from the
// ordered payloads -- after the position pass, whose positions of these runs they overwrite.  Ascending payloads =
// ascending (low bits, element) = groups contiguous, rows ascending.
__device__ __forceinline__ void stripe_note_descent(const u32* __restrict__ key32s, const u64* __restrict__ pays, u64 q, u32 k,
                                                    u32* __restrict__ worklist, u32* __restrict__ d_count) {
    u64 p = q - 1;                                        // q: a descent (same key as q - 1, smaller payload).  Any earlier one in this run?
    while (p > 0 && key32s[p - 1] == k) {
        if (pays[p] < pays[p - 1]) return;
        --p;
    }
    worklist[atomicAdd(d_count, 1u)] = (u32)p;            // p = head of the run
}

// ---- the inverse permutation pos[e] = q, written window by window ------------------------------------------
// Stored directly, pos[e] = q is one 4-byte write per element to a random place of a T_all x 4 B array (200 MB for
// the benchmark's 5e7 elements, four times the L2): nearly every write lands on a sector that is not resident and
// costs a partial-sector write to HBM.  Instead the tag kernel appends (e << 32 | q) to the bucket of e's window of
// pos[] (2^lg elements, a slice that fits the L2 several times over), and stripe_pos_window_kernel writes the
// buckets out in window order: each window's lines are written while they stay in L2 and leave it whole, once.
// Every element of the stream occurs once, so the size of every bucket is known before the tag kernel runs, the
// order inside a bucket does not matter, and pos[] is the same whatever order the CTAs append in.

// log2 of the window: the largest power of two with 4 B x window <= L2 / 3 (so that the window, the bucket stream
// passing through and the tags being written share the L2), or `requested` (a power of two, rounded down; 0 = the
// rule); raised until the T_all elements span at most STRIPE_MAX_WINDOWS windows
__host__ __device__ __forceinline__ int stripe_pos_window_log2(u64 l2_bytes, u64 requested, u64 T_all) {
    int lg = 0;
    if (requested) while ((2ull << lg) <= requested) ++lg;
    else while ((12ull << (lg + 1)) <= l2_bytes) ++lg;
    while (T_all && ((T_all - 1) >> lg) >= (u64)STRIPE_MAX_WINDOWS) ++lg;
    return lg < 31 ? lg : 31;                             // elements are u32
}

// bucket offsets: boff[w] = number of stream elements e < w << lg, for w = 0 .. nw (boff[nw] = T), and the
// append cursors cur[w] = boff[w].  The stream holds the elements [ebeg[r], eend[r]) of every row r (whole rows, or
// a key-range shard's slices), doff[r] of them in rows < r; the rows' CSR ranges off[] ascend, so the count below
// x is doff[r] + the part of row r's range below x, for the row r whose CSR range holds x.
__global__ void __launch_bounds__(256) stripe_window_offsets_kernel(const u64* __restrict__ off, int n, const u64* __restrict__ ebeg,
                                                                   const u64* __restrict__ eend, const u64* __restrict__ doff,
                                                                   u64 T_all, u64 T, int lg, u32 nw, u32* __restrict__ boff,
                                                                   u32* __restrict__ cur) {
    for (u32 w = blockIdx.x * blockDim.x + threadIdx.x; w <= nw; w += gridDim.x * blockDim.x) {
        const u64 x = (u64)w << lg;
        u64 below = T;
        if (x < T_all) {
            const u32 r = stripe_row_of(off, n, x);
            const u64 b = ebeg[r], len = eend[r] - b;
            below = doff[r] + (x > b ? (x - b < len ? x - b : len) : 0);
        }
        boff[w] = (u32)below;
        if (w < nw) cur[w] = (u32)below;
    }
}

// sorted (key, payload) stream -> tags (row | head flag), and the (element, position) pairs of the inverse
// permutation appended to the buckets of their pos[] windows.  A CTA takes tiles of U x blockDim consecutive stream
// positions; per tile each element takes a rank in its window from a shared counter, one atomicAdd per (tile,
// window) on the window's cursor reserves the tile's run of the bucket, and the elements are written into it.
// Without buckets (null `bucket`: pos[] is a single window, T_all <= 2^lg) pos[e] = q is stored here -- the whole
// array stays in L2, so the store costs what the window pass's would, without the 8 B per element of buckets.
// U positions per thread, their loads issued together: the chain of dependent loads (payload -> block table -> row
// offsets) hits L1 and is bound by latency; the tags and buckets are written in order.
static constexpr int STRIPE_TAG_U = 8;                // stream positions per thread and tile (tiles of 2048 at 256 threads)
static constexpr int STRIPE_TAG_TILE = STRIPE_TAG_U * 256;
template <typename TagT>
__global__ void __launch_bounds__(256) stripe_tag_kernel(const u32* __restrict__ key32s, const u64* __restrict__ pays,
                                                        const u64* __restrict__ off, const u32* __restrict__ eblk, u64 T,
                                                        TagT* __restrict__ tags, u32* __restrict__ pos, u32* __restrict__ worklist,
                                                        u32* __restrict__ d_count, u32 swz, u64* __restrict__ bucket = nullptr,
                                                        u32* __restrict__ cur = nullptr, int lg = 0, u32 nw = 0) {
    constexpr int U = STRIPE_TAG_U;
    SMB_SHARED u32 s_cnt[STRIPE_MAX_WINDOWS];             // elements of the tile per window, then ...
    SMB_SHARED u32 s_base[STRIPE_MAX_WINDOWS];            // ... where the tile's run of each bucket starts
    const u64 tile = (u64)U * blockDim.x;
    for (u64 t0 = (u64)blockIdx.x * tile; t0 < T; t0 += (u64)gridDim.x * tile) {
        if (bucket) {
            for (u32 w = threadIdx.x; w < nw; w += blockDim.x) s_cnt[w] = 0;
            __syncthreads();
        }
        u64 p[U], pp[U];
        u32 k[U], kp[U], r[U], rk[U];
        u64 nx[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const u64 q = t0 + (u64)u * blockDim.x + threadIdx.x;
            const bool in = q < T;
            p[u] = in ? pays[q] : 0;
            k[u] = in ? key32s[q] : 0;
            pp[u] = (in && q) ? pays[q - 1] : ~0ull;
            kp[u] = (in && q) ? key32s[q - 1] : 0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] = eblk[(u32)p[u] >> STRIPE_EBLK_LOG2];
#pragma unroll
        for (int u = 0; u < U; ++u) nx[u] = off[r[u] + 1];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const u64 q = t0 + (u64)u * blockDim.x + threadIdx.x;
            if (q >= T) continue;
            const u32 e = (u32)p[u];
            const bool head = q == 0 || k[u] != kp[u] || (p[u] >> 32) != (pp[u] >> 32);
            u32 rr = r[u];
            u64 end = nx[u];
            while (end <= (u64)e) end = off[++rr + 1];    // e < T_all = off[n]: stops at the owning row, empty rows skipped
            tags[q] = (TagT)(stripe_col(rr, swz) | (head ? StripeTag<TagT>::HEAD : 0u));
            if (bucket) rk[u] = atomicAdd(&s_cnt[e >> lg], 1u);
            else pos[e] = (u32)q;                         // one window: all of pos[] stays in L2
            // a run that mixes hashes (null worklist: the keys hold every bit, no such runs)
            if (worklist && q && k[u] == kp[u] && p[u] < pp[u]) stripe_note_descent(key32s, pays, q, k[u], worklist, d_count);
        }
        if (!bucket) continue;                            // uniform: a kernel parameter
        __syncthreads();
        for (u32 w = threadIdx.x; w < nw; w += blockDim.x) {
            const u32 c = s_cnt[w];
            if (c) s_base[w] = atomicAdd(cur + w, c);
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const u64 q = t0 + (u64)u * blockDim.x + threadIdx.x;
            if (q >= T) continue;
            const u32 e = (u32)p[u];
            bucket[s_base[e >> lg] + rk[u]] = ((u64)e << 32) | q;
        }
    }
    // STRIPE_TAG_PAD head flags behind the end: the count kernel reads ahead of a group without bounds checks
    const u64 gt = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (gt < (u64)STRIPE_TAG_PAD) tags[T + gt] = (TagT)StripeTag<TagT>::HEAD;
}

// the buckets in window order -> pos[e] = q.  Each block takes STRIPE_POS_PER_BLOCK consecutive pairs and blocks
// start in index order, so the resident blocks work on one or two windows of pos[] at a time; the pairs are read once
// (evict-first: they must not push the window out of the L2).
static constexpr int STRIPE_POS_UNROLL = 4;
__global__ void __launch_bounds__(256) stripe_pos_window_kernel(const u64* __restrict__ bucket, u64 T, u32* __restrict__ pos) {
    const u64 i0 = (u64)blockIdx.x * blockDim.x * STRIPE_POS_UNROLL + threadIdx.x;
    u64 v[STRIPE_POS_UNROLL];
#pragma unroll
    for (int u = 0; u < STRIPE_POS_UNROLL; ++u) {
        const u64 i = i0 + (u64)u * blockDim.x;
        v[u] = i < T ? ld_stream_u64(bucket + i) : ~0ull;
    }
#pragma unroll
    for (int u = 0; u < STRIPE_POS_UNROLL; ++u)
        if (v[u] != ~0ull) pos[v[u] >> 32] = (u32)v[u];
}

// the listed runs again, in order (see stripe_note_descent)
template <typename TagT>
__global__ void __launch_bounds__(128) stripe_fix_kernel(const u32* __restrict__ key32s, const u64* __restrict__ pays, u64 T,
                                                        const u32* __restrict__ worklist, const u32* __restrict__ d_count,
                                                        const u64* __restrict__ off, int n, u64* tmp, TagT* tags, u32* pos, u32 swz) {
    const u32 count = *d_count;
    const u32 lane = lane_id();
    const u32 warps = gridDim.x * (blockDim.x >> 5);
    for (u32 i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < count; i += warps) {
        const u64 head = worklist[i];
        const u32 k = key32s[head];
        u64 tail = head + 1;                              // end of the run: 32 positions probed at a time
        for (;;) {
            const u64 q = tail + lane;
            const bool same = q < T && key32s[q] == k;
            const u32 m = __ballot_sync(0xffffffffu, !same);
            if (m) { tail += (u64)(__ffs((int)m) - 1); break; }
            tail += 32;
        }
        for (u64 a = head + lane; a < tail; a += 32) {
            const u64 v = pays[a];
            u64 rank = 0;
            for (u64 b = head; b < tail; ++b) rank += pays[b] < v ? 1u : 0u;
            tmp[head + rank] = v;
        }
        __syncwarp();                                     // tmp[head, tail) written by this warp, read by it below
        for (u64 q = head + lane; q < tail; q += 32) {
            const u64 v = tmp[q];
            const bool first = q == head || (tmp[q - 1] >> 32) != (v >> 32);
            const u32 e = (u32)v;
            tags[q] = (TagT)(stripe_col(stripe_row_of(off, n, (u64)e), swz) | (first ? StripeTag<TagT>::HEAD : 0u));
            pos[e] = (u32)q;
        }
        __syncwarp();
    }
}

// ---- the count kernel -------------------------------------------------------------------------------------
struct StripeArgs {
    const void* tags;        // u16 or u32 (template parameter of the kernel)
    const u32* pos;
    const u64* ebeg;         // per row: the CSR elements [ebeg[r], eend[r]) that are in the stream -- the whole row
    const u64* eend;         //   (off, off + 1), or its slice of one key range when the stream holds a shard of the keys
    const u32* sizes;        // row lengths (whole rows: the Jaccard denominators)
    u64 T;                   // elements in the stream
    int n, rows_per_block, row_begin, row_end;
    double* out;             // float64 Jaccard rows, row `row_begin` first, leading dimension n (null: counts only)
    u32* out_counts;         // raw counters of the rows instead (a key-range shard's partial counts), same layout
    u16* out_counts16;       // ... as 16-bit counters (rows shorter than 65 536 hashes: half the bytes to exchange)
    u32 swz;                 // the tags hold stripe_col(row, swz)
};

// A counter of the stripe is bumped through the 32-bit shared-memory address of its row: one address add and one
// ATOMS per increment.  (atomicAdd on the generic pointer made the compiler rebuild the shared-window base --
// S2UR, UMOV, ULEA, IMAD, LEA -- for every increment under its 32-register budget: 13 instructions against 9.)
#ifdef SMB_SIMT_EMUL
typedef u32* StripeRowRef;                                            // the emulator has no shared address space
inline StripeRowRef stripe_row_ref(u32* row) { return row; }
inline void stripe_inc_if(StripeRowRef row, u32 col, bool on) { if (on) atomicAdd(row + col, 1u); }
#else
typedef u32 StripeRowRef;
__device__ __forceinline__ StripeRowRef stripe_row_ref(u32* row) { return (u32)__cvta_generic_to_shared(row); }
__device__ __forceinline__ void stripe_inc_if(StripeRowRef row, u32 col, bool on) {
    // (ptxas keeps a short branch around the ATOMS either way: its increment form aggregates over the converged lanes)
    if (on) asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(row + (col << 2)) : "memory");
}
#endif

// One CTA = rows [r0, r1) of the result.  Work items are (row, chunk of 32 consecutive elements), handed to the
// warps chunk index first, so that all rows of the CTA -- and, as CTAs start together, all CTAs of a wave --
// move through the hash-ordered stream together.  For every element with a successor in its group the warp
// reads the 32 tags behind it (two elements' reads in flight), and 32 more while no group head has turned up; the
// lanes in front of the next group head increment their counters.  UPPER: only later members (= higher rows) are counted, i.e. the cells (i, j > i);
// stripe_mirror_kernel fills the rest.  Otherwise the members in front are counted too (full rows, used when a
// block of rows is computed on its own).
template <typename TagT, bool UPPER, int CTAS>
__global__ void __launch_bounds__(1024, CTAS) join_stripe_kernel(StripeArgs a) {
    constexpr u32 HEAD = StripeTag<TagT>::HEAD;
    SMB_DYN_SHARED(unsigned char, stripe_smem);
    u64* s_beg = reinterpret_cast<u64*>(stripe_smem);                       // [rows]
    u64* s_end = s_beg + STRIPE_MAX_ROWS;                                   // [rows]
    u32* s_ctl = reinterpret_cast<u32*>(stripe_smem + 2 * STRIPE_MAX_ROWS * sizeof(u64));   // [0] next item, [1] chunks of the longest row
    u32* stripe = reinterpret_cast<u32*>(stripe_smem + STRIPE_HEADER);      // [rows][n]
    const TagT* __restrict__ tags = reinterpret_cast<const TagT*>(a.tags);
    const int r0 = a.row_begin + (int)blockIdx.x * a.rows_per_block;
    const int r1 = min(a.row_end, r0 + a.rows_per_block);
    const int rows = r1 - r0;
    const u32 n = (u32)a.n;
    for (u32 i = threadIdx.x; i < (u32)rows; i += blockDim.x) { s_beg[i] = a.ebeg[r0 + i]; s_end[i] = a.eend[r0 + i]; }
    if (threadIdx.x == 0) { s_ctl[0] = 0; s_ctl[1] = 0; }
    for (u32 i = threadIdx.x; i < (u32)rows * n; i += blockDim.x) stripe[i] = 0;
    __syncthreads();
    for (u32 i = threadIdx.x; i < (u32)rows; i += blockDim.x) atomicMax(&s_ctl[1], (u32)((s_end[i] - s_beg[i] + 31) >> 5));
    __syncthreads();
    const u32 lane = lane_id();
    const u32 n_items = s_ctl[1] * (u32)rows;
    const u32 le_mask = (2u << lane) - 1u;                // lanes <= lane
    const u32 lt_mask = (1u << lane) - 1u;                // lanes <  lane

    for (;;) {
        u32 k = 0;
        if (lane == 0) k = atomicAdd(&s_ctl[0], 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= n_items) break;
        const u32 c = k / (u32)rows, r = k - c * (u32)rows;
        const u64 e0 = s_beg[r] + ((u64)c << 5);
        const u64 re = s_end[r];
        if (e0 >= re) continue;                            // a shorter row: no such chunk
        const u64 e = e0 + lane;
        const bool have = e < re;
        const u32 my_q = have ? ld_stream_u32(a.pos + e) : 0u;
        u32* row_ptr = stripe + (size_t)r * n;

        // ---- members behind the element (higher rows): the 32 tags behind it, two elements' reads in flight per
        // round, then 32 more at a time only while no group head has turned up.  The kernel is bound by the sectors it
        // reads from L2 / HBM, not by the latency of a read: reading 64 tags up front (the benchmark's elements
        // have ~29 members behind them on average) fetched tags past the group's end that nobody counts.  A lane
        // counts its tag when no group head lies at or in front of it (m & le_mask == 0); a tag is the stripe column of
        // its row (stripe_col), and that of a tag that is not counted is still a valid column (the padding tags are
        // HEAD | 0), so addresses need no guard.  Every read lies inside the STRIPE_TAG_PAD head flags behind the stream:
        // a read of 32 tags is only issued when the previous one ended inside the group, whose end is at most T.
        const StripeRowRef row_ref = stripe_row_ref(row_ptr);
        const u32 lane1 = lane + 1u;
        u32 nxt = HEAD;
        if (have) nxt = (u32)tags[(size_t)my_q + 1];
        u32 todo = __ballot_sync(0xffffffffu, nxt < HEAD);
        while (todo) {
            const int j0 = __ffs(todo) - 1;
            todo &= todo - 1;
            const bool two = todo != 0;                    // uniform in the warp
            const int j1 = two ? __ffs(todo) - 1 : j0;
            todo &= todo - 1;                              // 0 stays 0
            // 32-bit position + lane + 1 (no wrap: T < 2^32 - 128), widened once per element
            const TagT* __restrict__ p0 = tags + (__shfl_sync(0xffffffffu, my_q, j0) + lane1);
            const TagT* __restrict__ p1 = tags + (__shfl_sync(0xffffffffu, my_q, j1) + lane1);
            const u32 t0 = (u32)p0[0];
            u32 t1 = HEAD;
            if (two) t1 = (u32)p1[0];
            u32 m = __ballot_sync(0xffffffffu, t0 >= HEAD);
            stripe_inc_if(row_ref, t0 & (HEAD - 1u), (m & le_mask) == 0);
            for (u32 it = 1; m == 0; ++it) {               // more than 32 members behind
                const u32 tt = (u32)p0[32 * it];
                m = __ballot_sync(0xffffffffu, tt >= HEAD);
                stripe_inc_if(row_ref, tt & (HEAD - 1u), (m & le_mask) == 0);
            }
            if (two) {
                m = __ballot_sync(0xffffffffu, t1 >= HEAD);
                stripe_inc_if(row_ref, t1 & (HEAD - 1u), (m & le_mask) == 0);
                for (u32 it = 1; m == 0; ++it) {
                    const u32 tt = (u32)p1[32 * it];
                    m = __ballot_sync(0xffffffffu, tt >= HEAD);
                    stripe_inc_if(row_ref, tt & (HEAD - 1u), (m & le_mask) == 0);
                }
            }
        }
        if (UPPER) continue;

        // ---- members in front of the element (lower rows); the head of the group is one of them
        const u32 self = have ? (u32)tags[my_q] : HEAD;
        todo = __ballot_sync(0xffffffffu, (self & HEAD) == 0);
        while (todo) {
            const int j = __ffs(todo) - 1;
            todo &= todo - 1;
            const u32 q = __shfl_sync(0xffffffffu, my_q, j);
            u32 m = 0;
            for (u32 it = 0; m == 0; ++it) {
                const u32 d = 1 + 32 * it + lane;
                const bool vv = q >= d;
                const u32 tt = vv ? (u32)tags[q - d] : HEAD;
                m = __ballot_sync(0xffffffffu, !vv || (tt & HEAD) != 0);
                if (vv && (m & lt_mask) == 0) atomicAdd(row_ptr + (tt & ~HEAD), 1u);
            }
        }
    }
    __syncthreads();
    // counts -> float64 rows, written once (streaming stores: the matrix is not read again by this kernel)
    for (int al = 0; al < rows; ++al) {
        const int row = r0 + al;
        const u32* __restrict__ srow = stripe + (size_t)al * n;
        if (a.out_counts) {                                // a shard of the keys: partial counts, summed over the shards later
            u32* __restrict__ crow = a.out_counts + (size_t)(row - a.row_begin) * n;
            for (u32 j = threadIdx.x; j < n; j += blockDim.x)
                if (!UPPER || j >= (u32)row) crow[j] = srow[stripe_col(j, a.swz)];     // UPPER: the caller mirrors (a shard's counts are symmetric)
            continue;
        }
        if (a.out_counts16) {
            u16* __restrict__ crow = a.out_counts16 + (size_t)(row - a.row_begin) * n;
            for (u32 j = threadIdx.x; j < n; j += blockDim.x)
                if (!UPPER || j >= (u32)row) crow[j] = (u16)srow[stripe_col(j, a.swz)];
            continue;
        }
        const u64 si = a.sizes[row];
        double* __restrict__ orow = a.out + (size_t)(row - a.row_begin) * n;
        for (u32 j = threadIdx.x; j < n; j += blockDim.x) {
            if (UPPER && j < (u32)row) continue;
            st_stream_f64(orow + j, stripe_jaccard(srow[stripe_col(j, a.swz)], si, a.sizes[j], (u32)row == j));
        }
    }
}

// a shard's row slices -> 32-bit sort keys + payloads (element index = position in the whole CSR), written back to back
__global__ void __launch_bounds__(256) stripe_keys_slice_kernel(const u64* __restrict__ h, const u64* __restrict__ ebeg,
                                                               const u64* __restrict__ dst_off, int n, int low_bits,
                                                               u32* __restrict__ key32, u64* __restrict__ payload) {
    const u64 low_mask = low_bits ? ((1ull << low_bits) - 1ull) : 0ull;
    for (int r = blockIdx.x; r < n; r += gridDim.x) {
        const u64 src = ebeg[r], d0 = dst_off[r], m = dst_off[r + 1] - d0;
        for (u64 i = threadIdx.x; i < m; i += blockDim.x) {
            const u64 x = h[src + i];
            key32[d0 + i] = (u32)(x >> low_bits);
            payload[d0 + i] = ((x & low_mask) << 32) | (src + i);
        }
    }
}

// ebeg[r] = off[r] + beg[r], eend[r] = ebeg[r] + cnt[r]: the slices of join_row_range_kernel as CSR element ranges
__global__ void __launch_bounds__(256) stripe_slice_ranges_kernel(const u64* __restrict__ off, const u64* __restrict__ beg,
                                                                 const u64* __restrict__ cnt, int n, u64* __restrict__ ebeg,
                                                                 u64* __restrict__ eend) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    ebeg[r] = off[r] + beg[r];
    eend[r] = off[r] + beg[r] + cnt[r];
}

// u32 counters -> u16 (the upper-triangle shards of the tile kernel / the global-reduction join, narrowed for the exchange)
__global__ void __launch_bounds__(256) stripe_narrow_counts_kernel(const u32* __restrict__ in, u64 total, u16* __restrict__ out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) out[i] = (u16)in[i];
}

// counters of rows [row_begin, row_end) (row_begin first, whole rows), summed over the shards -> float64 Jaccard rows
template <typename CountT>
__global__ void __launch_bounds__(256) stripe_finalize_counts_kernel(const CountT* __restrict__ counts, const u64* __restrict__ off,
                                                                    int n, int row_begin, int row_end, double* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = row_begin + (int)blockIdx.y;
    if (j >= n || i >= row_end) return;
    const size_t cell = (size_t)(i - row_begin) * n + j;
    st_stream_f64(out + cell, stripe_jaccard((u32)counts[cell], off[i + 1] - off[i], off[j + 1] - off[j], i == j));
}

// out[i][j] = out[j][i] for i in [row_begin, row_end), j < i: 64 x 64 tiles through shared memory (four cells
// per thread, so that a CTA has 32 KB of float64 in flight: with 32 x 32 tiles the kernel was bound by latency),
// reads and writes both coalesced.  `full` points at row 0 of the whole matrix (rows < row_end
// are complete in their upper part).
static constexpr int STRIPE_MIRROR_TILE = 64;
template <typename T>
__global__ void __launch_bounds__(1024) stripe_mirror_kernel(T* __restrict__ full, int n, int row_begin, int row_end) {
    constexpr int W = STRIPE_MIRROR_TILE;
    SMB_SHARED T tile[W][W + 1];
    const int ti = row_begin / W + (int)blockIdx.y;        // tile row (destination rows)
    const int tj = (int)blockIdx.x;                        // tile column (destination columns), tj <= ti
    if (tj > ti) return;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    // source tile = rows of tile column tj, columns of tile row ti (the upper part)
#pragma unroll
    for (int a = 0; a < W; a += 32)
#pragma unroll
        for (int b = 0; b < W; b += 32) {
            const int sr = tj * W + ty + a, sc = ti * W + tx + b;
            tile[ty + a][tx + b] = (sr < n && sc < n) ? full[(size_t)sr * n + sc] : T(0);
        }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < W; a += 32)
#pragma unroll
        for (int b = 0; b < W; b += 32) {
            const int dr = ti * W + ty + a, dc = tj * W + tx + b;
            if (dr >= row_begin && dr < row_end && dc < dr && dc < n) full[(size_t)dr * n + dc] = tile[tx + b][ty + a];
        }
}

}  // namespace smb
