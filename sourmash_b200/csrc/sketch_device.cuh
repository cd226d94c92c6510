// sketch_device.cuh -- the rolled hashing kernels of sketch_kernels.cu (hash_kmers_kernel<K>, and the
// experimental one-pass hash_kmers_fused_kernel) with their argument block, and the kernels that turn
// the candidates of a row into a sketch row (block-wide bitonic sort, unique, run lengths).  In a header so that
// tests/host_emul/simt_sketch_emul.cu can compile the kernels themselves for the host (tests/host_emul/simt.h)
// and run them -- tiling, survivor staging, flushes included -- against the oracle without a GPU.
#pragma once
#include "common.cuh"
#include "kmer_roll.cuh"

namespace smb {

static constexpr int HASH_THREADS = 128;
static constexpr int STAGE_CAP = 1024;          // per-CTA survivor staging (u64 entries)

struct HashArgs {
    const u8* bases;              // 16-byte aligned allocation, readable up to the next 16-byte boundary
    const u64* stream_off;        // [n_streams] byte offset of stream s (any alignment)
    const u64* stream_len;        // [n_streams] length in bytes
    const u32* stream_row;        // [n_streams] output sketch of stream s (NULL: s)
    const u32* tile_start;        // [n_streams + 1] prefix sum of tiles per stream
    int n_streams;
    int W;                        // windows per thread (multiple of 16)
    u64 seed, max_hash;
    u64* cand;                    // candidate storage
    const u64* cand_off;          // [n_rows + 1]
    u32* cand_cnt;                // [n_rows]
    u32 tile_base;                // first tile of this launch (launches may cover a range of tiles)
    int row_stride, row_index;    // row = sketch * row_stride + row_index
    u64* raw_out;                 // RAW mode: per-window hashes of stream 0 (0 = invalid)
};

__device__ __forceinline__ int find_stream(const u32* __restrict__ tile_start, int n_streams, u32 tile) {
    int lo = 0, hi = n_streams;                    // last stream with tile_start <= tile
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (tile_start[mid] <= tile) lo = mid; else hi = mid; }
    return lo;
}

template <int K, bool RAW>
__global__ void __launch_bounds__(HASH_THREADS) hash_kmers_kernel(HashArgs a) {
    SMB_SHARED u64 s_buf[STAGE_CAP];
    SMB_SHARED u32 s_cnt;
    SMB_SHARED u32 s_base;
    SMB_SHARED int s_stream;
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_cnt = 0;
        s_stream = find_stream(a.tile_start, a.n_streams, blockIdx.x + a.tile_base);
    }
    __syncthreads();
    const int stream = s_stream;
    // aligned coordinates: the stream starts `lead` bytes into its first 16-byte line; the
    // lead bytes belong to whatever precedes the stream and are masked to "invalid".
    const u64 s0 = a.stream_off[stream];
    const u64 b0 = s0 & ~15ull;
    const u32 lead = (u32)(s0 - b0);
    const u64 Lp = (u64)lead + a.stream_len[stream];
    const u8* __restrict__ base = a.bases + b0;
    const u64 tile = blockIdx.x + a.tile_base - a.tile_start[stream];
    const u64 w0 = (tile * HASH_THREADS + tid) * (u64)a.W;
    const int sk = a.stream_row ? (int)a.stream_row[stream] : stream;
    const int row = sk * a.row_stride + a.row_index;

    hash_thread_windows<K>(base, Lp, lead, w0, a.W, a.seed, [&](u64 w, bool valid, u64 h) {
        if (RAW) {
            if (w >= lead && w + K <= Lp) a.raw_out[w - lead] = valid ? h : 0ull;
        } else if (valid && h != 0ull && h <= a.max_hash) {
            u32 slot = atomicAdd(&s_cnt, 1u);
            if (slot < STAGE_CAP) {
                s_buf[slot] = h;
            } else {                                  // staging full: append directly
                u32 g = atomicAdd(&a.cand_cnt[row], 1u);
                u64 capr = a.cand_off[row + 1] - a.cand_off[row];
                if (g < capr) a.cand[a.cand_off[row] + g] = h;
            }
        }
    });
    if (RAW) return;
    __syncthreads();
    const u32 n = min(s_cnt, (u32)STAGE_CAP);
    if (n == 0) return;
    if (tid == 0) s_base = atomicAdd(&a.cand_cnt[row], n);
    __syncthreads();
    const u64 off = a.cand_off[row];
    const u64 capr = a.cand_off[row + 1] - off;
    for (u32 i = tid; i < n; i += HASH_THREADS) {
        u64 g = (u64)s_base + i;
        if (g < capr) a.cand[off + g] = s_buf[i];
    }
}

// ---------------------------------------------------------------------------------------
// The default for k = 21, 31, 51 requested together (SMB_SKETCH_FUSED=0 switches it off; kmer_roll.cuh hash_thread_windows_fused): k = 21, 31
// and 51 of `sourmash sketch dna`'s default parameter string in ONE pass over the bases -- one
// rolling 51-state, the shorter k-mers read off it as prefixes -- instead of three launches that each
// decode and roll the same bases.  Logic checked on the CPU by
// tests/test_host_emulation.py::test_roll_fused_21_31_51_matches_oracle; on an H100 12.4 ms against 13.8 ms for the three
// launches over 100 x 5 Mbp (bench.py --workload sketch, SMB_SKETCH_FUSED=0 for the second).
// ---------------------------------------------------------------------------------------
struct FusedArgs {
    HashArgs a;                   // row_index / max_hash unused
    int row_index[3];             // output row of k = 21, 31, 51 inside a sketch's group of rows
    u64 max_hash[3];
};

__global__ void __launch_bounds__(HASH_THREADS) hash_kmers_fused_kernel(FusedArgs f) {
    SMB_SHARED u64 s_buf[3][STAGE_CAP];
    SMB_SHARED u32 s_cnt[3];
    SMB_SHARED u32 s_base[3];
    SMB_SHARED int s_stream;
    const HashArgs& a = f.a;
    const int tid = threadIdx.x;
    if (tid < 3) s_cnt[tid] = 0;
    if (tid == 0) s_stream = find_stream(a.tile_start, a.n_streams, blockIdx.x + a.tile_base);
    __syncthreads();
    const int stream = s_stream;
    const u64 s0 = a.stream_off[stream];
    const u64 b0 = s0 & ~15ull;
    const u32 lead = (u32)(s0 - b0);
    const u64 Lp = (u64)lead + a.stream_len[stream];
    const u8* __restrict__ base = a.bases + b0;
    const u64 tile = blockIdx.x + a.tile_base - a.tile_start[stream];
    const u64 w0 = (tile * HASH_THREADS + tid) * (u64)a.W;
    const int sk = a.stream_row ? (int)a.stream_row[stream] : stream;
    const int row0 = sk * a.row_stride;

    hash_thread_windows_fused(base, Lp, lead, w0, a.W, a.seed, [&](u64, int which, bool valid, u64 h) {
        if (valid && h != 0ull && h <= f.max_hash[which]) {
            const u32 slot = atomicAdd(&s_cnt[which], 1u);
            if (slot < STAGE_CAP) {
                s_buf[which][slot] = h;
            } else {                                  // staging full: append directly
                const int row = row0 + f.row_index[which];
                const u32 g = atomicAdd(&a.cand_cnt[row], 1u);
                const u64 capr = a.cand_off[row + 1] - a.cand_off[row];
                if (g < capr) a.cand[a.cand_off[row] + g] = h;
            }
        }
    });
    __syncthreads();
    if (tid < 3) {
        const u32 n = min(s_cnt[tid], (u32)STAGE_CAP);
        s_cnt[tid] = n;
        s_base[tid] = n ? atomicAdd(&a.cand_cnt[row0 + f.row_index[tid]], n) : 0u;
    }
    __syncthreads();
#pragma unroll 1
    for (int which = 0; which < 3; ++which) {
        const u32 n = s_cnt[which];
        const int row = row0 + f.row_index[which];
        const u64 off = a.cand_off[row];
        const u64 capr = a.cand_off[row + 1] - off;
        for (u32 i = tid; i < n; i += HASH_THREADS) {
            const u64 g = (u64)s_base[which] + i;
            if (g < capr) a.cand[off + g] = s_buf[which][i];
        }
    }
}

// ---- row materialisation: sort + unique (+ run lengths) of each row's candidates (moved from sketch_kernels.cu) ----
static constexpr int SORT_THREADS = 1024;
static constexpr int SORT_MAX = 16384;            // rows up to this many candidates sort in smem

__global__ void __launch_bounds__(SORT_THREADS) sort_unique_small_kernel(
    u64* __restrict__ cand, const u64* __restrict__ cand_off, const u32* __restrict__ cand_cnt,
    u32* __restrict__ out_cnt, u64* __restrict__ abund) {
    SMB_DYN_SHARED(unsigned char, smem_raw);
    const int r = blockIdx.x;
    const u64 off = cand_off[r];
    const u64 capr = cand_off[r + 1] - off;
    u32 n = cand_cnt[r];
    if ((u64)n > capr || n > SORT_MAX) return;          // overflowed / big row: handled on host path
    if (n == 0) { if (threadIdx.x == 0) out_cnt[r] = 0; return; }
    u32 np2 = 1; while (np2 < n) np2 <<= 1;
    u64* s = reinterpret_cast<u64*>(smem_raw);
    u32* heads = reinterpret_cast<u32*>(smem_raw + (size_t)np2 * 8);
    const int tid = threadIdx.x;
    for (u32 i = tid; i < np2; i += SORT_THREADS) s[i] = i < n ? cand[off + i] : SMB_U64_MAX;
    __syncthreads();
    for (u32 k = 2; k <= np2; k <<= 1) {
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            for (u32 i = tid; i < np2; i += SORT_THREADS) {
                u32 ixj = i ^ j;
                if (ixj > i) {
                    u64 x = s[i], y = s[ixj];
                    bool up = (i & k) == 0;
                    if ((x > y) == up) { s[i] = y; s[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
    // unique: stable compaction of run heads
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u32 carry;
    if (tid == 0) carry = 0;
    __syncthreads();
    const int lane = tid & 31, warp = tid >> 5;
    for (u32 base = 0; base < n; base += SORT_THREADS) {
        u32 i = base + tid;
        bool head = i < n && (i == 0 || s[i] != s[i - 1]);
        u32 bal = __ballot_sync(0xffffffffu, head);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        u32 before = 0;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        u32 pos = carry + before + __popc(bal & ((1u << lane) - 1u));
        if (head) { cand[off + pos] = s[i]; heads[pos] = i; }
        __syncthreads();
        if (tid == 0) { u32 t = 0; for (int w2 = 0; w2 < SORT_THREADS / 32; ++w2) t += warp_tot[w2]; carry += t; }
        __syncthreads();
    }
    const u32 m = carry;
    if (abund) {
        for (u32 p = tid; p < m; p += SORT_THREADS) {
            u32 nxt = p + 1 < m ? heads[p + 1] : n;
            abund[off + p] = (u64)(nxt - heads[p]);
        }
    }
    if (tid == 0) out_cnt[r] = m;
}

__global__ void __launch_bounds__(SORT_THREADS) unique_sorted_row_kernel(
    const u64* __restrict__ sorted, u64 n, u64* __restrict__ out, u64* __restrict__ abund,
    u64* __restrict__ head_idx, u32* __restrict__ out_cnt) {
    SMB_SHARED u32 warp_tot[32];
    SMB_SHARED u64 carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (u64 base = 0; base < n; base += SORT_THREADS) {
        u64 i = base + tid;
        bool head = i < n && (i == 0 || sorted[i] != sorted[i - 1]);
        u32 bal = __ballot_sync(0xffffffffu, head);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        u32 before = 0;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        u64 pos = carry + before + __popc(bal & ((1u << lane) - 1u));
        if (head) { out[pos] = sorted[i]; head_idx[pos] = i; }
        __syncthreads();
        if (tid == 0) { u32 t = 0; for (int w2 = 0; w2 < SORT_THREADS / 32; ++w2) t += warp_tot[w2]; carry += t; }
        __syncthreads();
    }
    const u64 m = carry;
    if (abund) {
        for (u64 p = tid; p < m; p += SORT_THREADS) {
            u64 nxt = p + 1 < m ? head_idx[p + 1] : n;
            abund[p] = nxt - head_idx[p];
        }
    }
    if (tid == 0) *out_cnt = (u32)m;
}

}  // namespace smb
