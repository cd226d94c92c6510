// compare_kernels.cu -- sorted-u64 hash-set intersection kernels for sm_90a (H100).
//
// Replaces the reference's per-pair CPU loops:
//   count_common          src/core/src/sketch/minhash.rs:539-558 (+ Intersection :915-953)
//   intersection_size     src/core/src/sketch/minhash.rs:593-621, free fn :1765-1807
//   intersection          src/core/src/sketch/minhash.rs:560-589, free fn :1721-1763
//   jaccard               src/core/src/sketch/minhash.rs:624-631
// driven in the reference by Python loops (src/sourmash/compare.py:14-187,
// src/sourmash/index/__init__.py:115-170,777-909).
//
// Design: integer/byte work, no tensor cores.  The hot kernel keeps TA "table" rows
// resident in shared memory as sorted keys + a bucket directory (bucket = key >> shift, the
// keys are murmur outputs, i.e. uniform), and streams the other operand's rows through
// registers with coalesced 8-byte loads: each streamed element costs one directory lookup
// plus two key compares per table ("directory galloping"), instead of a two-pointer walk
// over |A|+|B| elements.  Counts are reduced with warp REDUX and written as u32.
#include <stdlib.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <memory>

#include "common.cuh"
#include "kernels.h"
#include "split_table.cuh"
#include "join_walk.cuh"
#include "join_kernels.cuh"
#include "join_stripe.cuh"
#include "range_search.cuh"
#include "range_kernels.cuh"
#include "db_index.cuh"
#include "db_index_kernels.cuh"
#include "search_kernels.cuh"
#include "multigather_kernels.cuh"
#include "tile_kernels.cuh"
#include "pair_kernels.cuh"
#include "sketch_combine.cuh"
#include "angular_search.cuh"

namespace smb {

// stream-ordered scratch allocations released at scope exit, error paths included
struct JoinScratch {
    cudaStream_t s;
    void* p[16] = {};
    int n = 0;
    explicit JoinScratch(cudaStream_t st) : s(st) {}
    cudaError_t alloc(void** out, size_t bytes) {
        cudaError_t e = cudaMallocAsync(out, bytes ? bytes : 16, s);
        if (e == cudaSuccess && n < 16) p[n++] = *out;
        return e;
    }
    ~JoinScratch() { for (int i = 0; i < n; ++i) cudaFreeAsync(p[i], s); }
};

static int tile_threads() {
    static int v = [] { const char* e = getenv("SMB_TILE_THREADS"); int t = e ? atoi(e) : 1024; return (t == 256 || t == 512 || t == 1024) ? t : 1024; }();
    return v;
}
static int tile_cols_override() {
    static int v = [] { const char* e = getenv("SMB_TILE_COLS"); return e ? atoi(e) : 0; }();
    return v;
}

// ------------------------------------------------------------------------------------
// bucket shift: (max key) >> shift < 2^nb_log2
// ------------------------------------------------------------------------------------

// max over the last (largest) key of every row -> *d_max (zeroed by the caller)
void launch_max_last(const u64* hA, const u64* offA, int nA, const u64* hB, const u64* offB, int nB,
                     unsigned long long* d_max, cudaStream_t s) {
    int total = nA + nB;
    if (total <= 0) return;
    int blocks = (total + 255) / 256;
    if (blocks > SMB_SMS * 4) blocks = SMB_SMS * 4;
    max_last_kernel<<<blocks, 256, 0, s>>>(hA, offA, nA, hB, offB, nB, d_max); count_launches(1);
}

// ------------------------------------------------------------------------------------
// tile kernel
// ------------------------------------------------------------------------------------
// Bucket = key >> shift with buckets 0 .. (max_key >> shift): the directory covers exactly the
// occupied key range, and shift is the finest one whose directory still fits next to the keys.
// Prefer more tables per CTA (fewer passes over the streamed rows) as long as the buckets stay
// sparse (<= ~0.45 keys per bucket at the largest row), because denser buckets mean the
// deferred long-bucket scan runs in nearly every batch.
PairwisePlan plan_pairwise(uint64_t max_len_a, uint64_t max_key, int n_b) {
    (void)n_b;
    return plan_pairwise_impl(max_len_a, max_key, tile_cols_override());
}

static int tile_variant() {       // SMB_TILE_VARIANT=u64 selects the v1 kernel for A/B measurements
    static int v = [] { const char* e = getenv("SMB_TILE_VARIANT"); return (e && e[0] == 'u') ? 0 : 1; }();
    return v;
}

template <int TA>
static void launch_tile_ta(const TileArgs& args, size_t smem, cudaStream_t s) {
    // split-word kernel for every row size that fits shared memory (15-bit positions); the u64
    // kernels stay selectable (SMB_TILE_VARIANT=u64) for A/B measurements
    auto kern = tile_variant() && args.cap < 32760 ? pairwise_tile_split_kernel<TA, 4>
              : (args.cap < 16380 ? pairwise_tile_kernel<TA, 4, true> : pairwise_tile_kernel<TA, 4, false>);
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int tiles = (args.nA + TA - 1) / TA;
    int my_tiles = (tiles - args.tile_offset + args.tile_stride - 1) / args.tile_stride;
    if (args.tile_count >= 0 && my_tiles > args.tile_count) my_tiles = args.tile_count;
    if (my_tiles <= 0) return;
    dim3 grid(my_tiles, (args.nB + args.cols_per_cta - 1) / args.cols_per_cta);
    kern<<<grid, tile_threads(), smem, s>>>(args); count_launches(1);
}

void launch_pairwise_tile(const PairwisePlan& plan, const u64* hA, const u64* offA, int nA,
                          const u64* hB, const u64* offB, int nB, u32* out, size_t ldo,
                          bool symmetric, TileShard tiles, cudaStream_t s) {
    if (nA <= 0 || nB <= 0) return;
    TileArgs a{hA, offA, nA, hB, offB, nB, out, ldo,
               plan.shift, plan.nb, plan.cap, plan.cols_per_cta, symmetric ? 1 : 0,
               tiles.shard, tiles.n_shards > 0 ? tiles.n_shards : 1, tiles.count};
    switch (plan.tables_per_cta) {
        case 1: launch_tile_ta<1>(a, plan.smem_bytes, s); break;
        case 2: launch_tile_ta<2>(a, plan.smem_bytes, s); break;
        case 3: launch_tile_ta<3>(a, plan.smem_bytes, s); break;
        default: launch_tile_ta<4>(a, plan.smem_bytes, s); break;
    }
}

// ------------------------------------------------------------------------------------
// generic fallback: warp per pair, binary search of the shorter row in the longer row
// ------------------------------------------------------------------------------------


void launch_pairwise_generic(const u64* hA, const u64* offA, int nA, const u64* hB,
                             const u64* offB, int nB, u32* out, size_t ldo, bool symmetric,
                             TileShard tiles, cudaStream_t s) {
    if (nA <= 0 || nB <= 0) return;
    u64 npairs = (u64)nA * (u64)nB;
    u64 blocks = (npairs + 7) / 8;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    pairwise_generic_kernel<<<(unsigned)blocks, 256, 0, s>>>(hA, offA, nA, hB, offB, nB, out, ldo,
                                                            symmetric ? 1 : 0, tiles.shard,
                                                            tiles.n_shards > 0 ? tiles.n_shards : 1); count_launches(1);
}

// ------------------------------------------------------------------------------------
// bottom-k ("num") sketches -- minhash.rs:593-617.  M = first `num` of A ∪ B.
// The union rank of a_i is i + lower_bound(B, a_i) - (#matches among a_0..a_{i-1}); a common
// element counts iff its rank < num.  One warp per pair; prefix of matches by ballot.
// ------------------------------------------------------------------------------------

void launch_pairwise_num(const u64* hA, const u64* offA, int nA, const u64* hB, const u64* offB,
                         int nB, u32 num, u32* common, u32* usize, size_t ldo, bool symmetric,
                         cudaStream_t s) {
    if (nA <= 0 || nB <= 0) return;
    u64 npairs = (u64)nA * (u64)nB;
    u64 blocks = (npairs + 7) / 8;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    pairwise_num_kernel<<<(unsigned)blocks, 256, 0, s>>>(hA, offA, nA, hB, offB, nB, num, common,
                                                        usize, ldo, symmetric ? 1 : 0); count_launches(1);
}

// ------------------------------------------------------------------------------------
// angular similarity of abundance sketches (minhash.rs:635-680): warp per pair,
// dot = sum a_i*b_j over common hashes (u64, wrapping like the reference's release build),
// value = 1 - 2*acos(min(dot / (|a| |b|), 1)) / pi.  acos runs on the device (<= 2 ulp from
// libm, far inside the 1e-12 tolerance).
// ------------------------------------------------------------------------------------


void launch_pairwise_angular(const u64* h, const u64* ab, const u64* off, int n,
                             unsigned long long* d_sumsq, double* out, cudaStream_t s) {
    if (n <= 0) return;
    int b1 = (n + 7) / 8; if (b1 > SMB_SMS * 16) b1 = SMB_SMS * 16;
    row_sumsq_kernel<<<b1, 256, 0, s>>>(ab, off, n, d_sumsq); count_launches(1);
    u64 npairs = (u64)n * (u64)n;
    u64 blocks = (npairs + 7) / 8;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    pairwise_angular_kernel<<<(unsigned)blocks, 256, 0, s>>>(h, ab, off, n, d_sumsq, out); count_launches(1);
}

// ------------------------------------------------------------------------------------
// counts -> float64 matrix (jaccard = common / max(1, union), minhash.rs:624-631;
// IEEE div.rn.f64 is bit-identical to the reference's f64 divide).
// ------------------------------------------------------------------------------------

void launch_finalize_matrix(const u32* common, const u32* usize, size_t ldo, const u64* offA,
                            const u64* offB, int nA, int nB, int mode, bool symmetric, double* out,
                            cudaStream_t s) {
    if (nA <= 0 || nB <= 0) return;
    dim3 grid((nB + 255) / 256, nA);
    finalize_matrix_kernel<<<grid, 256, 0, s>>>(common, usize, ldo, offA, offB, nA, nB, mode,
                                                symmetric ? 1 : 0, out); count_launches(1);
}


void launch_finalize_rows(const u32* common, size_t n, const u64* off, int n_rows, int row_begin,
                          int row_end, double* out, cudaStream_t s) {
    (void)n_rows;
    if (row_end <= row_begin) return;
    dim3 grid(((int)n + 255) / 256, row_end - row_begin);
    finalize_rows_kernel<<<grid, 256, 0, s>>>(common, n, off, row_begin, row_end, out); count_launches(1);
}

// ------------------------------------------------------------------------------------
// one (large) query vs many subjects: global-memory directory over the query
// ------------------------------------------------------------------------------------
// dir[b] = #query keys with (key >> shift) < b, b in [0, nb].  Pass 1 presets "unset", pass 2
// lets every key that opens a bucket write its index and fill short runs of empty buckets
// behind it, pass 3 resolves the remaining (long) empty runs by binary search -- no thread ever
// walks a long gap serially, whatever the key distribution.




void launch_build_global_dir(const u64* q, u64 nq, int shift, u64 nb, u32* dir, cudaStream_t s) {
    const u64 cap_blocks = (u64)SMB_SMS * 32;
    u64 b1 = (nb + 1 + 255) / 256; if (b1 > cap_blocks) b1 = cap_blocks;
    global_dir_fill_kernel<<<(unsigned)b1, 256, 0, s>>>(dir, nb + 1, DIR_UNSET); count_launches(1);
    if (nq) {
        u64 b2 = (nq + 255) / 256; if (b2 > cap_blocks) b2 = cap_blocks;
        global_dir_heads_kernel<<<(unsigned)b2, 256, 0, s>>>(q, nq, (u32)shift, dir); count_launches(1);
    }
    global_dir_resolve_kernel<<<(unsigned)b1, 256, 0, s>>>(q, nq, (u32)shift, nb, dir); count_launches(1);
}


void launch_build_query_bitmap(const u64* q, u64 nq, int shift, int fine_log2,
                               u32* bitmap, cudaStream_t s) {
    if (nq == 0) return;
    u64 blocks = (nq + 255) / 256;
    if (blocks > (u64)SMB_SMS * 32) blocks = (u64)SMB_SMS * 32;
    build_query_bitmap_kernel<<<(unsigned)blocks, 256, 0, s>>>(q, nq, (u32)shift, fine_log2, bitmap); count_launches(1);
}


void launch_one_vs_many_global(const u64* q, u64 nq, const u32* dir, int shift, u64 nb,
                               const u32* bitmap, int fine_log2, const u64* hB,
                               const u64* offB, int nB, u32* out, cudaStream_t s) {
    if (nB <= 0) return;
    int blocks = (nB + 7) / 8;
    if (blocks > SMB_SMS * 16) blocks = SMB_SMS * 16;
    one_vs_many_global_kernel<<<blocks, 256, 0, s>>>(q, nq, dir, (u32)shift, nb, bitmap, fine_log2,
                                                     hB, offB, nB, out); count_launches(1);
}

// ------------------------------------------------------------------------------------
// Range-major copy of a resident set + the streaming one-vs-many pass over it (range_kernels.cuh): the path for
// queries too large for shared memory.  SMB_SEARCH_LAYOUT=global keeps the global-directory kernel (A/B runs).
// ------------------------------------------------------------------------------------
struct RangeMajor {
    cudaStream_t stream = 0;
    void *m_rm = nullptr, *m_slice = nullptr, *m_coarse = nullptr;
    int n = 0, P = 0, nc = 0;
    u64 width = 0, T = 0;
    u32 bm_shift = 0;
    ~RangeMajor() {
        if (m_rm) cudaFreeAsync(m_rm, stream);
        if (m_slice) cudaFreeAsync(m_slice, stream);
        if (m_coarse) cudaFreeAsync(m_coarse, stream);
    }
};

int range_major_parts(u64 T) {
    const char* e = getenv("SMB_RM_RANGES");              // tests: few ranges on small sets
    if (e && atoi(e) > 0) return atoi(e);
    // two CTAs per SM, a whole number of waves; fewer, larger parts for small sets
    return T >= (32u << 20) ? SMB_SMS * 10 : SMB_SMS * 2;
}

// *out stays null (with cudaSuccess) when the layout does not apply (positions must fit 32 bits)
cudaError_t range_major_build(const u64* h, const u64* off, int n, u64 T, u64 max_key, RangeMajor** out, cudaStream_t s) {
    *out = nullptr;
    const int P = range_major_parts(T);
    if (n <= 0 || T == 0 || T >= 0xffffffffull || (u64)n * (u64)(P + 1) >= 0x7fffffffull) return cudaSuccess;
    auto rm = new RangeMajor();
    std::unique_ptr<RangeMajor> guard(rm);
    rm->stream = s; rm->n = n; rm->P = P; rm->T = T;
    rm->width = range_width(max_key, P);
    rm->bm_shift = range_bitmap_shift(rm->width, 1ull << RM_BITMAP_LOG2);
    cudaError_t e;
    const size_t cells = (size_t)n * (size_t)P;
    if ((e = cudaMallocAsync(&rm->m_rm, (T + 64) * sizeof(u64), s)) != cudaSuccess) return e;
    if ((e = cudaMallocAsync(&rm->m_slice, (cells + 1) * sizeof(u32), s)) != cudaSuccess) return e;
    JoinScratch scratch(s);
    u32 *bounds = nullptr, *cnt = nullptr;
    if ((e = scratch.alloc((void**)&bounds, (cells + n) * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&cnt, (cells + 1) * sizeof(u32))) != cudaSuccess) return e;
    rm_bounds_kernel<<<SMB_SMS * 16, 256, 0, s>>>(h, off, n, rm->width, P, bounds);
    const unsigned grid = (unsigned)std::min<u64>((cells + 256) / 256, (u64)SMB_SMS * 32);
    rm_counts_kernel<<<grid, 256, 0, s>>>(bounds, n, P, cnt);
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt, (u32*)rm->m_slice, (long long)(cells + 1), s);
    void* d_scan = nullptr;
    if ((e = scratch.alloc(&d_scan, scan_bytes)) != cudaSuccess) return e;
    cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, cnt, (u32*)rm->m_slice, (long long)(cells + 1), s);
    rm_scatter_kernel<<<grid, 256, 0, s>>>(h, off, bounds, (const u32*)rm->m_slice, n, P, (u64*)rm->m_rm);
    rm->nc = (n >> RM_COARSE_LOG2) + 2;
    if ((e = cudaMallocAsync(&rm->m_coarse, (size_t)P * rm->nc * sizeof(u32), s)) != cudaSuccess) return e;
    rm_coarse_kernel<<<(unsigned)std::min<u64>(((u64)P * rm->nc + 255) / 256, (u64)SMB_SMS * 32), 256, 0, s>>>(
        (const u32*)rm->m_slice, n, P, rm->nc, (u32*)rm->m_coarse);
    count_launches(5);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    *out = guard.release();
    return cudaSuccess;
}
void range_major_destroy(RangeMajor* rm) { delete rm; }

// the pass over one key stream: one query (qid null) or the merged keys of a group (range_kernels.cuh)
static void launch_range_major_pass(const RangeMajor* rm, const u64* q, const u32* qid, u64 nq, u32* out, cudaStream_t s) {
    if (nq == 0 || rm->n == 0) return;
    RangeMajorArgs a{q, nq, (const u64*)rm->m_rm, (const u32*)rm->m_slice, (const u32*)rm->m_coarse, rm->nc, rm->n, rm->P, rm->width, (u32)RM_BITMAP_LOG2, rm->bm_shift, out, qid};
    const size_t smem = ((size_t)1 << (RM_BITMAP_LOG2 - 3)) + (size_t)(RM_THREADS / 32) * RM_QUEUE * sizeof(u32);
    cudaFuncSetAttribute(one_vs_many_range_major_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    one_vs_many_range_major_kernel<<<rm->P, RM_THREADS, smem, s>>>(a); count_launches(1);
}
void launch_one_vs_many_range_major(const RangeMajor* rm, const u64* q, u64 nq, u32* out, cudaStream_t s) {
    launch_range_major_pass(rm, q, nullptr, nq, out, s);
}

// Query keys per range of one many-query group.  The bitmap alone would take 32 768 (two probes set at most 12 % of its
// 2^19 bits), but the settled matches grow with the group: against configs[4] (every query with its own planted rows)
// groups of 8 queries (1 060 keys per range) beat one pass per query on an H100, groups of 32 (4 240) and 128 (17 000)
// were slower -- each match costs a binary search in the range's keys and a row attribution, done by one warp
static constexpr u64 RM_GROUP_KEYS_PER_RANGE = 1024;
u64 range_major_group_keys(const RangeMajor* rm) { return RM_GROUP_KEYS_PER_RANGE * (u64)rm->P; }

void launch_query_stats(const u64* q, const u64* d_qoff, int G, u32* ids, unsigned long long* d_stat, cudaStream_t s) {
    if (G <= 0) return;
    rm_query_ids_kernel<<<std::min(G, SMB_SMS * 8), 256, 0, s>>>(q, d_qoff, G, ids, d_stat); count_launches(1);
}

cudaError_t many_vs_many_range_major(const RangeMajor* rm, const u64* q, const u64* d_qoff, int G, u64 n_keys,
                                     u32* out, bool* unsorted, cudaStream_t s) {
    *unsorted = false;
    if (n_keys == 0 || rm->n == 0) return cudaSuccess;
    JoinScratch scratch(s);
    u64* keys = nullptr;
    u32 *ids_in = nullptr, *ids = nullptr;
    unsigned long long* d_stat = nullptr;
    cudaError_t e;
    if ((e = scratch.alloc((void**)&keys, n_keys * sizeof(u64))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&ids_in, n_keys * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&ids, n_keys * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&d_stat, 2 * sizeof(unsigned long long))) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d_stat, 0, 2 * sizeof(unsigned long long), s)) != cudaSuccess) return e;
    launch_query_stats(q, d_qoff, G, ids_in, d_stat, s);
    unsigned long long stat[2] = {0, 0};
    if ((e = cudaMemcpyAsync(stat, d_stat, sizeof(stat), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
    if (stat[1]) { *unsorted = true; return cudaSuccess; }
    int end_bit = 1;
    while (end_bit < 64 && (stat[0] >> end_bit)) ++end_bit;
    // stable: inside a run of equal keys the ids keep the query order
    size_t sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, q, keys, ids_in, ids, (long long)n_keys, 0, end_bit, s);
    void* d_sort = nullptr;
    if ((e = scratch.alloc(&d_sort, sort_bytes)) != cudaSuccess) return e;
    cub::DeviceRadixSort::SortPairs(d_sort, sort_bytes, q, keys, ids_in, ids, (long long)n_keys, 0, end_bit, s);
    count_launches(1);
    launch_range_major_pass(rm, keys, ids, n_keys, out, s);
    return cudaGetLastError();
}
bool range_search_enabled() {
    const char* layout = getenv("SMB_SEARCH_LAYOUT");
    return !(layout && !strcmp(layout, "global"));
}

// ------------------------------------------------------------------------------------
// row-level set operations used by gather (single block; rows are a few 1e3..1e6 keys)
// ------------------------------------------------------------------------------------



void launch_intersect_alive(const u64* q, u64 nq, const u8* alive, const u64* row, u64 rn, u64* out,
                            u32* d_n, cudaStream_t s) {
    intersect_alive_kernel<<<1, 1024, 0, s>>>(q, nq, alive, row, rn, out, d_n); count_launches(1);
}


void launch_mark_dead(const u64* q, u64 nq, u8* alive, const u64* gone, u64 n, cudaStream_t s) {
    if (n == 0) return;
    u64 blocks = (n + 255) / 256;
    if (blocks > (u64)SMB_SMS * 8) blocks = (u64)SMB_SMS * 8;
    mark_dead_kernel<<<(unsigned)blocks, 256, 0, s>>>(q, nq, alive, gone, n); count_launches(1);
}

void launch_counter_update_argmax_pick(u32* counters, const u32* delta, int n, const GatherPicks& g, cudaStream_t s) {
    counter_update_argmax_pick_kernel<<<1, 1024, 0, s>>>(counters, delta, n, g); count_launches(1);
}
void launch_intersect_alive_pick(const u64* q, u64 nq, u8* alive, const u64* hashes, const u64* off, const GatherPicks& g,
                                 u64* out, u32* d_n, cudaStream_t s) {
    intersect_alive_pick_kernel<<<1, 1024, 0, s>>>(q, nq, alive, hashes, off, g, out, d_n); count_launches(1);
}

void launch_make_row_offsets(const u32* d_n, u64* d_off2, cudaStream_t s) {
    make_row_offsets_kernel<<<1, 1, 0, s>>>(d_n, d_off2); count_launches(1);
}

void launch_mark_dead_n(const u64* q, u64 nq, u8* alive, const u64* gone, const u32* d_n, cudaStream_t s) {
    mark_dead_n_kernel<<<64, 256, 0, s>>>(q, nq, alive, gone, d_n); count_launches(1);
}

void launch_multi_gather_round(const MultiGatherArgs& a, u32 cta_total, size_t smem_bytes, cudaStream_t s) {
    if (a.n_queries <= 0) return;
    multi_counter_update_argmax_pick_kernel<<<a.n_queries, 1024, 0, s>>>(a); count_launches(1);
    multi_intersect_alive_pick_kernel<<<a.n_queries, 1024, 0, s>>>(a); count_launches(1);
    if (cta_total == 0) return;
    cudaFuncSetAttribute(multi_decrement_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    multi_decrement_kernel<<<cta_total, 512, smem_bytes, s>>>(a); count_launches(1);
}

void launch_intersect_rows(const u64* a, u64 na, const u64* b, u64 nb, u64* out, u32* d_n,
                           cudaStream_t s) {
    if (nb < na) { const u64* t = a; a = b; b = t; u64 tn = na; na = nb; nb = tn; }   // probe with the shorter row
    setop_rows_kernel<true><<<1, 1024, 0, s>>>(a, na, b, nb, out, d_n); count_launches(1);
}
void launch_subtract_rows(const u64* a, u64 na, const u64* b, u64 nb, u64* out, u32* d_n,
                          cudaStream_t s) {
    setop_rows_kernel<false><<<1, 1024, 0, s>>>(a, na, b, nb, out, d_n); count_launches(1);
}


void launch_counter_update_argmax(u32* counters, const u32* delta, int n,
                                  unsigned long long* d_best, cudaStream_t s) {
    counter_update_argmax_kernel<<<1, 1024, 0, s>>>(counters, delta, n, d_best); count_launches(1);
}

// ------------------------------------------------------------------------------------
// All-vs-all counts by inverted join (sort by hash, count co-occurrences).
//
// |A_i ∩ A_j| = number of hashes that occur in both rows, so the whole count matrix is the sum,
// over every distinct hash h, of one increment for every pair of rows containing h.  Sorting the
// (hash, row) pairs of the whole set groups the rows of each hash together (radix sort, ~55 key
// bits, stable => row ids ascending inside a group); a group of m rows contributes C(m,2)
// increments.  The work is output sensitive: sum over pairs of |A_i ∩ A_j| increments plus one
// sort, instead of |A_i| + |A_j| probes for every pair -- unrelated pairs, the bulk of a real
// all-vs-all matrix, cost nothing.  The planner falls back to the tile kernel when the estimated
// number of increments says the join would be slower (e.g. thousands of near-identical sketches).
// Multi-GPU: rank r joins the hashes of key range r (every hash lives in exactly one range), the
// partial matrices add up.
// ------------------------------------------------------------------------------------
// Slice rows to [key_lo, key_hi) (bounded_hi == 0: no upper bound), sort the (hash, row) pairs.
// Returns the number of elements; *keys_out / *ids_out point into `work`, which the caller frees.
struct JoinWork {
    void* mem = nullptr;
    cudaStream_t stream = 0;
    ~JoinWork() { if (mem) cudaFreeAsync(mem, stream); }
    u64 *keys_a = nullptr, *keys_b = nullptr;
    u32 *ids_a = nullptr, *ids_b = nullptr;
    u64 T = 0;
};
static cudaError_t join_sort_slice(const u64* h, const u64* off, int n, u64 key_lo, u64 key_hi,
                                   int bounded_hi, int key_bits, JoinWork& W, cudaStream_t s) {
    JoinScratch scratch(s);
    u64* d_beg = nullptr;
    cudaError_t e;
    const size_t nn = (size_t)n + 1;
    if ((e = scratch.alloc((void**)&d_beg, nn * 3 * sizeof(u64))) != cudaSuccess) return e;
    u64 *d_cnt = d_beg + nn, *d_doff = d_cnt + nn;
    join_row_range_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, s>>>(h, off, n, key_lo, key_hi, bounded_hi, d_beg, d_cnt);
    count_launches(1);
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_cnt, d_doff, (int)nn, s);
    void* d_scan = nullptr;
    if ((e = scratch.alloc(&d_scan, scan_bytes)) != cudaSuccess) return e;
    cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_cnt, d_doff, (int)nn, s);
    u64 T = 0;
    cudaMemcpyAsync(&T, d_doff + n, sizeof(u64), cudaMemcpyDeviceToHost, s);
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
    W.T = T;
    if (T == 0) return cudaSuccess;
    const size_t Tp = (size_t)((T + 63) & ~63ull);
    if ((e = cudaMallocAsync(&W.mem, Tp * (2 * sizeof(u64) + 2 * sizeof(u32)), s)) != cudaSuccess) return e;
    W.keys_a = (u64*)W.mem; W.keys_b = W.keys_a + Tp;
    W.ids_a = (u32*)(W.keys_b + Tp); W.ids_b = W.ids_a + Tp;
    int blocks = n < SMB_SMS * 16 ? n : SMB_SMS * 16;
    join_gather_kernel<<<blocks, 256, 0, s>>>(h, off, d_beg, d_doff, n, W.keys_a, W.ids_a); count_launches(1);
    size_t sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, W.keys_a, W.keys_b, W.ids_a, W.ids_b, (long long)T, 0, key_bits, s);
    void* d_sort = nullptr;
    if ((e = scratch.alloc(&d_sort, sort_bytes)) != cudaSuccess) return e;
    cub::DeviceRadixSort::SortPairs(d_sort, sort_bytes, W.keys_a, W.keys_b, W.ids_a, W.ids_b, (long long)T, 0, key_bits, s);
    count_launches(1);
    return cudaGetLastError();
}

static int key_bit_length(u64 max_key) { int b = 1; while (b < 64 && (max_key >> b)) ++b; return b; }

cudaError_t join_estimate(const u64* h, const u64* off, int n, u64 max_key, unsigned long long* d_out2,
                          double* est_increments, double* est_elements, unsigned long long* max_group,
                          cudaStream_t s) {
    // deterministic sample: the lowest 1/64 of the key range (identical on every rank that holds the
    // same set, so all ranks take the same decision)
    const u64 hi = max_key / JOIN_SAMPLE + 1;
    JoinWork W;
    cudaError_t e = join_sort_slice(h, off, n, 0, hi, 1, key_bit_length(hi), W, s);
    W.stream = s;
    if (e != cudaSuccess) return e;
    unsigned long long r[2] = {0, 0};
    cudaMemsetAsync(d_out2, 0, 2 * sizeof(unsigned long long), s);
    if (W.T) {
        u64 blocks = (W.T + 255) / 256;
        if (blocks > (u64)SMB_SMS * 32) blocks = (u64)SMB_SMS * 32;
        join_estimate_kernel<<<(unsigned)blocks, 256, 0, s>>>(W.keys_b, W.T, d_out2); count_launches(1);
    }
    cudaMemcpyAsync(r, d_out2, sizeof r, cudaMemcpyDeviceToHost, s);
    e = cudaStreamSynchronize(s);
    *est_increments = (double)r[0] * JOIN_SAMPLE;
    *est_elements = (double)W.T * JOIN_SAMPLE;
    *max_group = r[1];
    return e;
}

// ------------------------------------------------------------------------------------
// Stripe layout of the inverted join (join_stripe.cuh): the default all-vs-all path.  CTAs own complete
// rows of the result as shared-memory counters; no count matrix in HBM, no global atomics, float64 rows
// written once.  SMB_JOIN_LAYOUT=plain selects the global-reduction join (join_counts) for A/B runs,
// SMB_JOIN_LAYOUT=stripe_full counts both directions in every launch (no mirror pass).
// ------------------------------------------------------------------------------------
struct JoinStripe {
    cudaStream_t stream = 0;
    void* mem = nullptr;      // tags + pos + sizes + order + sel (+ the slice ranges of a key-range shard)
    void* tags = nullptr;
    u32 *pos = nullptr, *sizes = nullptr;
    u32* order = nullptr;     // the rows in the order they are counted: ascending label (stripe_label_kernel), row inside a label
    u32* sel = nullptr;       // sel[row_begin, row_end): the rows of a launch over that range, in `order`'s order
    u32* succ = nullptr;      // successor bit of every CSR element (stripe_tag_kernel): the count kernel's test for later members
    const u64 *ebeg = nullptr, *eend = nullptr;
    u64 T = 0;                // elements in the stream (all of the set, or one key range of it)
    int n = 0, rows_per_block = 0, upper_only = 1, tag16 = 0, sharded = 0;
    unsigned swz = 0;         // tags hold stripe_col(row, swz): counters of rows a fixed stride apart spread over the banks
    int ctas_per_sm = 1;      // 2: rows_per_block sized for two resident CTAs (64 warps per SM; the count kernel is bound by issue latency)
    size_t smem = 0;
    ~JoinStripe() { if (mem) cudaFreeAsync(mem, stream); }
};

// shared memory of one CTA when two are to be resident: 2 x (dynamic + 1 KB reserved per CTA) <= 228 KB per SM
static constexpr size_t STRIPE_SMEM_TWO_CTAS = 112 * 1024;
template <typename TagT, bool UPPER, int CTAS>
static cudaError_t stripe_set_smem_one() {
    cudaError_t e = cudaFuncSetAttribute(join_stripe_kernel<TagT, UPPER, CTAS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         CTAS == 2 ? (int)STRIPE_SMEM_TWO_CTAS : MAX_DYN_SMEM);
    if (e != cudaSuccess || CTAS != 2) return e;
    return cudaFuncSetAttribute(join_stripe_kernel<TagT, UPPER, CTAS>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                cudaSharedmemCarveoutMaxShared);
}
template <typename TagT>
static cudaError_t stripe_set_smem() {
    cudaError_t e;
    if ((e = stripe_set_smem_one<TagT, true, 1>()) != cudaSuccess) return e;
    if ((e = stripe_set_smem_one<TagT, false, 1>()) != cudaSuccess) return e;
    if ((e = stripe_set_smem_one<TagT, true, 2>()) != cudaSuccess) return e;
    return stripe_set_smem_one<TagT, false, 2>();
}

// js->order from the finished stream: one label per row, then a stable sort of the rows by label (rows ascending
// inside a label; a set with no shared hashes keeps the identity order)
static cudaError_t stripe_make_order(JoinStripe* js, JoinScratch& scratch, cudaStream_t s) {
    const int n = js->n;
    u32* lab = nullptr;
    cudaError_t e;
    if ((e = scratch.alloc((void**)&lab, 3 * (size_t)n * sizeof(u32))) != cudaSuccess) return e;
    u32 *lab_out = lab + n, *rowid = lab_out + n;
    const unsigned grid = (unsigned)std::min((n + 7) / 8, SMB_SMS * 8);       // one warp per row
    if (js->tag16) stripe_label_kernel<u16><<<grid, 256, 0, s>>>((const u16*)js->tags, js->pos, js->ebeg, js->eend, n, js->swz, lab, rowid);
    else stripe_label_kernel<u32><<<grid, 256, 0, s>>>((const u32*)js->tags, js->pos, js->ebeg, js->eend, n, js->swz, lab, rowid);
    count_launches(1);
    const int bits = key_bit_length((u64)n);
    size_t sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, lab, lab_out, rowid, js->order, n, 0, bits, s);
    void* d_sort = nullptr;
    if ((e = scratch.alloc(&d_sort, sort_bytes)) != cudaSuccess) return e;
    cub::DeviceRadixSort::SortPairs(d_sort, sort_bytes, lab, lab_out, rowid, js->order, n, 0, bits, s);
    count_launches(1);
    return cudaGetLastError();
}

// *out stays null (with cudaSuccess) when the layout does not apply: 2^32 - 256 or more elements, or a row of n
// counters that does not fit in shared memory.  n_shards > 1: the stream holds only the hashes of key range
// `shard` (every hash lies in exactly one range, so the counts of the shards add up); that costs one 8-byte
// readback (the number of elements in the range sizes the sort).  Otherwise nothing synchronises.
cudaError_t join_stripe_create_shard(const u64* h, const u64* off, int n, u64 T_all, u64 max_key, int shard, int n_shards,
                                     JoinStripe** out, cudaStream_t s) {
    *out = nullptr;
    int R = n > 0 ? stripe_rows_per_block((size_t)MAX_DYN_SMEM, n) : 0;
    int ctas = 1;
    {   // two CTAs per SM when a row block of at least one row fits half the shared memory (SMB_STRIPE_CTAS=1: A/B switch)
        const int R2 = n > 0 ? stripe_rows_per_block(STRIPE_SMEM_TWO_CTAS, n) : 0;
        const char* c = getenv("SMB_STRIPE_CTAS");
        if (R2 >= 1 && !(c && !strcmp(c, "1"))) { R = R2; ctas = 2; }
    }
    if (R < 1 || T_all == 0 || T_all >= 0xffffff00ull) return cudaSuccess;   // 32-bit stream positions, read-ahead included
    cudaError_t e;
    if ((e = stripe_set_smem<u16>()) != cudaSuccess) return e;      // per device, so not cached in a flag
    if ((e = stripe_set_smem<u32>()) != cudaSuccess) return e;
    auto js = new JoinStripe();
    std::unique_ptr<JoinStripe> guard(js);
    js->stream = s; js->n = n; js->rows_per_block = R; js->ctas_per_sm = ctas;
    {
        const char* z = getenv("SMB_STRIPE_SWIZZLE");                // A/B: 0 = counters in column order
        js->swz = (z && !strcmp(z, "0")) ? 0u : ((unsigned)n & ~31u);
    }
    js->tag16 = n < 32768;
    js->sharded = n_shards > 1;
    {
        const char* layout = getenv("SMB_JOIN_LAYOUT");
        js->upper_only = !(layout && !strcmp(layout, "stripe_full"));
        const char* tag = getenv("SMB_STRIPE_TAGS");                 // A/B: force 32-bit tags
        if (tag && !strcmp(tag, "u32")) js->tag16 = 0;
    }
    js->smem = (size_t)STRIPE_HEADER + (size_t)R * n * sizeof(u32);
    JoinScratch scratch(s);
    const size_t np = ((size_t)n + 64) & ~(size_t)63;
    // the slices of the rows that fall into the shard's key range, and how many elements that is
    u64 T = T_all;
    u64 *d_beg = nullptr, *d_cnt = nullptr, *d_doff = nullptr;
    if (js->sharded) {
        u64 lo, hi;
        bool bounded;
        join_shard_range(max_key, shard, n_shards, lo, hi, bounded);
        const size_t nn = (size_t)n + 1;
        if ((e = scratch.alloc((void**)&d_beg, nn * 3 * sizeof(u64))) != cudaSuccess) return e;
        d_cnt = d_beg + nn; d_doff = d_cnt + nn;
        join_row_range_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, s>>>(h, off, n, lo, hi, bounded ? 1 : 0, d_beg, d_cnt);
        count_launches(1);
        size_t scan_bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_cnt, d_doff, (int)nn, s);
        void* d_scan = nullptr;
        if ((e = scratch.alloc(&d_scan, scan_bytes)) != cudaSuccess) return e;
        cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_cnt, d_doff, (int)nn, s);
        cudaMemcpyAsync(&T, d_doff + n, sizeof(u64), cudaMemcpyDeviceToHost, s);
        if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
    }
    js->T = T;
    const size_t Tp = (size_t)((T + 63) & ~63ull);
    const size_t Tall_p = (size_t)((T_all + 63) & ~63ull);
    const size_t Tt = Tp + STRIPE_TAG_PAD;                          // the tag stream + its padding of head flags
    const size_t succ_words = Tall_p / 32;                          // even: the slice ranges behind stay 8-byte aligned
    // tags | pos (indexed by CSR element: the whole set's size) | sizes | order | sel | succ (ditto) | slice ranges of a shard
    if ((e = cudaMallocAsync(&js->mem, (Tt + Tall_p + 3 * np + succ_words) * sizeof(u32) + (js->sharded ? 2 * np * sizeof(u64) : 0), s)) !=
        cudaSuccess)
        return e;
    js->tags = js->mem;
    js->pos = (u32*)js->mem + Tt;
    js->sizes = js->pos + Tall_p;
    js->order = js->sizes + np;
    js->sel = js->order + np;
    js->succ = js->sel + np;
    stripe_sizes_kernel<<<(n + 255) / 256, 256, 0, s>>>(off, n, js->sizes); count_launches(1);
    if (js->sharded) {
        u64* eb = (u64*)(js->succ + succ_words);
        stripe_slice_ranges_kernel<<<(n + 255) / 256, 256, 0, s>>>(off, d_beg, d_cnt, n, eb, eb + np); count_launches(1);
        js->ebeg = eb; js->eend = eb + np;
    } else {
        js->ebeg = off; js->eend = off + 1;
    }
    if (T == 0) {                                                   // no hash in this key range: every partial count is zero
        cudaMemsetAsync(js->succ, 0, succ_words * sizeof(u32), s);
        if (js->tag16)
            stripe_hash_tag_kernel<u16><<<1, 256, 0, s>>>(nullptr, nullptr, 0, off, nullptr, 0, (u16*)js->tags, js->pos, nullptr, nullptr, 0u,
                                                          nullptr, nullptr, 0, 0u, nullptr);
        else
            stripe_hash_tag_kernel<u32><<<1, 256, 0, s>>>(nullptr, nullptr, 0, off, nullptr, 0, (u32*)js->tags, js->pos, nullptr, nullptr, 0u,
                                                          nullptr, nullptr, 0, 0u, nullptr);
        count_launches(1);
        if ((e = stripe_make_order(js, scratch, s)) != cudaSuccess) return e;
        *out = guard.release();
        return cudaSuccess;
    }
    // windows and sub-windows of pos[] for the position pass (SMB_STRIPE_POS_WINDOW and SMB_STRIPE_POS_SUBWINDOW, numbers
    // of elements, override the rules for tests)
    const char* pw = getenv("SMB_STRIPE_POS_WINDOW");
    const char* psw = getenv("SMB_STRIPE_POS_SUBWINDOW");
    int pos_lg = 0, sub_lg = 0;
    stripe_pos_levels(SMB_L2_BYTES, pw ? strtoull(pw, nullptr, 10) : 0ull, psw ? strtoull(psw, nullptr, 10) : 0ull, T_all, pos_lg, sub_lg);
    const u32 nw = (u32)(((T_all - 1) >> pos_lg) + 1);
    const u32 nsub = (u32)(((T_all - 1) >> sub_lg) + 1);
    // the sort's bit window: the top 32 significant bits of the hashes, relative to the shard's lo
    u64 lo = 0, max_rel = max_key;
    if (js->sharded) {
        u64 hi;
        bool bounded;
        join_shard_range(max_key, shard, n_shards, lo, hi, bounded);
        max_rel = bounded ? hi - lo - 1 : max_key - lo;
    }
    int begin_bit = 0, end_bit = 0;
    stripe_sort_window(max_rel, begin_bit, end_bit);
    u64 *hs_in = nullptr, *hs = nullptr, *bucket = nullptr;
    u32 *es_in = nullptr, *es = nullptr, *eblk = nullptr, *d_count = nullptr, *boff = nullptr, *sboff = nullptr;
    if ((e = scratch.alloc((void**)&hs, Tp * sizeof(u64))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&es_in, Tp * 2 * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&bucket, Tp * sizeof(u64))) != cudaSuccess) return e;
    es = es_in + Tp;
    const u64 nblk = (T_all >> STRIPE_EBLK_LOG2) + 1;
    if ((e = scratch.alloc((void**)&eblk, (nblk + 1) * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&d_count, 16)) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&boff, (2 * (size_t)nw + 1) * sizeof(u32))) != cudaSuccess) return e;   // offsets | cursors
    if ((e = scratch.alloc((void**)&sboff, (2 * (size_t)nsub + 1) * sizeof(u32))) != cudaSuccess) return e;  // ... of the sub-windows
    const unsigned grid = (unsigned)std::min<u64>((T + 255) / 256, (u64)SMB_SMS * 32);
    // 1. the sort's input: the resident hashes themselves and an iota of their elements, or a shard's slices gathered
    //    as (hash - lo, element)
    if (js->sharded) {
        if ((e = scratch.alloc((void**)&hs_in, Tp * sizeof(u64))) != cudaSuccess) return e;
        const int blocks = n < SMB_SMS * 16 ? n : SMB_SMS * 16;
        stripe_gather_slice_kernel<<<blocks, 256, 0, s>>>(h, js->ebeg, d_doff, n, lo, hs_in, es_in);
    } else {
        stripe_iota_kernel<<<grid, 256, 0, s>>>(T, es_in);
    }
    count_launches(1);
    // 2. four radix passes over the window (fewer when the hashes are short)
    const u64* keys_in = js->sharded ? hs_in : h;
    size_t sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys_in, hs, es_in, es, (long long)T, begin_bit, end_bit, s);
    void* d_sort = nullptr;
    if ((e = scratch.alloc(&d_sort, sort_bytes)) != cudaSuccess) return e;
    cub::DeviceRadixSort::SortPairs(d_sort, sort_bytes, keys_in, hs, es_in, es, (long long)T, begin_bit, end_bit, s);
    count_launches(1);
    // 3. tags + inverse permutation + successor bits: the tag kernel appends (element, position, bit) entries to the
    //    buckets of the pos[] windows, the partition splits them into the buckets of the sub-windows (the sort's
    //    temporary storage is free: it holds cub's alternate buffers), and the sub-window pass writes pos[] and succ
    //    from shared memory; when pos[] is one window it stays in L2 as a whole and the tag kernel stores positions and
    //    bits directly.  Runs of equal window bits that hold more than one hash are noticed on the way (the iota is
    //    free: worklist) and redone in order after the position pass, one warp per run (the buckets are free again:
    //    the ordered positions of those runs)
    u32* worklist = begin_bit ? es_in : nullptr;
    if (begin_bit) cudaMemsetAsync(d_count, 0, sizeof(u32), s);
    stripe_eblk_kernel<<<(unsigned)std::min<u64>((nblk + 255) / 256, (u64)SMB_SMS * 8), 256, 0, s>>>(off, n, T_all, eblk);
    count_launches(1);
    const bool windows = nw > 1;
    const u64* doff = js->sharded ? d_doff : off;
    if (windows) {
        stripe_window_offsets_kernel<<<(nw + 256) / 256, 256, 0, s>>>(off, n, js->ebeg, js->eend, doff, T_all, T, pos_lg, nw, boff, boff + nw + 1);
        stripe_window_offsets_kernel<<<(nsub + 256) / 256, 256, 0, s>>>(off, n, js->ebeg, js->eend, doff, T_all, T, sub_lg, nsub, sboff,
                                                                        sboff + nsub + 1);
        count_launches(2);
    } else {
        cudaMemsetAsync(js->succ, 0, succ_words * sizeof(u32), s);  // the tag kernel sets the bits
    }
    const unsigned tag_grid = (unsigned)std::min<u64>((T + STRIPE_TAG_TILE - 1) / STRIPE_TAG_TILE, (u64)SMB_SMS * 16);
    if (js->tag16)
        stripe_hash_tag_kernel<u16><<<tag_grid, 256, 0, s>>>(hs, es, begin_bit, off, eblk, T, (u16*)js->tags, js->pos, worklist, d_count, js->swz,
                                                             windows ? bucket : nullptr, boff + nw + 1, pos_lg, nw, js->succ);
    else
        stripe_hash_tag_kernel<u32><<<tag_grid, 256, 0, s>>>(hs, es, begin_bit, off, eblk, T, (u32*)js->tags, js->pos, worklist, d_count, js->swz,
                                                             windows ? bucket : nullptr, boff + nw + 1, pos_lg, nw, js->succ);
    count_launches(1);
    if (windows) {
        u64* sub = (u64*)d_sort;
        if (sort_bytes < T * sizeof(u64) && (e = scratch.alloc((void**)&sub, T * sizeof(u64))) != cudaSuccess) return e;
        const u64 chunks = std::min<u64>(((1ull << pos_lg) + STRIPE_SUB_TILE - 1) / STRIPE_SUB_TILE, 1024);
        const size_t part_smem = (size_t)STRIPE_SUB_TILE * sizeof(u64);
        if ((e = cudaFuncSetAttribute(stripe_sub_partition_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)part_smem)) != cudaSuccess)
            return e;
        stripe_sub_partition_kernel<<<dim3((unsigned)chunks, nw), STRIPE_SUB_THREADS, part_smem, s>>>(bucket, boff, pos_lg, sub_lg, sboff + nsub + 1,
                                                                                                       sub);
        const size_t sub_smem = ((size_t)4 << sub_lg) + ((size_t)1 << sub_lg) / 8;
        if ((e = cudaFuncSetAttribute(stripe_pos_sub_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sub_smem)) != cudaSuccess) return e;
        if ((e = cudaFuncSetAttribute(stripe_pos_sub_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared)) !=
            cudaSuccess)
            return e;
        stripe_pos_sub_kernel<<<nsub, STRIPE_SUB_THREADS, sub_smem, s>>>(sub, sboff, T_all, sub_lg, js->pos, js->succ);
        count_launches(2);
    }
    if (begin_bit) {
        u32* tmp = (u32*)bucket;
        if (js->tag16)
            stripe_hash_fix_kernel<u16><<<SMB_SMS * 4, 128, 0, s>>>(hs, es, begin_bit, T, worklist, d_count, off, n, tmp, (u16*)js->tags, js->pos,
                                                                    js->swz, js->succ);
        else
            stripe_hash_fix_kernel<u32><<<SMB_SMS * 4, 128, 0, s>>>(hs, es, begin_bit, T, worklist, d_count, off, n, tmp, (u32*)js->tags, js->pos,
                                                                    js->swz, js->succ);
        count_launches(1);
    }
    if ((e = stripe_make_order(js, scratch, s)) != cudaSuccess) return e;
    *out = guard.release();
    return cudaSuccess;
}
cudaError_t join_stripe_create(const u64* h, const u64* off, int n, u64 T, u64 max_key, JoinStripe** out, cudaStream_t s) {
    return join_stripe_create_shard(h, off, n, T, max_key, 0, 1, out, s);
}

static cudaError_t stripe_launch(const JoinStripe* js, int row_begin, int row_end, double* d_out, u32* d_counts, u16* d_counts16,
                                 cudaStream_t s) {
    if (row_end <= row_begin) return cudaSuccess;
    const u32* rows = js->order;                                    // the whole set: the order itself
    if (row_end - row_begin < js->n) {
        rows = js->sel + row_begin;                                 // the callers' ranges do not overlap, so no launch
                                                                    // overwrites the rows of one still in flight
        stripe_select_rows_kernel<<<1, 1024, 0, s>>>(js->order, js->n, row_begin, row_end, js->sel + row_begin);
        count_launches(1);
    }
    StripeArgs a{js->tags, js->pos, js->ebeg, js->eend, js->sizes, js->T, js->n, js->rows_per_block, row_begin, row_end, d_out,
                 d_counts, d_counts16, js->swz, rows, js->succ};
    const int blocks = (row_end - row_begin + js->rows_per_block - 1) / js->rows_per_block;
    const bool upper = js->upper_only;
    const bool two = js->ctas_per_sm == 2;
#define SMB_STRIPE_LAUNCH(TAG, UP, C) join_stripe_kernel<TAG, UP, C><<<blocks, 1024, js->smem, s>>>(a)
    if (js->tag16) {
        if (upper) { if (two) SMB_STRIPE_LAUNCH(u16, true, 2); else SMB_STRIPE_LAUNCH(u16, true, 1); }
        else { if (two) SMB_STRIPE_LAUNCH(u16, false, 2); else SMB_STRIPE_LAUNCH(u16, false, 1); }
    } else {
        if (upper) { if (two) SMB_STRIPE_LAUNCH(u32, true, 2); else SMB_STRIPE_LAUNCH(u32, true, 1); }
        else { if (two) SMB_STRIPE_LAUNCH(u32, false, 2); else SMB_STRIPE_LAUNCH(u32, false, 1); }
    }
#undef SMB_STRIPE_LAUNCH
    count_launches(1);
    return cudaGetLastError();
}
// raw counters of ALL rows (n x n, whole rows): the partial counts of a key-range shard.  Counted for the cells
// (i, j > i) only and mirrored -- the counts of one key range are symmetric like the total -- unless SMB_JOIN_LAYOUT=stripe_full.
cudaError_t join_stripe_counts(const JoinStripe* js, void* d_counts, int bits, cudaStream_t s) {
    cudaError_t e = bits == 16 ? stripe_launch(js, 0, js->n, nullptr, nullptr, (u16*)d_counts, s)
                               : stripe_launch(js, 0, js->n, nullptr, (u32*)d_counts, nullptr, s);
    if (e != cudaSuccess) return e;
    if (js->upper_only) launch_mirror_counts(d_counts, bits, js->n, s);
    return cudaGetLastError();
}
// counters of rows [row_begin, row_end) summed over the shards -> float64 Jaccard rows
void launch_finalize_counts_rows(const void* d_counts, int bits, const u64* off, int n, int row_begin, int row_end, double* d_out,
                                 cudaStream_t s) {
    if (row_end <= row_begin || n <= 0) return;
    dim3 grid((n + 255) / 256, row_end - row_begin);
    if (bits == 16) stripe_finalize_counts_kernel<u16><<<grid, 256, 0, s>>>((const u16*)d_counts, off, n, row_begin, row_end, d_out);
    else stripe_finalize_counts_kernel<u32><<<grid, 256, 0, s>>>((const u32*)d_counts, off, n, row_begin, row_end, d_out);
    count_launches(1);
}
// c[j][i] = c[i][j] for j > i: upper-triangle counters completed to whole rows
void launch_mirror_counts(void* d_counts, int bits, int n, cudaStream_t s) {
    if (n <= 0) return;
    const int t = (n + STRIPE_MIRROR_TILE - 1) / STRIPE_MIRROR_TILE;
    if (bits == 16) stripe_mirror_kernel<u16><<<dim3((unsigned)t, (unsigned)t), 1024, 0, s>>>((u16*)d_counts, n, 0, n);
    else stripe_mirror_kernel<u32><<<dim3((unsigned)t, (unsigned)t), 1024, 0, s>>>((u32*)d_counts, n, 0, n);
    count_launches(1);
}
void launch_narrow_counts(const u32* in, u64 total, u16* out, cudaStream_t s) {
    if (!total) return;
    stripe_narrow_counts_kernel<<<(unsigned)std::min<u64>((total + 255) / 256, (u64)SMB_SMS * 32), 256, 0, s>>>(in, total, out);
    count_launches(1);
}

// float64 Jaccard rows [row_begin, row_end) of the all-vs-all matrix into d_out (row_begin first)
cudaError_t join_stripe_rows(const JoinStripe* js, const u64* off, int row_begin, int row_end, double* d_out,
                             cudaStream_t s) {
    (void)off;
    return stripe_launch(js, row_begin, row_end, d_out, nullptr, nullptr, s);
}
// upper-only mode: the cells (i, j < i) of rows [row_begin, row_end) from the finished upper parts of rows
// < row_end; d_full = row 0 of the whole n x n matrix.  No-op in the two-direction mode.
cudaError_t join_stripe_mirror(const JoinStripe* js, int row_begin, int row_end, double* d_full, cudaStream_t s) {
    if (!js->upper_only || row_end <= row_begin) return cudaSuccess;
    const int t0 = row_begin / STRIPE_MIRROR_TILE, t1 = (row_end + STRIPE_MIRROR_TILE - 1) / STRIPE_MIRROR_TILE;
    dim3 grid((unsigned)t1, (unsigned)(t1 - t0));
    stripe_mirror_kernel<double><<<grid, 1024, 0, s>>>(d_full, js->n, row_begin, row_end); count_launches(1);
    return cudaGetLastError();
}
bool join_stripe_upper_only(const JoinStripe* js) { return js->upper_only != 0; }
void join_stripe_two_directions(JoinStripe* js) { js->upper_only = 0; }
void join_stripe_destroy(JoinStripe* js) { delete js; }
bool join_stripe_enabled() {
    const char* layout = getenv("SMB_JOIN_LAYOUT");
    return !(layout && !strcmp(layout, "plain"));
}

// ------------------------------------------------------------------------------------
// Inverted index over a resident set (db_index.cuh): built on request, then one-vs-many counts cost
// one directory probe per query hash and one increment per match instead of a pass over the set.
// Logic checked on the CPU by tests/test_host_emulation.py::test_db_index_*; not measured yet.
// ------------------------------------------------------------------------------------
// run lengths -> start offsets: start[u] = sum of counts[0..u); done in place by an exclusive scan
struct DbIndex {
    cudaStream_t stream = 0;
    void *m_keys = nullptr, *m_start = nullptr, *m_rows = nullptr, *m_dir = nullptr;
    DbIndexView view{};
    u64 n_elements = 0;
    ~DbIndex() {
        if (m_keys) cudaFreeAsync(m_keys, stream);
        if (m_start) cudaFreeAsync(m_start, stream);
        if (m_rows) cudaFreeAsync(m_rows, stream);
        if (m_dir) cudaFreeAsync(m_dir, stream);
    }
};

// (hash, payload) pairs stably sorted by hash over the significant bits of max_key: equal hashes keep the order of
// their payloads.  The payload is the caller's: row ids for the index, element indices for sketchset_combine.
static cudaError_t sort_hash_pairs(const u64* h, u64* keys_out, const u32* payload, u32* payload_out, u64 T,
                                   u64 max_key, cudaStream_t s) {
    const int key_bits = key_bit_length(max_key);
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, h, keys_out, payload, payload_out, (long long)T, 0, key_bits, s);
    void* tmp = nullptr;
    cudaError_t e = cudaMallocAsync(&tmp, bytes ? bytes : 16, s);
    if (e != cudaSuccess) return e;
    cub::DeviceRadixSort::SortPairs(tmp, bytes, h, keys_out, payload, payload_out, (long long)T, 0, key_bits, s);
    cudaFreeAsync(tmp, s);
    count_launches(1);
    return cudaGetLastError();
}

cudaError_t db_index_build(const u64* h, const u64* off, int n, u64 T, u64 max_key, DbIndex** out, cudaStream_t s) {
    *out = nullptr;
    if (n <= 0 || T == 0 || T > 0x7fffffffull) return cudaSuccess;       // CUB's run-length encode counts in int
    auto ix = new DbIndex();
    ix->stream = s; ix->n_elements = T;
    std::unique_ptr<DbIndex> guard(ix);
    cudaError_t e;
    JoinScratch scratch(s);
    u64* keys_sorted = nullptr;
    u32* ids = nullptr;
    if ((e = scratch.alloc((void**)&keys_sorted, T * sizeof(u64))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&ids, T * sizeof(u32))) != cudaSuccess) return e;
    if ((e = cudaMallocAsync(&ix->m_rows, T * sizeof(u32), s)) != cudaSuccess) return e;
    const int blocks = n < SMB_SMS * 16 ? n : SMB_SMS * 16;
    index_rowid_kernel<<<blocks, 256, 0, s>>>(off, n, ids); count_launches(1);
    // (hash, row) pairs sorted by hash; stable, so rows ascend inside a group
    if ((e = sort_hash_pairs(h, keys_sorted, ids, (u32*)ix->m_rows, T, max_key, s)) != cudaSuccess) return e;
    // distinct keys + group sizes, then sizes -> offsets
    if ((e = cudaMallocAsync(&ix->m_keys, T * sizeof(u64), s)) != cudaSuccess) return e;
    if ((e = cudaMallocAsync(&ix->m_start, (T + 1) * sizeof(u32), s)) != cudaSuccess) return e;
    u64* d_runs = (u64*)ids;                                               // ids is free again: reuse 8 bytes of it
    {
        size_t bytes = 0;
        cub::DeviceRunLengthEncode::Encode(nullptr, bytes, keys_sorted, (u64*)ix->m_keys, (u32*)ix->m_start, d_runs, (int)T, s);
        void* tmp = nullptr;
        if ((e = cudaMallocAsync(&tmp, bytes ? bytes : 16, s)) != cudaSuccess) return e;
        cub::DeviceRunLengthEncode::Encode(tmp, bytes, keys_sorted, (u64*)ix->m_keys, (u32*)ix->m_start, d_runs, (int)T, s);
        cudaFreeAsync(tmp, s);
        count_launches(1);
    }
    u64 n_keys = 0;
    cudaMemcpyAsync(&n_keys, d_runs, sizeof(u64), cudaMemcpyDeviceToHost, s);
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
    {
        size_t bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, bytes, (u32*)ix->m_start, (u32*)ix->m_start, (int)(n_keys + 1), s);
        void* tmp = nullptr;
        if ((e = cudaMallocAsync(&tmp, bytes ? bytes : 16, s)) != cudaSuccess) return e;
        // element n_keys is scratch: whatever it holds, the exclusive sum puts the total (= T) there
        cub::DeviceScan::ExclusiveSum(tmp, bytes, (u32*)ix->m_start, (u32*)ix->m_start, (int)(n_keys + 1), s);
        cudaFreeAsync(tmp, s);
        count_launches(1);
    }
    u32 shift;
    u64 nbk;
    db_index_dir_plan(n_keys, max_key, shift, nbk);
    if ((e = cudaMallocAsync(&ix->m_dir, (nbk + 2) * sizeof(u32), s)) != cudaSuccess) return e;
    launch_build_global_dir((const u64*)ix->m_keys, n_keys, (int)shift, nbk, (u32*)ix->m_dir, s);
    ix->view = DbIndexView{(const u64*)ix->m_keys, n_keys, (const u32*)ix->m_start, (const u32*)ix->m_rows,
                           (const u32*)ix->m_dir, shift, nbk};
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    *out = guard.release();
    return cudaSuccess;
}
void db_index_destroy(DbIndex* ix) { delete ix; }
u64 db_index_n_keys(const DbIndex* ix) { return ix->view.n_keys; }

// ------------------------------------------------------------------------------------
// Union / intersection / difference of all rows of a resident set (sketch_combine.cuh): a stable sort of
// (hash, element index), one pass over the runs, a scan and a scatter -- five launches and one readback (the output
// length) whatever the number of rows.
// ------------------------------------------------------------------------------------
cudaError_t sketchset_combine(const u64* h, const u64* abund, u64 n_rows, u64 T, u64 row0_end, u64 max_key, u32 op,
                              u64** out_h, u64** out_v, u64* out_n, cudaStream_t s) {
    *out_h = *out_v = nullptr;
    *out_n = 0;
    if (n_rows == 0 || T == 0) return cudaSuccess;
    if (T > 0x7fffffffull) return cudaErrorInvalidValue;              // cub's scan counts in int
    const bool values = abund && op == COMBINE_UNION;
    JoinScratch scratch(s);
    cudaError_t e;
    u32 *idx = nullptr, *idx_sorted = nullptr, *flag = nullptr, *pos = nullptr;
    u64 *keys = nullptr, *val = nullptr;
    unsigned long long* d_count = nullptr;
    if ((e = scratch.alloc((void**)&idx, T * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&idx_sorted, T * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&keys, T * sizeof(u64))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&flag, T * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&pos, T * sizeof(u32))) != cudaSuccess) return e;
    if ((e = scratch.alloc((void**)&d_count, sizeof(unsigned long long))) != cudaSuccess) return e;
    if (values && (e = scratch.alloc((void**)&val, T * sizeof(u64))) != cudaSuccess) return e;
    const unsigned blocks = (unsigned)std::min<u64>((T + 255) / 256, (u64)SMB_SMS * 32);
    combine_iota_kernel<<<blocks, 256, 0, s>>>(idx, T); count_launches(1);
    if ((e = sort_hash_pairs(h, keys, idx, idx_sorted, T, max_key, s)) != cudaSuccess) return e;
    combine_runs_kernel<<<blocks, 256, 0, s>>>(keys, idx_sorted, T, values ? abund : nullptr, op, n_rows, row0_end,
                                               flag, val);
    count_launches(1);
    {
        size_t bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, bytes, flag, pos, (int)T, s);
        void* tmp = nullptr;
        if ((e = cudaMallocAsync(&tmp, bytes ? bytes : 16, s)) != cudaSuccess) return e;
        cub::DeviceScan::ExclusiveSum(tmp, bytes, flag, pos, (int)T, s);
        cudaFreeAsync(tmp, s);
        count_launches(1);
    }
    // the output is at most T long: allocated at that bound, so the one readback is the length itself
    u64 *oh = nullptr, *ov = nullptr;
    if ((e = cudaMallocAsync((void**)&oh, T * sizeof(u64), s)) != cudaSuccess) return e;
    if (values && (e = cudaMallocAsync((void**)&ov, T * sizeof(u64), s)) != cudaSuccess) { cudaFreeAsync(oh, s); return e; }
    combine_scatter_kernel<<<blocks, 256, 0, s>>>(keys, val, flag, pos, T, oh, ov, d_count); count_launches(1);
    unsigned long long n = 0;
    cudaMemcpyAsync(&n, d_count, sizeof n, cudaMemcpyDeviceToHost, s);
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
        cudaFreeAsync(oh, s);
        if (ov) cudaFreeAsync(ov, s);
        return e;
    }
    *out_h = oh; *out_v = ov; *out_n = n;
    return cudaSuccess;
}

// ------------------------------------------------------------------------------------
// One abundance query against every row of a set with abundances (angular_search.cuh): with the global directory's
// three builder launches and the bitmap, at most five launches whatever the number of rows; no readback.
// ------------------------------------------------------------------------------------
cudaError_t angular_search(AngularSearchArgs a, cudaStream_t s) {
    if (a.n_rows <= 0) return cudaSuccess;
    cudaError_t e;
    if ((e = cudaMemsetAsync(a.prod, 0, (size_t)a.n_rows * sizeof(unsigned long long), s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(a.bsq, 0, (size_t)a.n_rows * sizeof(unsigned long long), s)) != cudaSuccess) return e;
    if (a.n_chunks == 0) return cudaSuccess;
    JoinScratch scratch(s);
    a.split = a.nq <= ANGULAR_SPLIT_MAX ? 1 : 0;
    if (a.split) {
        const u64 entries = a.nq > 256 ? a.nq : 256;                     // about one key per bucket
        u32 sh = 0;
        while (sh < 63 && (a.q_top >> sh) >= entries) ++sh;
        a.shift = sh; a.nb = (a.q_top >> sh) + 1;
    } else {
        int nb_log2 = 12;                                                // as one_vs_many_dev
        while (nb_log2 < 26 && (1ull << nb_log2) < 2 * a.nq) ++nb_log2;
        u32 sh = 0;
        while (sh < 63 && (a.q_top >> sh) >= (1ull << nb_log2)) ++sh;
        a.shift = sh; a.nb = (a.q_top >> sh) + 1;
        a.fine_log2 = 3;
        u32 *dir = nullptr, *bm = nullptr;
        const size_t bm_words = ((size_t)a.nb << a.fine_log2) / 32 + 2;
        if ((e = scratch.alloc((void**)&dir, (a.nb + 2) * sizeof(u32))) != cudaSuccess) return e;
        if ((e = scratch.alloc((void**)&bm, bm_words * sizeof(u32))) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(bm, 0, bm_words * sizeof(u32), s)) != cudaSuccess) return e;
        launch_build_global_dir(a.q, a.nq, (int)sh, a.nb, dir, s);
        launch_build_query_bitmap(a.q, a.nq, (int)sh, a.fine_log2, bm, s);
        a.gdir = dir; a.bitmap = bm;
    }
    const size_t smem = a.split ? angular_split_smem(a.nq, a.nb) : 0;
    cudaFuncSetAttribute(angular_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const u64 ctas_per_sm = smem + 1024 <= (size_t)110 * 1024 ? 2 : 1;   // two CTAs of 512 threads fill an SM
    u64 blocks = (a.n_chunks + ANGULAR_THREADS / 32 - 1) / (ANGULAR_THREADS / 32);   // one chunk per warp at most
    if (blocks > (u64)SMB_SMS * ctas_per_sm) blocks = (u64)SMB_SMS * ctas_per_sm;
    angular_search_kernel<<<(unsigned)blocks, ANGULAR_THREADS, smem, s>>>(a); count_launches(1);
    return cudaGetLastError();
}

void launch_index_count(const DbIndex* ix, const u64* q, u64 nq, u32* counts, cudaStream_t s) {
    if (nq == 0 || ix->view.n_keys == 0) return;
    u64 blocks = (nq + 255) / 256;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    index_count_kernel<<<(unsigned)blocks, 256, 0, s>>>(ix->view, q, nq, nullptr, counts); count_launches(1);
}
// the same with the number of query hashes read from device memory (at most max_nq): no host round trip
void launch_index_count_n(const DbIndex* ix, const u64* q, const u32* d_nq, u64 max_nq, u32* counts, cudaStream_t s) {
    if (max_nq == 0 || ix->view.n_keys == 0) return;
    u64 blocks = (max_nq + 255) / 256;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    index_count_kernel<<<(unsigned)blocks, 256, 0, s>>>(ix->view, q, max_nq, d_nq, counts); count_launches(1);
}

cudaError_t join_counts(const u64* h, const u64* off, int n, u64 max_key, int shard, int n_shards,
                        u32* common, size_t ld, cudaStream_t s) {
    u64 lo, hi;
    bool bounded;
    join_shard_range(max_key, shard, n_shards, lo, hi, bounded);
    JoinWork W;
    cudaError_t e = join_sort_slice(h, off, n, lo, hi, bounded ? 1 : 0, key_bit_length(max_key), W, s);
    W.stream = s;
    if (e != cudaSuccess) return e;
    if (W.T) {
        join_count_kernel<<<(unsigned)((W.T + 255) / 256), 256, 0, s>>>(W.keys_b, W.ids_b, W.T, common, ld);
        count_launches(1);
    }
    return cudaGetLastError();
}

}  // namespace smb

