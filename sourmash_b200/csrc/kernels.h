// kernels.h -- host-callable launchers for the sm_90a kernels (internal C++ interface
// between capi.cu and the .cu kernel files; the public boundary is include/sourmash_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "aa_kmers.cuh"

namespace smb {

// ---------------------------------------------------------------- intersection path
struct PairwisePlan {
    int tables_per_cta;   // TA (1..4); 0 => tile kernel not applicable, use generic kernel
    int shift;            // bucket = key >> shift
    int nb;               // number of buckets = (max_key >> shift) + 1
    int cap;              // key capacity per table
    int cols_per_cta;
    size_t smem_bytes;
};

// Chooses the tile-kernel configuration for table rows of at most max_len_a keys when no key
// of either operand exceeds max_key.
PairwisePlan plan_pairwise(uint64_t max_len_a, uint64_t max_key, int n_b);

// max over the last (largest) key of every row of both CSR sets -> *d_max (zeroed by the caller)
void launch_max_last(const uint64_t* hA, const uint64_t* offA, int nA, const uint64_t* hB,
                     const uint64_t* offB, int nB, unsigned long long* d_max, cudaStream_t s);

// Multi-GPU sharding of row tiles: this launch handles tiles shard, shard + n_shards, ...
struct TileShard { int shard; int n_shards; int count = -1; };   // count >= 0: at most that many tiles

// common[i*ldo + j] = |A_i ∩ B_j| for every (i, j) (symmetric: only j > i, A == B).
// Tile kernel: A rows become shared-memory bucket tables, B rows stream through registers.
void launch_pairwise_tile(const PairwisePlan& plan, const uint64_t* hA, const uint64_t* offA,
                          int nA, const uint64_t* hB, const uint64_t* offB, int nB, uint32_t* out,
                          size_t ldo, bool symmetric, TileShard tiles, cudaStream_t s);

// Inverted index over a resident set (db_index.cuh): hash -> rows.  db_index_build leaves *out null
// when the set is empty or has more than 2^31 - 1 elements.  launch_index_count adds, for every query
// hash, 1 to the counter of every row that holds it (counters zeroed by the caller): the same counts
// as the one-vs-many passes, for work proportional to the query and its matches.
struct DbIndex;
cudaError_t db_index_build(const uint64_t* h, const uint64_t* off, int n, uint64_t n_elements, uint64_t max_key,
                           DbIndex** out, cudaStream_t s);
void db_index_destroy(DbIndex* ix);
uint64_t db_index_n_keys(const DbIndex* ix);
void launch_index_count(const DbIndex* ix, const uint64_t* q, uint64_t nq, uint32_t* counts, cudaStream_t s);
void launch_index_count_n(const DbIndex* ix, const uint64_t* q, const uint32_t* d_nq, uint64_t max_nq, uint32_t* counts,
                          cudaStream_t s);

// Range-major copy of a resident set and the streaming one-vs-many pass over it (range_kernels.cuh): the key
// space is cut into P equal ranges, part p of the copy holds every row's elements of range p back to back, CTA p
// keeps a Bloom bitmap of the query keys of its range in shared memory and streams its part.  range_major_build
// leaves *out null when the layout does not apply (the caller uses the global-directory kernel).
struct RangeMajor;
bool range_search_enabled();                          // false with SMB_SEARCH_LAYOUT=global
cudaError_t range_major_build(const uint64_t* h, const uint64_t* off, int n, uint64_t n_elements, uint64_t max_key,
                              RangeMajor** out, cudaStream_t s);
void range_major_destroy(RangeMajor* rm);
void launch_one_vs_many_range_major(const RangeMajor* rm, const uint64_t* q, uint64_t nq, uint32_t* out, cudaStream_t s);
// The same pass for a group of G queries, the database read once: q holds their keys back to back (d_qoff: G + 1
// offsets from 0, on the device), out the G x n counters (query-major, zeroed by the caller).  The keys are merged by
// a radix sort into one stream with the query ids alongside.  *unsorted is set, and nothing counted, when a query is
// not sorted and unique.  range_major_group_keys bounds n_keys (the per-range bitmaps stay sparse).
uint64_t range_major_group_keys(const RangeMajor* rm);
cudaError_t many_vs_many_range_major(const RangeMajor* rm, const uint64_t* q, const uint64_t* d_qoff, int G, uint64_t n_keys,
                                     uint32_t* out, bool* unsorted, cudaStream_t s);
// stat[0] = max key, stat[1] > 0 iff a query of the CSR is not sorted and unique (ids: null, or the query of every key)
void launch_query_stats(const uint64_t* q, const uint64_t* d_qoff, int G, uint32_t* ids, unsigned long long* d_stat,
                        cudaStream_t s);

// All-vs-all counts by inverted join (compare_kernels.cu): sort the (hash, row) pairs of the set,
// one increment per pair of rows sharing a hash.  join_estimate sorts the lowest 1/JOIN_SAMPLE of
// the key range and extrapolates the number of increments / elements (d_out2: 2 x u64 scratch);
// join_counts adds the counts of key range `shard` of `n_shards` into the zeroed upper triangle.
static constexpr unsigned long long JOIN_SAMPLE = 64;
cudaError_t join_estimate(const uint64_t* h, const uint64_t* off, int n, uint64_t max_key,
                          unsigned long long* d_out2, double* est_increments, double* est_elements,
                          unsigned long long* max_group, cudaStream_t s);
cudaError_t join_counts(const uint64_t* h, const uint64_t* off, int n, uint64_t max_key, int shard,
                        int n_shards, uint32_t* common, size_t ld, cudaStream_t s);

// Stripe layout of the join (join_stripe.cuh; the default, SMB_JOIN_LAYOUT=plain switches it off): CTAs own
// complete rows of the result in shared memory and write float64 Jaccard rows directly.
// join_stripe_create leaves *out null when the layout does not apply (caller uses join_counts).
struct JoinStripe;
bool join_stripe_enabled();
cudaError_t join_stripe_create(const uint64_t* h, const uint64_t* off, int n, uint64_t n_elements, uint64_t max_key,
                               JoinStripe** out, cudaStream_t s);
// n_shards > 1: the stream of key range `shard` only; join_stripe_counts then writes the shard's partial counters of
// whole rows (u32, both directions), which add up over the shards; launch_finalize_counts_rows turns summed counters
// of a block of rows into float64 Jaccard rows; launch_mirror_counts completes upper-triangle counters to whole rows.
cudaError_t join_stripe_create_shard(const uint64_t* h, const uint64_t* off, int n, uint64_t n_elements, uint64_t max_key,
                                     int shard, int n_shards, JoinStripe** out, cudaStream_t s);
void launch_mirror_counts(void* d_counts, int bits, int n, cudaStream_t s);          // bits: 32 or 16 (counter width)
void launch_narrow_counts(const uint32_t* in, uint64_t total, uint16_t* out, cudaStream_t s);
cudaError_t join_stripe_counts(const JoinStripe* js, void* d_counts, int bits, cudaStream_t s);
void launch_finalize_counts_rows(const void* d_counts, int bits, const uint64_t* off, int n, int row_begin, int row_end,
                                 double* d_out, cudaStream_t s);
cudaError_t join_stripe_rows(const JoinStripe* js, const uint64_t* off, int row_begin, int row_end, double* d_out,
                             cudaStream_t s);
// join_stripe_rows counts / writes only the cells (i, j >= i); join_stripe_mirror then fills (i, j < i) of rows
// [row_begin, row_end) from the rows above (d_full = row 0 of the n x n matrix).  A block of rows computed on
// its own (smb_compare_jaccard_rows_dev) -- and SMB_JOIN_LAYOUT=stripe_full -- use the two-direction mode.
cudaError_t join_stripe_mirror(const JoinStripe* js, int row_begin, int row_end, double* d_full, cudaStream_t s);
bool join_stripe_upper_only(const JoinStripe* js);
void join_stripe_two_directions(JoinStripe* js);
void join_stripe_destroy(JoinStripe* js);

// Fallback for arbitrary row sizes: one warp per pair, binary search of the shorter row's
// elements in the longer row.
void launch_pairwise_generic(const uint64_t* hA, const uint64_t* offA, int nA, const uint64_t* hB,
                             const uint64_t* offB, int nB, uint32_t* out, size_t ldo,
                             bool symmetric, TileShard tiles, cudaStream_t s);

// Bottom-k ("num") sketches: common = |A ∩ B ∩ M|, usize = |M|, M = first `num` of A ∪ B.
void launch_pairwise_num(const uint64_t* hA, const uint64_t* offA, int nA, const uint64_t* hB,
                         const uint64_t* offB, int nB, uint32_t num, uint32_t* common,
                         uint32_t* usize, size_t ldo, bool symmetric, cudaStream_t s);

// counts -> float64 matrix.  mode: 0 jaccard (scaled), 1 jaccard (num; needs usize),
// 2 raw containment c/|col j| written at [i][j] (no bias correction; host applies it).
void launch_finalize_matrix(const uint32_t* common, const uint32_t* usize, size_t ldo,
                            const uint64_t* offA, const uint64_t* offB, int nA, int nB, int mode,
                            bool symmetric, double* out, cudaStream_t s);

// all-vs-all angular similarity of abundance sketches (symmetric f64 matrix, ones on the diagonal)
void launch_pairwise_angular(const uint64_t* h, const uint64_t* ab, const uint64_t* off, int n,
                             unsigned long long* d_sumsq, double* out, cudaStream_t s);

// rows [row_begin, row_end) of the symmetric jaccard matrix from upper-triangular counts
void launch_finalize_rows(const uint32_t* common, size_t n, const uint64_t* off, int n_rows,
                          int row_begin, int row_end, double* out, cudaStream_t s);

// One query vs many subjects with a query too large for shared memory: global-memory bucket
// directory over the query (dir has nb+1 u32 entries), every subject element probes it.
void launch_build_global_dir(const uint64_t* q, uint64_t nq, int shift, uint64_t nb, uint32_t* dir,
                             cudaStream_t s);
// bitmap (nullable, zeroed by the caller, (nb << fine_log2) bits): occupancy of the query at
// 2^fine_log2 times the directory's resolution, bit index = key >> max(shift - fine_log2, 0)
void launch_build_query_bitmap(const uint64_t* q, uint64_t nq, int shift, int fine_log2,
                               uint32_t* bitmap, cudaStream_t s);
void launch_one_vs_many_global(const uint64_t* q, uint64_t nq, const uint32_t* dir, int shift,
                               uint64_t nb, const uint32_t* bitmap, int fine_log2, const uint64_t* hB,
                               const uint64_t* offB, int nB, uint32_t* out, cudaStream_t s);

// gather: query fixed in HBM + per-hash alive flags.  intersect_alive: hashes of `row` that are in q
// and alive (sorted, count in *d_n); mark_dead: clear the flags of the given hashes.
void launch_intersect_alive(const uint64_t* q, uint64_t nq, const uint8_t* alive, const uint64_t* row,
                            uint64_t rn, uint64_t* out, uint32_t* d_n, cudaStream_t s);
void launch_mark_dead(const uint64_t* q, uint64_t nq, uint8_t* alive, const uint64_t* gone, uint64_t n,
                      cudaStream_t s);

// device-side glue for the sync-free gather round: offsets {0, *d_n} of a 1-row CSR, and
// mark_dead with the count read from the device
void launch_make_row_offsets(const uint32_t* d_n, uint64_t* d_off2, cudaStream_t s);
// gather rounds picked on the device (search_kernels.cuh): the argmax appends (row, count) to the pick list and raises
// `done` below the threshold; the intersect kernel takes its row from the last pick
#ifndef SMB_GATHER_PICKS_DEFINED
#define SMB_GATHER_PICKS_DEFINED
struct GatherPicks { uint32_t* rows; uint32_t* sizes; uint32_t* state; uint32_t threshold, max_rounds; };
#endif
void launch_counter_update_argmax_pick(uint32_t* counters, const uint32_t* delta, int n, const GatherPicks& g, cudaStream_t s);
void launch_intersect_alive_pick(const uint64_t* q, uint64_t nq, uint8_t* alive, const uint64_t* hashes,
                                 const uint64_t* off, const GatherPicks& g, uint64_t* out, uint32_t* d_n, cudaStream_t s);
void launch_mark_dead_n(const uint64_t* q, uint64_t nq, uint8_t* alive, const uint64_t* gone,
                        const uint32_t* d_n, cudaStream_t s);

// gather rounds of many queries at once (multigather_kernels.cuh): per-query state in segments, three launches per round
// for all queries.  The decrement launch runs cta_total CTAs with smem_bytes of dynamic shared memory (one split table
// of kstride keys and nb + 2 directory entries).
#ifndef SMB_MULTI_GATHER_ARGS_DEFINED
#define SMB_MULTI_GATHER_ARGS_DEFINED
struct MultiGatherArgs {
    const uint64_t* q_hashes;
    const uint64_t* q_begin;   const uint64_t* q_end;
    const uint32_t* cand_rows; const uint64_t* cand_off;
    uint32_t* counts;          uint32_t* delta;
    const uint64_t* pick_off;  uint32_t* pick_rows; uint32_t* pick_sizes;
    uint32_t* state;
    uint32_t* live;
    const uint32_t* threshold;
    uint32_t* consumed;
    uint64_t* isect;           const uint64_t* isect_off;
    uint32_t* isect_n;
    const uint64_t* db_hashes; const uint64_t* db_off;
    const uint32_t* cta_start;
    int n_queries, cols_per_cta, shift, nb, kstride;
};
#endif
void launch_multi_gather_round(const MultiGatherArgs& a, uint32_t cta_total, size_t smem_bytes, cudaStream_t s);

// Materialise A ∩ B of two sorted rows (gather's intersect_mh); returns count in *d_n.
void launch_intersect_rows(const uint64_t* a, uint64_t na, const uint64_t* b, uint64_t nb,
                           uint64_t* out, uint32_t* d_n, cudaStream_t s);
// out = a \ b (sorted rows), count in *d_n  (gather's query.remove_many(found)).
void launch_subtract_rows(const uint64_t* a, uint64_t na, const uint64_t* b, uint64_t nb,
                          uint64_t* out, uint32_t* d_n, cudaStream_t s);
// counters[j] -= delta[j]; then (best value, lowest index) of counters -> d_best[0..1].
void launch_counter_update_argmax(uint32_t* counters, const uint32_t* delta, int n,
                                  unsigned long long* d_best, cudaStream_t s);

// ---------------------------------------------------------------- sketch path
// Streams are byte sequences inside one 16-byte aligned HBM allocation that is readable up to
// the next 16-byte boundary past its end.  Any non-ACGT byte inside a stream (record separator,
// N, ...) invalidates the windows covering it.  Output row = stream * row_stride + row_index.
struct HashLaunch {
    const uint8_t* bases;
    const uint64_t* stream_off;          // device [n_streams] byte offsets (any alignment)
    const uint64_t* stream_len;          // device [n_streams]
    const uint32_t* stream_row;          // device [n_streams] sketch fed by each stream (NULL: identity)
    int n_streams;
    const uint32_t* tile_start_rolled;   // device [n_streams+1] prefix of ceil((off%16+len)/(threads*W))
    uint32_t total_tiles_rolled;
    const uint32_t* tile_start_generic;  // device [n_streams+1] prefix of ceil(len/256)
    uint32_t total_tiles_generic;
    int W;                               // windows per thread, multiple of 16
    uint64_t seed, max_hash;
    uint64_t* cand;                      // candidate storage
    const uint64_t* cand_off;            // device [n_rows+1]
    uint32_t* cand_cnt;                  // device [n_rows] (zeroed by caller)
    int row_stride;
};
bool k_has_rolled_kernel(uint32_t k);
int hash_threads();
// survivors (0 < h <= max_hash, all k bases valid) of every window -> candidate rows
void launch_hash_kmers_k(const HashLaunch& L, uint32_t ksize, int row_index, cudaStream_t s);
// same, restricted to a range of tiles (a group of streams) -- lets uploads and hashing overlap
void launch_hash_kmers_range(const HashLaunch& L, uint32_t ksize, int row_index, uint32_t tile_lo_r,
                             uint32_t tile_hi_r, uint32_t tile_lo_g, uint32_t tile_hi_g, cudaStream_t s);
// Default when k = 21, 31 and 51 are requested together (SMB_SKETCH_FUSED=0 switches it off): one pass over the bases (one rolling
// 51-state, the shorter k-mers as prefixes); row_index[i] / max_hash[i] belong to k = 21, 31, 51
bool sketch_fused_enabled();
void launch_hash_kmers_fused_range(const HashLaunch& L, const int row_index[3], const uint64_t max_hash[3],
                                   uint32_t tile_lo, uint32_t tile_hi, cudaStream_t s);
// per-window hashes of stream 0 in order; 0 marks an invalid window (seq_to_hashes)
void launch_window_hashes(const HashLaunch& L, uint32_t ksize, uint64_t* raw_out, cudaStream_t s);
// protein-family sketches (aa_kmers.cuh): windows of kaa residues, read as they are
// (translate == false; streams hold residues) or from DNA translated in six frames (two hashes per
// window of 3*kaa bases).  Uses the generic (256 positions per CTA) tiling of HashLaunch.
uint32_t aa_max_k(bool translate);
void launch_hash_aa_range(const HashLaunch& L, const AaTables* d_tables, uint32_t kaa, bool translate,
                          int row_index, uint32_t tile_lo, uint32_t tile_hi, cudaStream_t s);
// per-window hashes of stream 0 (length len) in the reference's seq_to_hashes order
void launch_aa_window_hashes(const HashLaunch& L, const AaTables* d_tables, uint32_t kaa, bool translate,
                             uint64_t len, uint64_t* raw_out, cudaStream_t s);
// first non-ACGT position of a sequence (UINT64_MAX if none)
void launch_first_invalid(const uint8_t* bases, uint64_t len, unsigned long long* d_pos,
                          cudaStream_t s);
// murmur3 of an arbitrary byte string (hash_murmur / add_word)
void launch_murmur_bytes(const uint8_t* data, uint64_t len, uint64_t seed, uint64_t* d_out,
                         cudaStream_t s);

// rows with <= sort_small_max() candidates: block bitonic sort + unique (+ run lengths) in place
int sort_small_max();
void launch_sort_unique_small(uint64_t* cand, const uint64_t* cand_off, const uint32_t* cand_cnt,
                              int n_rows, uint32_t* out_cnt, uint64_t* abund, cudaStream_t s);
// bigger rows: CUB radix sort + unique; scratch_sorted / scratch_heads hold n u64 each
cudaError_t sort_unique_big_row(uint64_t* row, uint64_t n, uint64_t* scratch_sorted,
                                uint64_t* scratch_heads, uint64_t* abund_row, uint32_t* d_out_cnt,
                                cudaStream_t s);
void launch_compact_rows(const uint64_t* src, const uint64_t* src_off, const uint32_t* cnt,
                         const uint64_t* dst_off, uint64_t* dst, int n_rows, cudaStream_t s);
// angular similarity terms (minhash.rs:635-680): out[0] = sum a_i*b_j over common hashes,
// out[1] = sum a_i^2, out[2] = sum b_j^2
void launch_angular_terms(const uint64_t* a, const uint64_t* aa, uint64_t na, const uint64_t* b,
                          const uint64_t* ba, uint64_t nb, unsigned long long* d_out,
                          cudaStream_t s);
// per row: number of hashes <= max_hash (downsample_scaled == prefix of the sorted row)
void launch_row_prefix_counts(const uint64_t* h, const uint64_t* off, int n_rows,
                              uint64_t max_hash, uint32_t* out_cnt, cudaStream_t s);

// kernel-launch accounting (smb_kernel_launches)
void count_launches(int n);

}  // namespace smb
