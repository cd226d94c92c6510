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

// Union / intersection / difference of all n_rows rows of a resident set (sketch_combine.cuh), in hash order.
// UNION keeps every hash (with abund: the sum of its abundances in *out_v), ALL the hashes of every row, FIRST_ONLY
// the hashes of row 0 (elements [0, row0_end)) that no other row holds.  *out_h / *out_v are device arrays the
// caller frees with cudaFreeAsync (*out_v only for UNION with abund).  cudaErrorInvalidValue: more than 2^31 - 1
// elements (cub's scan counts in int).
enum : uint32_t { COMBINE_UNION = 0, COMBINE_ALL = 1, COMBINE_FIRST_ONLY = 2 };
cudaError_t sketchset_combine(const uint64_t* h, const uint64_t* abund, uint64_t n_rows, uint64_t T, uint64_t row0_end,
                              uint64_t max_key, uint32_t op, uint64_t** out_h, uint64_t** out_v, uint64_t* out_n,
                              cudaStream_t s);

// Taxonomic LCA table and per-query LCA counts (lca_kernels.cuh).  The trie is parent[] / depth[] over n_nodes nodes,
// node 0 the root, parent[i] < i.  lca_table_build: the n (hash, node) pairs of every database (LCA_NO_NODE: the
// pair contributes nothing), sorted by hash, every run of equal hashes <= max_hash folded into its LCA node; *out_h
// (sorted, distinct) and *out_lca are device arrays of *out_n entries the caller frees with cudaFreeAsync.
// lca_counts: for the CSR of n_q queries (Tq elements), every distinct (query, LCA node) of the hashes the table
// holds, with the summed weights (abund[e], or 1 per element without abund) and the smallest element position in the
// query; rows ordered by (query, node), in device arrays of *out_n entries freed by the caller.  Both refuse more than
// 2^31 - 1 elements with cudaErrorInvalidValue (cub's scan counts in int).
constexpr uint32_t LCA_NO_NODE = 0xffffffffu;
cudaError_t lca_table_build(const uint64_t* h, const uint32_t* nodes, uint64_t n, uint64_t max_hash, uint64_t max_key,
                            const uint32_t* parent, const uint8_t* depth, uint64_t** out_h, uint32_t** out_lca,
                            uint64_t* out_n, cudaStream_t s);
cudaError_t lca_counts(const uint64_t* t_h, const uint32_t* t_lca, uint64_t n_t, const uint64_t* qh,
                       const uint64_t* q_off, uint32_t n_q, uint64_t Tq, const uint64_t* abund, uint32_t** out_q,
                       uint32_t** out_node, uint64_t** out_w, uint64_t** out_first, uint64_t* out_n, cudaStream_t s);

// The LCA database build (`lca index`, lca_kernels.cuh) over a resident set of n_rows rows (row r is idx r) and T
// elements.  Device arrays, freed by the caller with cudaFreeAsync: hash[K] the distinct hashes in the reference's key
// order (first insertion), koff[K + 1] each key's first element, idx[T] the idx of the elements in key order
// (ascending within a key), key_of[T] each element's key, at[T + 1] each element's first byte in the JSON text of
// "hashval_to_idx" without its braces (at[T]: the text's size).  More than 2^31 - 2 elements: cudaErrorInvalidValue.
// lca_index_plan: from key k0, the longest key range of at most max_bytes, braces included (at least one key):
// plan = {k1, bytes without braces, first element, end element}.  lca_index_text: the text of elements [d0, d1),
// whole keys, into device memory.
struct LcaIndexDev {
    uint64_t* hash = nullptr;
    uint32_t* koff = nullptr;
    uint32_t* idx = nullptr;
    uint32_t* key_of = nullptr;
    uint64_t* at = nullptr;
    uint64_t K = 0, T = 0;
};
cudaError_t lca_index_build(const uint64_t* h, const uint64_t* row_off, uint32_t n_rows, uint64_t T, uint64_t max_key,
                            LcaIndexDev* out, cudaStream_t s);
cudaError_t lca_index_plan(const LcaIndexDev& x, uint64_t k0, uint64_t max_bytes, uint64_t plan[4], cudaStream_t s);
cudaError_t lca_index_text(const LcaIndexDev& x, uint64_t d0, uint64_t d1, char* out, cudaStream_t s);

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

// `sig kmers` (kmer_match_kernels.cuh): every window of every record hashed, the windows whose hash is in Q emitted as
// (record << 32 | ordinal, hash); ordinal = the window's index in seq_to_hashes order.  The caller fills the arguments
// (chunks of W windows per record, the probe layout, zeroed results); the launch picks the kernel from mode / K.
struct KmerMatchArgs {
    const uint8_t* bases;               // 16-byte aligned, readable up to the next 16-byte boundary past the end
    const uint64_t* rec_off;            // [n_rec] byte offset of every record
    const uint64_t* rec_len;            // [n_rec]
    const uint64_t* chunk_start;        // [n_rec + 1] prefix of the chunks of every record
    uint64_t n_chunks;
    int n_rec, W;                       // W: windows (window starts) per chunk
    int mode;                           // 0 rolled DNA (K = 21, 31, 51), 1 any other DNA k, 2 residues, 3 translated DNA
    uint32_t K;                         // DNA: k; protein family: residues per window
    uint64_t seed, max_hash;            // max_hash: UINT64_MAX for num sketches
    // Q
    const uint64_t* q;                  // sorted-unique, without a trailing UINT64_MAX
    uint64_t nq, q_top;                 // q_top = q[nq - 1] (0 when nq == 0)
    int q_has_max;                      // Q holds UINT64_MAX
    int split;                          // 1: shared-memory split table of nq keys; 0: global directory
    uint32_t shift;                     // bucket = key >> shift, buckets [0, nb)
    uint64_t nb;
    const uint32_t* gdir;               // global directory (nb + 1 entries) ...
    const uint32_t* bitmap;             // ... and occupancy bitmap at 2^fine_log2 times its resolution
    int fine_log2;
    const AaTables* tabs;
    // results
    uint64_t* keys; uint64_t* hashes; uint64_t cap;
    unsigned long long* count;          // matches found (may exceed cap)
    uint8_t* rec_hit;                   // [n_rec] at least one match
    uint8_t* rec_invalid;               // [n_rec] DNA: a window holds a non-ACGT byte (nullable)
};
bool kmer_match_split_fits(uint64_t nq);        // Q this large fits the shared-memory split table
// (key, hash) pairs sorted by the key bits [0, end_bit), into the *_out arrays
cudaError_t sort_kmer_matches(const uint64_t* keys, const uint64_t* hashes, uint64_t* keys_out, uint64_t* hashes_out,
                              uint64_t m, int end_bit, cudaStream_t s);
void launch_kmer_match(const KmerMatchArgs& a, cudaStream_t s);
// found hashes of a scaled query: flag[i] = 1 when some match holds q[i]; matches of records with skip[r] != 0 (nullable)
// do not count
void launch_match_mark_found(const uint64_t* keys, const uint64_t* hashes, uint64_t n, const uint8_t* skip,
                             const uint64_t* q, uint64_t nq, uint8_t* flag, cudaStream_t s);
// num query: record recs[i] (bottom-num sketch = row i of bh / boff) passes when a hash common with Q is among the first
// num of the union; rec_hit[recs[i]] is set to the result, flag[j] = 1 for the common q[j] of passing records that are
// not skipped (skip[recs[i]] != 0, nullable)
void launch_match_num_common(const uint64_t* bh, const uint64_t* boff, const uint32_t* recs, int n, const uint64_t* q,
                             uint64_t nq, uint32_t num, const uint8_t* skip, uint8_t* rec_hit, uint8_t* flag,
                             cudaStream_t s);

// Angular search (angular_search.cuh): for one abundance query and every row r of a set with abundances, over the
// elements <= max_hash of both, prod[r] = sum of q_abund * s_abund over shared hashes and bsq[r] = sum of s_abund^2
// (u64, wrapping).  The caller fills the query and subject fields; angular_search plans the probe layout, builds the
// global directory when the query is too large for the split table, zeroes prod / bsq and launches.
static constexpr uint64_t ANGULAR_CHUNK = 1024;        // elements of a row per warp task
// Queries up to this many keys become the shared-memory split table: 8 bytes per key plus a directory of about one u16
// entry per key is at most 164 KB, inside a CTA's 227 KB.  The table format itself stops at 32 759 keys, which would
// need 262 KB of keys alone.
static constexpr uint64_t ANGULAR_SPLIT_MAX = 16382;
struct AngularSearchArgs {
    // query, cut at max_hash, sorted-unique, without a trailing UINT64_MAX
    const uint64_t* q; const uint64_t* qa;
    uint64_t nq, q_top;                 // q_top = q[nq - 1] (0 when nq == 0)
    int q_has_max;                      // the query holds UINT64_MAX (max_hash == UINT64_MAX) ...
    uint64_t q_max_abund;               // ... with this abundance
    // probe layout (filled by angular_search)
    int split;                          // 1: shared-memory split table; 0: global directory + occupancy bitmap
    uint32_t shift; uint64_t nb;        // bucket = key >> shift, buckets [0, nb)
    const uint32_t* gdir; const uint32_t* bitmap; int fine_log2;
    // subjects
    const uint64_t* h; const uint64_t* ab; const uint64_t* off;
    const uint64_t* chunk_start;        // [n_rows + 1] prefix of ceil(row length / ANGULAR_CHUNK)
    uint64_t n_chunks; int n_rows;
    uint64_t max_hash;
    unsigned long long* prod; unsigned long long* bsq;   // [n_rows]
};
cudaError_t angular_search(AngularSearchArgs a, cudaStream_t s);

// covered[p] = 1 iff q[p] (sorted-unique, q_max = q[nq - 1]) is held by one of the rows rows[0..n_rows) of the CSR
// (hB, offB); the other nq bytes are 0.  Rows are read in place.
cudaError_t launch_query_cover(const uint64_t* q, uint64_t nq, uint64_t q_max, const uint64_t* hB,
                               const uint64_t* offB, const uint32_t* rows, uint64_t n_rows, uint8_t* covered,
                               cudaStream_t s);

// kernel-launch accounting (smb_kernel_launches)
void count_launches(int n);

}  // namespace smb
