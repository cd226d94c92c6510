/*
 * sourmash_b200.h -- C ABI of libsourmash_b200.so, the H100 (sm_90a) implementation of
 * sourmash's two data-parallel hot paths (FracMinHash sketching, sorted-u64 intersection).
 *
 * The library is a drop-in for the subset of the reference's C ABI
 * (sourmash/include/sourmash.h, generated from src/core/src/ffi/ *.rs) that the
 * Python object model binds for these paths, plus NEW batched entry points (smb_*) that
 * replace the reference's per-pair / per-record Python loops.  Part 1 keeps the reference's
 * names, argument order, ownership and error protocol; each group cites what it replaces.
 * Everything is plain C: opaque handles, pointers and sizes, no torch / C++ types.
 *
 * Error protocol (reference: src/core/src/ffi/utils.rs:17-19,58-86,195-208; Python side
 * src/sourmash/utils.py:65-78): no return codes.  A failing call stores (code, message) in a
 * thread-local slot and returns a zeroed value; callers do
 *     sourmash_err_clear(); r = f(...); if (sourmash_err_get_last_code()) -> raise.
 * All hashing and set-intersection arithmetic runs on the GPU; if no CUDA device is usable
 * the call fails with SOURMASH_ERROR_CODE_CUDA (there is no CPU fallback).
 */
#ifndef SOURMASH_B200_H_INCLUDED
#define SOURMASH_B200_H_INCLUDED

#include <stdbool.h>
#include <stdint.h>
#include <stdlib.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ===================================================================================== */
/* Part 1: reference-compatible ABI (same symbols as include/sourmash.h)                  */
/* ===================================================================================== */

/* include/sourmash.h:11-17 */
enum { /* HashFunctions */
  HASH_FUNCTIONS_MURMUR64_DNA = 1,
  HASH_FUNCTIONS_MURMUR64_PROTEIN = 2,
  HASH_FUNCTIONS_MURMUR64_DAYHOFF = 3,
  HASH_FUNCTIONS_MURMUR64_HP = 4,
};
typedef uint32_t HashFunctions;

/* include/sourmash.h:19-53 (numeric values from src/core/src/errors.rs:101-141).
 * SOURMASH_ERROR_CODE_CUDA is new: raised when the GPU path cannot run. */
enum { /* SourmashErrorCode */
  SOURMASH_ERROR_CODE_NO_ERROR = 0,
  SOURMASH_ERROR_CODE_PANIC = 1,
  SOURMASH_ERROR_CODE_INTERNAL = 2,
  SOURMASH_ERROR_CODE_MSG = 3,
  SOURMASH_ERROR_CODE_UNKNOWN = 4,
  SOURMASH_ERROR_CODE_MISMATCH_K_SIZES = 101,
  SOURMASH_ERROR_CODE_MISMATCH_DNA_PROT = 102,
  SOURMASH_ERROR_CODE_MISMATCH_SCALED = 103,
  SOURMASH_ERROR_CODE_MISMATCH_SEED = 104,
  SOURMASH_ERROR_CODE_MISMATCH_SIGNATURE_TYPE = 105,
  SOURMASH_ERROR_CODE_NON_EMPTY_MIN_HASH = 106,
  SOURMASH_ERROR_CODE_MISMATCH_NUM = 107,
  SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING = 108,
  SOURMASH_ERROR_CODE_CANNOT_UPSAMPLE_SCALED = 109,
  SOURMASH_ERROR_CODE_NO_MIN_HASH_FOUND = 110,
  SOURMASH_ERROR_CODE_EMPTY_SIGNATURE = 111,
  SOURMASH_ERROR_CODE_MULTIPLE_SKETCHES_FOUND = 112,
  SOURMASH_ERROR_CODE_INVALID_DNA = 1101,
  SOURMASH_ERROR_CODE_INVALID_PROT = 1102,
  SOURMASH_ERROR_CODE_INVALID_CODON_LENGTH = 1103,
  SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION = 1104,
  SOURMASH_ERROR_CODE_READ_DATA = 1201,
  SOURMASH_ERROR_CODE_STORAGE = 1202,
  SOURMASH_ERROR_CODE_HLL_PRECISION_BOUNDS = 1301,
  SOURMASH_ERROR_CODE_ANI_ESTIMATION_ERROR = 1401,
  SOURMASH_ERROR_CODE_IO = 100001,
  SOURMASH_ERROR_CODE_UTF8_ERROR = 100002,
  SOURMASH_ERROR_CODE_PARSE_INT = 100003,
  SOURMASH_ERROR_CODE_SERDE_ERROR = 100004,
  SOURMASH_ERROR_CODE_NIFFLER_ERROR = 100005,
  SOURMASH_ERROR_CODE_CSV_ERROR = 100006,
  SOURMASH_ERROR_CODE_ROCKS_DB_ERROR = 100007,
  SOURMASH_ERROR_CODE_CUDA = 200001,
};
typedef uint32_t SourmashErrorCode;

typedef struct SourmashComputeParameters SourmashComputeParameters;
typedef struct SourmashKmerMinHash SourmashKmerMinHash;
typedef struct SourmashSignature SourmashSignature;

/* include/sourmash.h:75-88: string returned by value; free with sourmash_str_free if owned */
typedef struct {
  char *data;
  uintptr_t len;
  bool owned;
} SourmashStr;

/* --- errors / init / strings: src/core/src/ffi/utils.rs:95-165,211-320 ------------------ */
void sourmash_init(void);
void sourmash_err_clear(void);
SourmashErrorCode sourmash_err_get_last_code(void);
SourmashStr sourmash_err_get_last_message(void);
SourmashStr sourmash_err_get_backtrace(void);
void sourmash_str_free(SourmashStr *s);
SourmashStr sourmash_str_from_cstr(const char *s);

/* --- hash primitive: src/core/src/ffi/mod.rs:22-31 -> lib.rs:57-59 ---------------------- */
uint64_t hash_murmur(const char *kmer, uint64_t seed);

/* --- residue encodings: src/core/src/ffi/minhash.rs:157-178 -> encodings.rs:298-343 ------- */
char sourmash_translate_codon(const char *codon);   /* 1..3 bases; else InvalidCodonLength */
char sourmash_aa_to_dayhoff(char aa);
char sourmash_aa_to_hp(char aa);

/* --- KmerMinHash: src/core/src/ffi/minhash.rs:18-483 (include/sourmash.h:169-273) -------- */
SourmashKmerMinHash *kmerminhash_new(uint64_t scaled, uint32_t k, HashFunctions hash_function,
                                     uint64_t seed, bool track_abundance, uint32_t n);
void kmerminhash_free(SourmashKmerMinHash *ptr);
void kmerminhash_slice_free(uint64_t *ptr, uintptr_t insize);
void kmerminhash_add_sequence(SourmashKmerMinHash *ptr, const char *sequence, bool force);
void kmerminhash_add_protein(SourmashKmerMinHash *ptr, const char *sequence);
const uint64_t *kmerminhash_seq_to_hashes(SourmashKmerMinHash *ptr, const char *sequence,
                                          uintptr_t insize, bool force, bool bad_kmers_as_zeroes,
                                          bool is_protein, uintptr_t *size);
void kmerminhash_clear(SourmashKmerMinHash *ptr);
void kmerminhash_add_hash(SourmashKmerMinHash *ptr, uint64_t h);
void kmerminhash_add_hash_with_abundance(SourmashKmerMinHash *ptr, uint64_t h, uint64_t abundance);
void kmerminhash_add_word(SourmashKmerMinHash *ptr, const char *word);
void kmerminhash_add_many(SourmashKmerMinHash *ptr, const uint64_t *hashes_ptr, uintptr_t insize);
void kmerminhash_add_from(SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other);
void kmerminhash_remove_hash(SourmashKmerMinHash *ptr, uint64_t h);
void kmerminhash_remove_many(SourmashKmerMinHash *ptr, const uint64_t *hashes_ptr, uintptr_t insize);
void kmerminhash_remove_from(SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other);
const uint64_t *kmerminhash_get_mins(const SourmashKmerMinHash *ptr, uintptr_t *size);
uintptr_t kmerminhash_get_mins_size(const SourmashKmerMinHash *ptr);
const uint64_t *kmerminhash_get_abunds(SourmashKmerMinHash *ptr, uintptr_t *size);
void kmerminhash_set_abundances(SourmashKmerMinHash *ptr, const uint64_t *hashes_ptr,
                                const uint64_t *abunds_ptr, uintptr_t insize, bool clear);
SourmashStr kmerminhash_md5sum(const SourmashKmerMinHash *ptr);
bool kmerminhash_is_protein(const SourmashKmerMinHash *ptr);
bool kmerminhash_dayhoff(const SourmashKmerMinHash *ptr);
bool kmerminhash_hp(const SourmashKmerMinHash *ptr);
uint64_t kmerminhash_seed(const SourmashKmerMinHash *ptr);
bool kmerminhash_track_abundance(const SourmashKmerMinHash *ptr);
void kmerminhash_disable_abundance(SourmashKmerMinHash *ptr);
void kmerminhash_enable_abundance(SourmashKmerMinHash *ptr);
uint32_t kmerminhash_num(const SourmashKmerMinHash *ptr);
uint32_t kmerminhash_ksize(const SourmashKmerMinHash *ptr);
uint64_t kmerminhash_max_hash(const SourmashKmerMinHash *ptr);
HashFunctions kmerminhash_hash_function(const SourmashKmerMinHash *ptr);
void kmerminhash_hash_function_set(SourmashKmerMinHash *ptr, HashFunctions hash_function);
void kmerminhash_merge(SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other);
bool kmerminhash_is_compatible(const SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other);
uint64_t kmerminhash_count_common(const SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other,
                                  bool downsample);
SourmashKmerMinHash *kmerminhash_intersection(const SourmashKmerMinHash *ptr,
                                              const SourmashKmerMinHash *other);
uint64_t kmerminhash_intersection_union_size(const SourmashKmerMinHash *ptr,
                                             const SourmashKmerMinHash *other, uint64_t *union_size);
double kmerminhash_jaccard(const SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other);
double kmerminhash_similarity(const SourmashKmerMinHash *ptr, const SourmashKmerMinHash *other,
                              bool ignore_abundance, bool downsample);
double kmerminhash_angular_similarity(const SourmashKmerMinHash *ptr,
                                      const SourmashKmerMinHash *other);

/* --- Signature (subset): src/core/src/ffi/signature.rs:24-217 (include/sourmash.h:364-396) */
SourmashSignature *signature_new(void);
void signature_free(SourmashSignature *ptr);
SourmashSignature *signature_from_params(const SourmashComputeParameters *ptr);
uintptr_t signature_len(const SourmashSignature *ptr);
bool signature_eq(const SourmashSignature *ptr, const SourmashSignature *other);
void signature_add_sequence(SourmashSignature *ptr, const char *sequence, bool force);
void signature_add_protein(SourmashSignature *ptr, const char *sequence);
SourmashKmerMinHash *signature_first_mh(const SourmashSignature *ptr);
SourmashKmerMinHash **signature_get_mhs(const SourmashSignature *ptr, uintptr_t *size);
void smb_mh_array_free(SourmashKmerMinHash** arr);   /* the array signature_get_mhs malloc'd (not the sketches); the reference header has no counterpart and leaks it */
void signature_set_mh(SourmashSignature *ptr, const SourmashKmerMinHash *other);
void signature_push_mh(SourmashSignature *ptr, const SourmashKmerMinHash *other);
SourmashStr signature_get_name(const SourmashSignature *ptr);
SourmashStr signature_get_filename(const SourmashSignature *ptr);
SourmashStr signature_get_license(const SourmashSignature *ptr);
void signature_set_name(SourmashSignature *ptr, const char *name);
void signature_set_filename(SourmashSignature *ptr, const char *name);

/* --- ComputeParameters: src/core/src/ffi/cmd/compute.rs:14-170 (include/sourmash.h:89-131) */
SourmashComputeParameters *computeparams_new(void);
void computeparams_free(SourmashComputeParameters *ptr);
const uint32_t *computeparams_ksizes(const SourmashComputeParameters *ptr, uintptr_t *size);
void computeparams_ksizes_free(uint32_t *ptr, uintptr_t insize);
void computeparams_set_ksizes(SourmashComputeParameters *ptr, const uint32_t *ksizes_ptr,
                              uintptr_t insize);
bool computeparams_dna(const SourmashComputeParameters *ptr);
bool computeparams_protein(const SourmashComputeParameters *ptr);
bool computeparams_dayhoff(const SourmashComputeParameters *ptr);
bool computeparams_hp(const SourmashComputeParameters *ptr);
bool computeparams_track_abundance(const SourmashComputeParameters *ptr);
uint32_t computeparams_num_hashes(const SourmashComputeParameters *ptr);
uint64_t computeparams_scaled(const SourmashComputeParameters *ptr);
uint64_t computeparams_seed(const SourmashComputeParameters *ptr);
void computeparams_set_dna(SourmashComputeParameters *ptr, bool v);
void computeparams_set_protein(SourmashComputeParameters *ptr, bool v);
void computeparams_set_dayhoff(SourmashComputeParameters *ptr, bool v);
void computeparams_set_hp(SourmashComputeParameters *ptr, bool v);
void computeparams_set_track_abundance(SourmashComputeParameters *ptr, bool v);
void computeparams_set_num_hashes(SourmashComputeParameters *ptr, uint32_t num);
void computeparams_set_scaled(SourmashComputeParameters *ptr, uint64_t scaled);
void computeparams_set_seed(SourmashComputeParameters *ptr, uint64_t new_seed);

/* ===================================================================================== */
/* Part 2: batched entry points (NEW; the reference iterates these in Python)             */
/* ===================================================================================== */

/* A set of sketches resident in HBM: CSR of sorted-unique u64 rows
 * (offsets[n_rows+1], hashes[offsets[n_rows]]), optionally with abundances. */
typedef struct SmbSketchSet SmbSketchSet;

/* device / context ------------------------------------------------------------------- */
int32_t smb_device_count(void);                 /* 0 if no usable CUDA device (no error set) */
const char* smb_device_probe_error(void);       /* the CUDA runtime's message when the probe failed, else "" (static storage) */
void smb_set_device(int32_t device);            /* per-thread; default = current CUDA device  */
void smb_set_stream(void *cuda_stream);         /* run subsequent work on this cudaStream_t   */
void smb_synchronize(void);
uint64_t smb_kernel_launches(void);             /* number of kernels launched by this library */
/* out[i] = pow(x[i], e) with the C library's pow -- the function behind Python's float ** float, which the reference's
 * ANI formulas use pair by pair (distance_utils.py:258-407: c ** (1/k)); numpy's vectorised power may differ in the last
 * bit, so the matrix forms of those formulas call this (host only, no device work). */
void smb_pow_f64(const double *x, double e, double *out, uintptr_t n);
void smb_set_profiling(bool on);                /* record CUDA events around the dominant kernels */
double smb_last_kernel_ms(int32_t which);       /* 0: last pairwise tile kernel, 1: last hash pass */
/* planner of the last all-vs-all count (this thread): {1 = inverted join / 0 = tile kernel,
 * estimated increments, estimated elements, largest hash group seen in the sample} */
void smb_last_compare_plan(double *out4);
void *smb_alloc_pinned(uintptr_t nbytes);       /* page-locked host memory for e2e transfers  */
void smb_free_pinned(void *ptr);
uint64_t smb_max_hash_for_scaled(uint64_t scaled);   /* sketch/minhash.rs:21-27 */

/* sketch sets ------------------------------------------------------------------------ */
/* copy host CSR to the device (abunds may be NULL) */
SmbSketchSet *smb_sketchset_from_host(const uint64_t *hashes, const uint64_t *offsets,
                                      uintptr_t n_rows, const uint64_t *abunds);
/* wrap device-resident CSR without copying (caller keeps the buffers alive);
 * h_offsets is the same offsets array on the host */
SmbSketchSet *smb_sketchset_from_device(const uint64_t *d_hashes, const uint64_t *d_offsets,
                                        const uint64_t *h_offsets, uintptr_t n_rows);
void smb_sketchset_free(SmbSketchSet *set);
uintptr_t smb_sketchset_len(const SmbSketchSet *set);
uint64_t smb_sketchset_total_hashes(const SmbSketchSet *set);
bool smb_sketchset_has_abunds(const SmbSketchSet *set);
void smb_sketchset_offsets(const SmbSketchSet *set, uint64_t *offsets_out);   /* n_rows+1 */
void smb_sketchset_to_host(const SmbSketchSet *set, uint64_t *hashes_out, uint64_t *abunds_out);
/* device-to-device copy into caller-owned buffers (e.g. torch tensors), stream ordered */
void smb_sketchset_copy_to_device(const SmbSketchSet *set, uint64_t *d_hashes_out,
                                  uint64_t *d_offsets_out);
const uint64_t *smb_sketchset_device_hashes(const SmbSketchSet *set);
const uint64_t *smb_sketchset_device_offsets(const SmbSketchSet *set);
/* new set holding, for every row, the prefix h <= max_hash (downsample_scaled,
 * sketch/minhash.rs:777-798) */
SmbSketchSet *smb_sketchset_downsample(const SmbSketchSet *set, uint64_t max_hash);
/* the given rows (any order) as a new resident set */
SmbSketchSet *smb_sketchset_take_rows(const SmbSketchSet *set, const uint32_t *rows, uintptr_t n);

/* sketching (replaces the per-record loop command_sketch.py:662-789 ->
 * signature_add_sequence -> SeqToHashes::next) --------------------------------------- */
/* Input: n_seqs records concatenated in `seqs` (record r = bytes [seq_offsets[r],
 * seq_offsets[r+1])); seq_to_sketch[r] (NULL = one sketch per record) says which output
 * sketch a record feeds.  Output row (sketch s, ksizes[j]) is s * n_ksizes + j.
 * scaled > 0: FracMinHash rows (h <= max_hash_for_scaled(scaled)); scaled == 0: bottom-`num`.
 * Invalid (non-ACGT) bases skip the windows covering them (force=True semantics).
 * n_kmers_out (nullable) receives the number of k-mer windows hashed. */
SmbSketchSet *smb_sketch_sequences(const uint8_t *seqs, const uint64_t *seq_offsets,
                                   uintptr_t n_seqs, const uint32_t *seq_to_sketch,
                                   uintptr_t n_sketches, const uint32_t *ksizes,
                                   uintptr_t n_ksizes, uint64_t scaled, uint32_t num, uint64_t seed,
                                   bool track_abundance, uint64_t *n_kmers_out);
/* Protein-family sketches (`sourmash sketch protein` / `sketch translate`,
 * signature.rs:307-392): hash_function is PROTEIN, DAYHOFF or HP; ksizes carry the ABI value
 * (3 x residues).  input_is_protein: records are residues (add_protein); otherwise DNA that is
 * translated in six frames (two hashes per window of ksize bases, no validity filter). */
SmbSketchSet *smb_sketch_sequences_aa(const uint8_t *seqs, const uint64_t *seq_offsets,
                                      uintptr_t n_seqs, const uint32_t *seq_to_sketch,
                                      uintptr_t n_sketches, const uint32_t *ksizes,
                                      uintptr_t n_ksizes, HashFunctions hash_function,
                                      bool input_is_protein, uint64_t scaled, uint32_t num,
                                      uint64_t seed, bool track_abundance, uint64_t *n_kmers_out);
/* Same with the bases already in HBM: d_bases holds the streams back to back, stream s at
 * byte h_stream_offsets[s] (16-byte aligned) with length h_stream_lens[s]; records inside a
 * stream separated by any non-ACGT byte.  One sketch per stream. */
SmbSketchSet *smb_sketch_streams_dev(const uint8_t *d_bases, const uint64_t *h_stream_offsets,
                                     const uint64_t *h_stream_lens, uintptr_t n_streams,
                                     const uint32_t *ksizes, uintptr_t n_ksizes, uint64_t scaled,
                                     uint32_t num, uint64_t seed, bool track_abundance,
                                     uint64_t *n_kmers_out);

/* Inverted index (hash -> rows) over a resident set, for databases that are queried repeatedly:
 * once built, smb_one_vs_many and the gather session on this set probe the index -- one directory
 * lookup per *query* hash and one increment per match -- instead of streaming every row of the set
 * (the job of the reference's RevIndex, src/core/src/index/revindex/, for the same counts).
 * Costs about 1.5x the set's size in HBM; at most 2^31 - 1 hashes.  Returns the number of distinct
 * hashes.  Results are identical with and without the index. */
uint64_t smb_sketchset_build_index(SmbSketchSet *set);
void smb_sketchset_drop_index(SmbSketchSet *set);
bool smb_sketchset_has_index(const SmbSketchSet *set);

/* intersection ------------------------------------------------------------------------ */
/* common[i*n_b + j] = |A_i ∩ B_j| (b == NULL: b = a, only i<j computed, mirrored, diagonal
 * = |A_i|).  num > 0 selects bottom-k semantics (minhash.rs:593-617) and fills usize_out
 * (nullable) with |M|.  Output on the host. */
void smb_pairwise_common(const SmbSketchSet *a, const SmbSketchSet *b, uint32_t num,
                         uint32_t *common_out, uint32_t *usize_out);
/* compare_all_pairs / compare_serial (src/sourmash/compare.py:14-64,328-358): float64
 * (n, n) Jaccard matrix, ones on the diagonal.  out on the host (pinned or pageable). */
void smb_compare_jaccard(const SmbSketchSet *set, uint32_t num, double *out);
/* all-vs-all angular similarity (KmerMinHash::angular_similarity, sketch/minhash.rs:635-680) of
 * a set that carries abundances; float64 (n, n), ones on the diagonal */
void smb_compare_angular(const SmbSketchSet *set, double *out);
/* same, result left in HBM (d_out: n*n doubles) -- used to time the kernels alone */
void smb_compare_jaccard_dev(const SmbSketchSet *set, uint32_t num, double *d_out);
/* Multi-GPU building blocks.  Shard `shard` of `n_shards` computes the common counts of its
 * share of row tiles (dealt cyclically) into d_common (n*n u32, zero-initialised by the
 * caller; only entries j > i of owned rows are written) -- partial matrices are then summed
 * across ranks (NCCL all-reduce) and each rank finalises a block of rows. */
void smb_pairwise_counts_shard_dev(const SmbSketchSet *set, uint32_t shard, uint32_t n_shards,
                                   uint32_t *d_common);
/* The same split with WHOLE ROWS as the unit of exchange (what a reduce-scatter by row blocks needs): shard `shard`
 * writes its partial counters of every cell (i, j), i != j, into d_counts (n*n u32, every cell written, nothing to
 * zero).  With the stripe layout the shard is key range `shard` of the hash space -- sort, tags and counting all
 * shrink with 1/n_shards; otherwise the upper-triangle shards above, mirrored.  Partial matrices add up. */
void smb_compare_counts_shard_dev(const SmbSketchSet *set, uint32_t shard, uint32_t n_shards, void *d_counts, uint32_t bits);
/* (bits = 32: uint32_t counters; bits = 16: uint16_t counters, allowed when every row is shorter than 65 536 hashes --
 * half the bytes to exchange; two of them added as one uint32_t never carry into each other) */
/* summed whole-row counters of rows [row_begin, row_end) (row_begin first, leading dimension n) -> float64 Jaccard rows */
void smb_finalize_counts_rows_dev(const SmbSketchSet *set, const void *d_counts_rows, uint32_t bits, uint64_t row_begin,
                                  uint64_t row_end, double *d_out);
/* d_out[(i - row_begin) * n + j] = jaccard(i, j) for row_begin <= i < row_end, from a complete
 * upper-triangular count matrix */
void smb_finalize_jaccard_rows_dev(const SmbSketchSet *set, const uint32_t *d_common,
                                   uint64_t row_begin, uint64_t row_end, double *d_out);
/* float64 rows [row_begin, row_end) of the all-vs-all Jaccard matrix of a scaled set into d_out
 * ((row_end - row_begin) x n, device memory).  With the stripe layout of the join (the default) only those
 * rows are counted, so one process per GPU can take a block of rows without exchanging counts; with
 * SMB_JOIN_LAYOUT=plain the whole count matrix is computed first. */
void smb_compare_jaccard_rows_dev(const SmbSketchSet *set, uint64_t row_begin, uint64_t row_end,
                                  double *d_out);
/* Index.find inner loop (src/sourmash/index/__init__.py:115-170): one query vs every row */
void smb_one_vs_many(const uint64_t *query, uintptr_t n_query, const SmbSketchSet *db,
                     uint32_t *common_out);
/* the same with the (sorted) query and the n_rows counters in device memory: nothing crosses PCIe */
void smb_one_vs_many_dev(const uint64_t *d_query, uintptr_t n_query, const SmbSketchSet *db,
                         uint32_t *d_common_out);
/* one_vs_many for many queries: counts_out[q * n_rows + r] = |query q ∩ row r| (a Q x n_rows host matrix).
 * q_hashes / q_offsets: the queries as CSR (n_queries + 1 offsets from 0, not decreasing), each sorted and unique.
 * Groups of consecutive queries share one streaming pass over the database (its range-major copy, built on first
 * use); an indexed set, SMB_SEARCH_LAYOUT=global, or a group of one query counts query by query.  The counts are
 * those of smb_one_vs_many for each query. */
void smb_many_vs_many(const uint64_t *q_hashes, const uint64_t *q_offsets, uintptr_t n_queries,
                      const SmbSketchSet *db, uint32_t *counts_out);
/* the same with the hashes and the Q x n_rows counters in device memory; the offsets stay on the host */
void smb_many_vs_many_dev(const uint64_t *d_q_hashes, const uint64_t *q_offsets, uintptr_t n_queries,
                          const SmbSketchSet *db, uint32_t *d_counts_out);
/* gather (CounterGather + GatherDatabases, src/sourmash/index/__init__.py:777-909,
 * src/sourmash/search.py:877-949): iterative min-set-cover.  Returns number of rounds;
 * match_ids/isect_sizes receive, per round, the chosen row and |match ∩ remaining query|.
 * threshold: stop when the best remaining overlap is < threshold (at least 1). */
uintptr_t smb_gather(const uint64_t *query, uintptr_t n_query, const SmbSketchSet *db,
                     uint32_t threshold, uint32_t *match_ids, uint32_t *isect_sizes,
                     uintptr_t max_rounds);

/* gather as a session -- the building blocks of smb_gather, exposed so that a database sharded
 * over several GPUs can run the same rounds with two tiny collectives per round
 * (all-gather of (count, row), broadcast of the winning intersection; SURVEY §8e):
 *   begin      counters[j] = |query ∩ S_j| for the local shard
 *   peek       best remaining (count, local row), lowest row wins ties
 *   intersect  remaining query ∩ local row -> host buffer, returns its size
 *   apply      counters -= |intersect ∩ S_j|, query -= intersect; returns remaining query size */
typedef struct SmbGatherState SmbGatherState;
SmbGatherState *smb_gather_begin(const uint64_t *query, uintptr_t n_query, const SmbSketchSet *db);
/* same; rows overlapping the query by fewer than min_count hashes are dropped up front (they
 * can never be picked), so later rounds only stream the surviving candidates */
SmbGatherState *smb_gather_begin_min(const uint64_t *query, uintptr_t n_query, const SmbSketchSet *db,
                                     uint32_t min_count);
void smb_gather_peek(SmbGatherState *st, uint32_t *best_count, uint32_t *best_row);
uintptr_t smb_gather_intersect(SmbGatherState *st, uint32_t row, uint64_t *out_hashes);
uintptr_t smb_gather_apply(SmbGatherState *st, const uint64_t *intersect, uintptr_t n);
void smb_gather_end(SmbGatherState *st);

/* multigather (src/sourmash/commands.py:1124-1386): the gather of many queries against one resident database.
 * q_hashes / q_offsets: the queries as CSR (n_queries + 1 offsets), each sorted and unique.  Per query:
 * thresholds[i] -- stop when the best remaining overlap is below it (at least 1; NULL: 1) -- and min_counts[i] --
 * only rows sharing at least that many hashes with the query take part (NULL: 1).  At most max_rounds picks per
 * query.  The rounds of all queries run together on the device, a fixed number of launches per round; an indexed
 * set, or candidate rows too large for the shared-memory table, take the session loop query by query -- the
 * results are the same.  Every query's result equals smb_gather's for that query alone.
 *   rounds    number of picks of query `query`
 *   picks     its picked rows, |row ∩ remaining query| and |row ∩ query| per round (arrays of rounds() entries;
 *             any may be NULL)
 *   consumed  for every hash of every query (q_offsets[n_queries] entries): the round that took it, UINT32_MAX if none
 *   round_launches  kernel launches of the batched rounds (prefetch not included) */
typedef struct SmbMultiGather SmbMultiGather;
SmbMultiGather *smb_multigather(const uint64_t *q_hashes, const uint64_t *q_offsets, uintptr_t n_queries,
                                const SmbSketchSet *db, const uint32_t *thresholds, const uint32_t *min_counts,
                                uintptr_t max_rounds);
uintptr_t smb_multigather_rounds(const SmbMultiGather *m, uintptr_t query);
void smb_multigather_picks(const SmbMultiGather *m, uintptr_t query, uint32_t *rows, uint32_t *sizes,
                           uint32_t *overlaps);
void smb_multigather_consumed(const SmbMultiGather *m, uint32_t *consumed_round);
uint64_t smb_multigather_round_launches(const SmbMultiGather *m);
void smb_multigather_free(SmbMultiGather *m);

/* ==========================================================================================
 * Part 3: native ingest (SURVEY §8 f1, f2) -- the data formats either side of the hot paths,
 * read without per-record Python so that they do not dominate end to end.
 * ======================================================================================== */
/* FASTA / FASTQ, plain or gzip (decided per file from its content); replaces the screed record
 * loop of src/sourmash/command_sketch.py:697-766.  Record name = the header line after the
 * marker, sequence = the record's lines joined.  Files are read by up to n_threads threads
 * (<= 0: one per core, at most 32); records keep input order.  The sequence bytes live in
 * page-locked memory when a GPU is present, so smb_sketch_records uploads them at full speed. */
typedef struct SmbRecords SmbRecords;
SmbRecords *smb_records_read(const char *const *paths, uintptr_t n_paths, int32_t n_threads);
void smb_records_free(SmbRecords *r);
uintptr_t smb_records_len(const SmbRecords *r);
uint64_t smb_records_total_bytes(const SmbRecords *r);
const uint8_t *smb_records_data(const SmbRecords *r);
const uint64_t *smb_records_starts(const SmbRecords *r);           /* n: byte offset of each record */
const uint64_t *smb_records_lengths(const SmbRecords *r);          /* n */
const uint32_t *smb_records_files(const SmbRecords *r);            /* n: index into paths */
const char *smb_records_names(const SmbRecords *r, const uint64_t **name_offsets);
/* The sequence bytes sit in one buffer (every file owns a 16-byte aligned region, records packed
 * inside it); a one-buffer pool keeps the page-locked allocation alive between calls.
 * smb_sketch_records sketches the records of a batch like smb_sketch_sequences /
 * smb_sketch_sequences_aa; hash_function DNA ignores input_is_protein */
SmbSketchSet *smb_sketch_records(const SmbRecords *r, const uint32_t *rec_to_sketch,
                                 uintptr_t n_sketches, const uint32_t *ksizes, uintptr_t n_ksizes,
                                 HashFunctions hash_function, bool input_is_protein, uint64_t scaled,
                                 uint32_t num, uint64_t seed, bool track_abundance,
                                 uint64_t *n_kmers_out);

/* Signature objects straight from a sketch set (the tail of _compute_individual,
 * command_sketch.py:770-789): signature g owns rows [g * n_ksizes, (g + 1) * n_ksizes); ksizes
 * are the ABI values.  Array freed with signatures_array_free, objects with signature_free. */
SourmashSignature **smb_signatures_from_sketchset(const SmbSketchSet *set, const uint32_t *ksizes,
                                                  uintptr_t n_ksizes, HashFunctions hash_function,
                                                  uint64_t scaled, uint32_t num, uint64_t seed,
                                                  uintptr_t *size);

/* .sig / .sig.gz JSON (src/core/src/signature.rs:401-445, sketch/minhash.rs:103-184) parsed
 * straight into CSR: every sketch of every signature of every file is one row (unsorted mins
 * are sorted like the reference's loader does).  Replaces loading N objects through
 * signatures_load_path + kmerminhash_get_mins for compare / search / gather over many files. */
typedef struct SmbSigs SmbSigs;
typedef struct {
  uint32_t sig_index;      /* signature object the sketch belongs to (name / filename) */
  uint32_t file;           /* index into paths */
  uint32_t ksize;          /* as stored: 3 x residues for protein-family sketches */
  uint32_t num;            /* 0 when max_hash != 0 (minhash.rs:146) */
  uint64_t max_hash;
  uint64_t seed;
  uint32_t hash_function;  /* HashFunctions */
  bool has_abund;
  uint64_t n_mins;
} SmbSketchInfo;
SmbSigs *smb_sigs_read(const char *const *paths, uintptr_t n_paths, int32_t n_threads);
/* flags for .zip inputs: 1 = ignore the manifest (use_manifest=False), 2 = without a manifest try
 * every member, not only *.sig / *.sig.gz (traverse_yield_all=True) */
SmbSigs *smb_sigs_read_opts(const char *const *paths, uintptr_t n_paths, int32_t n_threads,
                            uint32_t flags);
SmbSigs *smb_sigs_parse(const char *data, uintptr_t len);          /* JSON text or gzip of it */
/* the same batch from objects already in memory (first sketch of every signature, like
 * SourmashSignature.minhash): N sketches out of N objects in one call instead of
 * N x (signature_first_mh + kmerminhash_get_mins + getters) */
SmbSigs *smb_sigs_from_signatures(const SourmashSignature *const *sigs, uintptr_t n);
SmbSigs *smb_sigs_from_minhashes(const SourmashKmerMinHash *const *mhs, uintptr_t n);
void smb_sigs_free(SmbSigs *s);
uintptr_t smb_sigs_n_signatures(const SmbSigs *s);
uintptr_t smb_sigs_n_sketches(const SmbSigs *s);
bool smb_sigs_any_abund(const SmbSigs *s);
void smb_sigs_sketch_info(const SmbSigs *s, uintptr_t i, SmbSketchInfo *out);
void smb_sigs_sketch_info_all(const SmbSigs *s, SmbSketchInfo *out);   /* out[n_sketches] */
SourmashStr smb_sigs_sketch_md5(const SmbSigs *s, uintptr_t i);      /* the md5sum field as stored */
/* md5 of every sketch computed from its hashes (KmerMinHash::md5sum): out[32 * n_sketches] hex, no NULs */
void smb_sigs_md5_all(const SmbSigs *s, char *out);
SourmashStr smb_sigs_sig_name(const SmbSigs *s, uintptr_t j);
SourmashStr smb_sigs_sig_filename(const SmbSigs *s, uintptr_t j);
SourmashStr smb_sigs_sig_license(const SmbSigs *s, uintptr_t j);
SourmashStr smb_sigs_sig_location(const SmbSigs *s, uintptr_t j);  /* zip member the signature came from, else "" */
const uint64_t *smb_sigs_offsets(const SmbSigs *s);                /* n_sketches + 1 */
const uint64_t *smb_sigs_mins(const SmbSigs *s);
const uint64_t *smb_sigs_abunds(const SmbSigs *s);                 /* 1 where a sketch has none */
SourmashKmerMinHash *smb_sigs_minhash(const SmbSigs *s, uintptr_t i);   /* new owned object */
/* rows (NULL: all) as one SourmashSignature per sketch, like signatures_load_*: array freed with
 * signatures_array_free, objects with signature_free */
SourmashSignature **smb_sigs_signatures(const SmbSigs *s, const uint32_t *rows, uintptr_t n_rows,
                                        uintptr_t *size);
/* rows (NULL: all) -> device-resident CSR; max_hash != 0 keeps the prefix h <= max_hash of every
 * row (downsample_scaled, sketch/minhash.rs:777-798) */
SmbSketchSet *smb_sigs_to_sketchset(const SmbSigs *s, const uint32_t *rows, uintptr_t n_rows,
                                    uint64_t max_hash, bool with_abunds);

/* reference ABI for .sig I/O: src/core/src/ffi/signature.rs:219-343 (include/sourmash.h:389-414).
 * One SourmashSignature per sketch, filtered by ksize (0: any; compared with the stored ksize)
 * and molecule type (NULL: any).  The returned array is freed with signatures_array_free, the
 * objects with signature_free; buffers with nodegraph_buffer_free (the reference's name). */
SourmashSignature **signatures_load_path(const char *ptr, bool ignore_md5sum, uintptr_t ksize,
                                         const char *select_moltype, uintptr_t *size);
SourmashSignature **signatures_load_buffer(const char *ptr, uintptr_t insize, bool ignore_md5sum,
                                           uintptr_t ksize, const char *select_moltype,
                                           uintptr_t *size);
const uint8_t *signatures_save_buffer(const SourmashSignature *const *ptr, uintptr_t size,
                                      uint8_t compression, uintptr_t *osize);
SourmashStr signature_save_json(const SourmashSignature *ptr);
void nodegraph_buffer_free(uint8_t *ptr, uintptr_t insize);
void signatures_array_free(SourmashSignature **ptr, uintptr_t size);

/* --- .zip collections: src/core/src/ffi/storage.rs:15-141 (include/sourmash.h:469-486) -------
 * Read-only view of a zip file of signatures (members in central-directory order, zip64
 * included).  zipstorage_load resolves `path`, then `subdir + path` (storage/mod.rs:339-363);
 * a missing member fails with SOURMASH_ERROR_CODE_STORAGE; the buffer is freed with
 * nodegraph_buffer_free.  The string arrays are read as paths[i][0], like the reference's.
 * smb_sigs_read accepts such files directly and loads every member the reference's
 * ZipFileLinearIndex.signatures() would yield (src/sourmash/index/__init__.py:639-683):
 * SOURMASH-MANIFEST.csv locations filtered by its md5 column, else every *.sig / *.sig.gz. */
typedef struct SourmashZipStorage SourmashZipStorage;
SourmashZipStorage *zipstorage_new(const char *ptr, uintptr_t insize);
void zipstorage_free(SourmashZipStorage *ptr);
const uint8_t *zipstorage_load(const SourmashZipStorage *ptr, const char *path_ptr,
                               uintptr_t insize, uintptr_t *size);
SourmashStr **zipstorage_filenames(const SourmashZipStorage *ptr, uintptr_t *size);
SourmashStr **zipstorage_list_sbts(const SourmashZipStorage *ptr, uintptr_t *size);
void zipstorage_set_subdir(SourmashZipStorage *ptr, const char *path_ptr, uintptr_t insize);
SourmashStr zipstorage_path(const SourmashZipStorage *ptr);
SourmashStr zipstorage_subdir(const SourmashZipStorage *ptr);

#ifdef __cplusplus
}
#endif
#endif /* SOURMASH_B200_H_INCLUDED */
