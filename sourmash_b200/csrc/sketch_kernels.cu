// sketch_kernels.cu -- FracMinHash / MinHash sketch construction kernels for sm_90a (H100).
//
// Replaces the reference's per-k-mer CPU loop:
//   SeqToHashes::new / ::next (DNA branch)   src/core/src/signature.rs:190-232, 246-306
//   revcomp / COMPLEMENT / VALID             src/core/src/encodings.rs:85-101, 370-377
//   _hash_murmur                             src/core/src/lib.rs:57-59 (murmurhash3 0.0.5 x64_128 .0)
//   SigsTrait::add_sequence                  src/core/src/signature.rs:38-58 (drop Ok(0))
//   add_hash_with_abundance (scaled filter)  src/core/src/sketch/minhash.rs:313-383
//
// Design: this path is integer-issue bound (~150 SASS integer ops per k-mer, 1 byte of
// HBM traffic per k-mer), so the kernel is organised around instruction count, not bytes:
// every thread owns W consecutive windows and rolls the forward and reverse-complement
// k-mers through registers as little-endian ASCII words (exactly the words murmur3 consumes)
// plus a 2-bit packed copy used only for the lexicographic min(kmer, revcomp) decision.  Input
// bases are read with 16-byte vector loads; survivors (h <= max_hash, h != 0) are staged in a
// shared-memory buffer and flushed with one atomicAdd per CTA.  A block-level bitonic sort +
// unique materialises each sketch row.
#include <stdlib.h>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "kernels.h"
#include "kmer_roll.cuh"
#include "sketch_device.cuh"
#include "aa_kmers.cuh"
#include "kmer_match_kernels.cuh"

namespace smb {

// ---------------------------------------------------------------------------------------
// Any other k: one thread per window, bytes straight from global/L1 (slow path, same results).
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ u32 up_byte(u32 x) { return (x >= 'a' && x <= 'z') ? x - 32u : x; }
__device__ __forceinline__ bool valid_base(u32 u) { return u == 'A' || u == 'C' || u == 'G' || u == 'T'; }
__device__ __forceinline__ u32 comp_base(u32 u) { return u == 'A' ? 'T' : u == 'C' ? 'G' : u == 'G' ? 'C' : 'A'; }

// one window of any k: validity of its k bytes and the murmur3 of the canonical k-mer (0 when invalid)
__device__ __forceinline__ u64 dna_window_hash(const u8* __restrict__ base, u64 w, u32 K, u64 seed, bool& valid) {
    valid = true;
    for (u32 t = 0; t < K; ++t) valid = valid && valid_base(up_byte(base[w + t]));
    if (!valid) return 0;
    bool fwd = true;
    for (u32 t = 0; t < K; ++t) {
        u32 f = up_byte(base[w + t]), r = comp_base(up_byte(base[w + K - 1 - t]));
        if (f != r) { fwd = f < r; break; }
    }
    auto at = [&](u32 t) -> u64 {
        return fwd ? up_byte(base[w + t]) : comp_base(up_byte(base[w + K - 1 - t]));
    };
    u64 h1 = seed, h2 = seed;
    const u32 nblk = K / 16;
    for (u32 b = 0; b < nblk; ++b) {
        u64 k1 = 0, k2 = 0;
        for (int i = 7; i >= 0; --i) { k1 = (k1 << 8) | at(16 * b + i); k2 = (k2 << 8) | at(16 * b + 8 + i); }
        k1 *= SMB_C1; k1 = smb_rotl64(k1, 31); k1 *= SMB_C2; h1 ^= k1;
        h1 = smb_rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729ULL;
        k2 *= SMB_C2; k2 = smb_rotl64(k2, 33); k2 *= SMB_C1; h2 ^= k2;
        h2 = smb_rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5ULL;
    }
    const u32 tail = K & 15u, tb = 16 * nblk;
    if (tail > 8) {
        u64 k2 = 0;
        for (u32 i = tail; i > 8; --i) k2 = (k2 << 8) | at(tb + i - 1);
        k2 *= SMB_C2; k2 = smb_rotl64(k2, 33); k2 *= SMB_C1; h2 ^= k2;
    }
    if (tail > 0) {
        u64 k1 = 0;
        for (u32 i = tail < 8 ? tail : 8; i > 0; --i) k1 = (k1 << 8) | at(tb + i - 1);
        k1 *= SMB_C1; k1 = smb_rotl64(k1, 31); k1 *= SMB_C2; h1 ^= k1;
    }
    h1 ^= (u64)K; h2 ^= (u64)K;
    h1 += h2; h2 += h1;
    h1 = smb_fmix64(h1); h2 = smb_fmix64(h2);
    return h1 + h2;
}

template <bool RAW>
__global__ void __launch_bounds__(256) hash_kmers_generic_kernel(HashArgs a, u32 K) {
    __shared__ int s_stream;
    if (threadIdx.x == 0) s_stream = find_stream(a.tile_start, a.n_streams, blockIdx.x + a.tile_base);
    __syncthreads();
    const int stream = s_stream;
    const u64 L = a.stream_len[stream];
    const u8* __restrict__ base = a.bases + a.stream_off[stream];
    if (L < K || K == 0) return;
    const u64 nwin = L - K + 1;
    const u64 tile = blockIdx.x + a.tile_base - a.tile_start[stream];
    const u64 w = tile * 256ull + threadIdx.x;
    if (w >= nwin) return;
    const int sk = a.stream_row ? (int)a.stream_row[stream] : stream;
    const int row = sk * a.row_stride + a.row_index;
    bool valid;
    const u64 h = dna_window_hash(base, w, K, a.seed, valid);
    if (RAW) {
        a.raw_out[w] = valid ? h : 0ull;
    } else if (valid && h != 0ull && h <= a.max_hash) {
        u32 g = atomicAdd(&a.cand_cnt[row], 1u);
        u64 capr = a.cand_off[row + 1] - a.cand_off[row];
        if (g < capr) a.cand[a.cand_off[row] + g] = h;
    }
}

template <bool RAW>
static void launch_hash_one_k(HashArgs a, u32 K, bool rolled, u32 n_tiles, cudaStream_t s) {
    if (n_tiles == 0) return;
    if (rolled) {
        switch (K) {
            case 21: hash_kmers_kernel<21, RAW><<<n_tiles, HASH_THREADS, 0, s>>>(a); break;
            case 31: hash_kmers_kernel<31, RAW><<<n_tiles, HASH_THREADS, 0, s>>>(a); break;
            default: hash_kmers_kernel<51, RAW><<<n_tiles, HASH_THREADS, 0, s>>>(a); break;
        }
    } else {
        hash_kmers_generic_kernel<RAW><<<n_tiles, 256, 0, s>>>(a, K);
    }
    count_launches(1);
}

bool k_has_rolled_kernel(uint32_t k) { return k == 21 || k == 31 || k == 51; }
int hash_threads() { return HASH_THREADS; }

static HashArgs make_hash_args(const HashLaunch& L, bool rolled, u32 tile_lo) {
    HashArgs a{};
    a.bases = L.bases; a.stream_off = L.stream_off; a.stream_len = L.stream_len;
    a.stream_row = L.stream_row;
    a.n_streams = L.n_streams; a.W = L.W; a.seed = L.seed; a.max_hash = L.max_hash;
    a.cand = L.cand; a.cand_off = L.cand_off; a.cand_cnt = L.cand_cnt;
    a.row_stride = L.row_stride; a.raw_out = nullptr;
    a.tile_start = rolled ? L.tile_start_rolled : L.tile_start_generic;
    a.tile_base = tile_lo;
    return a;
}

void launch_hash_kmers_k(const HashLaunch& L, uint32_t ksize, int row_index, cudaStream_t s) {
    launch_hash_kmers_range(L, ksize, row_index, 0, L.total_tiles_rolled, 0, L.total_tiles_generic, s);
}

void launch_hash_kmers_range(const HashLaunch& L, uint32_t ksize, int row_index, uint32_t tile_lo_r,
                             uint32_t tile_hi_r, uint32_t tile_lo_g, uint32_t tile_hi_g, cudaStream_t s) {
    const bool rolled = k_has_rolled_kernel(ksize);
    const u32 lo = rolled ? tile_lo_r : tile_lo_g, hi = rolled ? tile_hi_r : tile_hi_g;
    HashArgs a = make_hash_args(L, rolled, lo);
    a.row_index = row_index;
    launch_hash_one_k<false>(a, ksize, rolled, hi - lo, s);
}

// k = 21, 31, 51 requested together are hashed by the one-pass kernel (one read of the bases instead of three,
// identical sketches); SMB_SKETCH_FUSED=0 keeps the three launches for A/B runs.
bool sketch_fused_enabled() {
    const char* e = getenv("SMB_SKETCH_FUSED");
    return !(e && e[0] == '0');
}
// k = 21, 31, 51 in one launch over tiles [tile_lo, tile_hi) of the rolled tiling; row_index[i] / max_hash[i]
// belong to k = 21, 31, 51 in this order
void launch_hash_kmers_fused_range(const HashLaunch& L, const int row_index[3], const uint64_t max_hash[3],
                                   uint32_t tile_lo, uint32_t tile_hi, cudaStream_t s) {
    if (tile_hi <= tile_lo) return;
    FusedArgs f{};
    f.a = make_hash_args(L, true, tile_lo);
    for (int i = 0; i < 3; ++i) { f.row_index[i] = row_index[i]; f.max_hash[i] = max_hash[i]; }
    hash_kmers_fused_kernel<<<tile_hi - tile_lo, HASH_THREADS, 0, s>>>(f);
    count_launches(1);
}

void launch_window_hashes(const HashLaunch& L, uint32_t ksize, uint64_t* raw_out, cudaStream_t s) {
    const bool rolled = k_has_rolled_kernel(ksize);
    HashArgs a = make_hash_args(L, rolled, 0);
    a.stream_row = nullptr; a.row_stride = 1; a.row_index = 0; a.raw_out = raw_out;
    launch_hash_one_k<true>(a, ksize, rolled, rolled ? L.total_tiles_rolled : L.total_tiles_generic, s);
}

// ---------------------------------------------------------------------------------------
// Protein-family sketches (csrc/aa_kmers.cuh): residues, or DNA translated in six frames.
// One CTA = AA_TILE window starts.  The residue of every position of the tile (forward codon and
// reverse-complement codon for translated input) is computed once into shared memory; each
// thread then hashes its window from there (byte gathers at stride 1 or 3 are conflict free:
// consecutive threads read consecutive bytes).  Survivors are staged per CTA as in the DNA kernel.
// ---------------------------------------------------------------------------------------
static constexpr int AA_TABLE_BYTES = (sizeof(AaTables) + 15) & ~15;

template <bool RAW>
__global__ void __launch_bounds__(AA_TILE) hash_aa_kernel(HashArgs a, const AaTables* __restrict__ tabs,
                                                          u32 kaa, u32 translate, AaFrames F) {
    extern __shared__ __align__(16) unsigned char aa_smem[];
    __shared__ u64 s_buf[2 * AA_TILE];
    __shared__ u32 s_cnt, s_base;
    __shared__ int s_stream;
    const int tid = threadIdx.x;
    AaTables* T = reinterpret_cast<AaTables*>(aa_smem);
    const u32 stride = translate ? 3u : 1u;
    const u32 nst = aa_stage_len(kaa, stride);
    u8* sf = aa_smem + AA_TABLE_BYTES;
    u8* sr = sf + ((nst + 15u) & ~15u);
    for (u32 i = tid; i < sizeof(AaTables) / 4; i += AA_TILE)
        reinterpret_cast<u32*>(T)[i] = reinterpret_cast<const u32*>(tabs)[i];
    if (tid == 0) {
        s_cnt = 0;
        s_stream = find_stream(a.tile_start, a.n_streams, blockIdx.x + a.tile_base);
    }
    __syncthreads();
    const int stream = s_stream;
    const u64 L = a.stream_len[stream];
    const u8* __restrict__ seq = a.bases + a.stream_off[stream];
    const u64 span = (u64)kaa * stride;
    if (kaa == 0 || L < span) return;
    const u64 t0 = (u64)(blockIdx.x + a.tile_base - a.tile_start[stream]) * AA_TILE;
    if (t0 + span > L) return;                          // no window starts in this tile
    for (u32 i = tid; i < nst; i += AA_TILE) aa_stage(*T, translate != 0, seq, L, t0, i, sf, sr);
    __syncthreads();
    const u64 p = t0 + tid;
    const bool valid = p + span <= L;
    const int sk = a.stream_row ? (int)a.stream_row[stream] : stream;
    const int row = sk * a.row_stride + a.row_index;
    if (valid) {
        const u64 hf = aa_hash_fwd(sf, (u32)tid, kaa, stride, a.seed);
        u64 hr = 0;
        if (translate) hr = aa_hash_rev(sr, (u32)tid, kaa, a.seed);
        if (RAW) {
            if (translate) {
                a.raw_out[aa_raw_index(F, p, false)] = hf;
                a.raw_out[aa_raw_index(F, L - p - span, true)] = hr;
            } else {
                a.raw_out[p] = hf;
            }
        } else {
            if (hf != 0ull && hf <= a.max_hash) s_buf[atomicAdd(&s_cnt, 1u)] = hf;
            if (translate && hr != 0ull && hr <= a.max_hash) s_buf[atomicAdd(&s_cnt, 1u)] = hr;
        }
    }
    if (RAW) return;
    __syncthreads();
    const u32 n = s_cnt;
    if (n == 0) return;
    if (tid == 0) s_base = atomicAdd(&a.cand_cnt[row], n);
    __syncthreads();
    const u64 off = a.cand_off[row];
    const u64 capr = a.cand_off[row + 1] - off;
    for (u32 i = tid; i < n; i += AA_TILE) {
        u64 g = (u64)s_base + i;
        if (g < capr) a.cand[off + g] = s_buf[i];
    }
}

size_t aa_smem_bytes(uint32_t kaa, bool translate) {
    const u32 nst = aa_stage_len(kaa ? kaa : 1, translate ? 3u : 1u);
    return (size_t)AA_TABLE_BYTES + 2 * (size_t)((nst + 15u) & ~15u);
}
uint32_t aa_max_k(bool translate) {
    // both staging arrays must fit next to the tables in 200 KB of dynamic shared memory
    const size_t budget = 200 * 1024 - AA_TABLE_BYTES - 64;
    return (uint32_t)((budget / 2 - AA_TILE) / (translate ? 3 : 1));
}

template <bool RAW>
static void launch_hash_aa(HashArgs a, const AaTables* d_tables, u32 kaa, bool translate, AaFrames F,
                           u32 n_tiles, cudaStream_t s) {
    if (n_tiles == 0 || kaa == 0) return;
    const size_t smem = aa_smem_bytes(kaa, translate);
    cudaFuncSetAttribute(hash_aa_kernel<RAW>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    hash_aa_kernel<RAW><<<n_tiles, AA_TILE, smem, s>>>(a, d_tables, kaa, translate ? 1u : 0u, F);
    count_launches(1);
}

void launch_hash_aa_range(const HashLaunch& L, const AaTables* d_tables, uint32_t kaa, bool translate,
                          int row_index, uint32_t tile_lo, uint32_t tile_hi, cudaStream_t s) {
    HashArgs a = make_hash_args(L, false, tile_lo);
    a.row_index = row_index;
    launch_hash_aa<false>(a, d_tables, kaa, translate, AaFrames{}, tile_hi - tile_lo, s);
}

void launch_aa_window_hashes(const HashLaunch& L, const AaTables* d_tables, uint32_t kaa, bool translate,
                             uint64_t len, uint64_t* raw_out, cudaStream_t s) {
    HashArgs a = make_hash_args(L, false, 0);
    a.stream_row = nullptr; a.row_stride = 1; a.row_index = 0; a.raw_out = raw_out;
    launch_hash_aa<true>(a, d_tables, kaa, translate, aa_frames(len, kaa), L.total_tiles_generic, s);
}

// ---------------------------------------------------------------------------------------
// `sig kmers`: fused hash + probe over all records (kmer_match_kernels.cuh)
// ---------------------------------------------------------------------------------------
// The split table must leave room for two CTAs per SM next to the staging: keys (8 B each) up to 128 KB.
bool kmer_match_split_fits(uint64_t nq) { return nq <= 16382; }

template <int MODE, int K>
static void launch_match_t(const KmerMatchArgs& a, cudaStream_t s) {
    size_t smem = a.split ? match_split_smem(a.nq, a.nb) : 0;
    if (MODE >= 2) smem = ((smem + 15) & ~(size_t)15) + sizeof(AaTables);
    cudaFuncSetAttribute(kmer_match_kernel<MODE, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const size_t per_cta = smem + (size_t)MATCH_STAGE * 16 + 1024;
    u64 ctas_per_sm = (u64)(220 * 1024) / per_cta;
    ctas_per_sm = ctas_per_sm < 1 ? 1 : ctas_per_sm > 4 ? 4 : ctas_per_sm;
    u64 blocks = (a.n_chunks + MATCH_THREADS - 1) / MATCH_THREADS;
    if (blocks > (u64)SMB_SMS * ctas_per_sm) blocks = (u64)SMB_SMS * ctas_per_sm;
    kmer_match_kernel<MODE, K><<<(unsigned)blocks, MATCH_THREADS, smem, s>>>(a);
    count_launches(1);
}

void launch_kmer_match(const KmerMatchArgs& a, cudaStream_t s) {
    if (a.n_chunks == 0) return;
    switch (a.mode) {
        case 0:
            if (a.K == 21) launch_match_t<0, 21>(a, s);
            else if (a.K == 31) launch_match_t<0, 31>(a, s);
            else launch_match_t<0, 51>(a, s);
            break;
        case 1: launch_match_t<1, 0>(a, s); break;
        case 2: launch_match_t<2, 0>(a, s); break;
        default: launch_match_t<3, 0>(a, s); break;
    }
}

cudaError_t sort_kmer_matches(const u64* keys, const u64* hashes, u64* keys_out, u64* hashes_out, u64 m, int end_bit,
                              cudaStream_t s) {
    size_t temp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys, keys_out, hashes, hashes_out, (long long)m, 0, end_bit, s);
    void* temp = nullptr;
    cudaError_t e = cudaMallocAsync(&temp, temp_bytes ? temp_bytes : 16, s);
    if (e != cudaSuccess) return e;
    e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_out, hashes, hashes_out, (long long)m, 0, end_bit, s);
    cudaFreeAsync(temp, s);
    return e != cudaSuccess ? e : cudaGetLastError();
}

void launch_match_mark_found(const u64* keys, const u64* hashes, u64 n, const u8* skip, const u64* q, u64 nq, u8* flag,
                             cudaStream_t s) {
    if (n == 0 || nq == 0) return;
    u64 blocks = (n + 255) / 256;
    if (blocks > (u64)SMB_SMS * 16) blocks = (u64)SMB_SMS * 16;
    match_mark_found_kernel<<<(unsigned)blocks, 256, 0, s>>>(keys, hashes, n, skip, q, nq, flag); count_launches(1);
}

void launch_match_num_common(const u64* bh, const u64* boff, const u32* recs, int n, const u64* q, u64 nq, u32 num,
                             const u8* skip, u8* rec_hit, u8* flag, cudaStream_t s) {
    if (n <= 0) return;
    match_num_common_kernel<<<(n + 255) / 256, 256, 0, s>>>(bh, boff, recs, n, q, nq, num, skip, rec_hit, flag); count_launches(1);
}

// ---------------------------------------------------------------------------------------
// first invalid base of a sequence (force == false path: signature.rs:271-279)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) first_invalid_kernel(const u8* __restrict__ b, u64 len,
                                                           unsigned long long* __restrict__ d_pos) {
    unsigned long long best = ~0ull;
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < len; p += (u64)gridDim.x * blockDim.x) {
        if (!valid_base(up_byte(b[p]))) { best = p; break; }      // positions ascend per thread
    }
    for (int d = 16; d; d >>= 1) {
        unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
        best = o < best ? o : best;
    }
    if (lane_id() == 0 && best != ~0ull) atomicMin(d_pos, best);
}

void launch_first_invalid(const u8* bases, u64 len, unsigned long long* d_pos, cudaStream_t s) {
    cudaMemsetAsync(d_pos, 0xff, sizeof(unsigned long long), s);
    if (len == 0) return;
    u64 blocks = (len + 255) / 256;
    if (blocks > (u64)SMB_SMS * 8) blocks = (u64)SMB_SMS * 8;
    first_invalid_kernel<<<(unsigned)blocks, 256, 0, s>>>(bases, len, d_pos); count_launches(1);
}

// ---------------------------------------------------------------------------------------
// row materialisation: sort + unique (+ run lengths) of each row's candidates
// ---------------------------------------------------------------------------------------


// unique (+ run lengths) of an already sorted row, in place; single block.

int sort_small_max() { return SORT_MAX; }

// murmur3 of an arbitrary byte string, single thread (hash_murmur / add_word utility)
__global__ void murmur_bytes_kernel(const u8* __restrict__ d, u64 len, u64 seed, u64* __restrict__ out) {
    u64 h1 = seed, h2 = seed;
    const u64 nblk = len / 16;
    for (u64 b = 0; b < nblk; ++b) {
        u64 k1 = 0, k2 = 0;
        for (int i = 7; i >= 0; --i) { k1 = (k1 << 8) | d[16 * b + i]; k2 = (k2 << 8) | d[16 * b + 8 + i]; }
        k1 *= SMB_C1; k1 = smb_rotl64(k1, 31); k1 *= SMB_C2; h1 ^= k1;
        h1 = smb_rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729ULL;
        k2 *= SMB_C2; k2 = smb_rotl64(k2, 33); k2 *= SMB_C1; h2 ^= k2;
        h2 = smb_rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5ULL;
    }
    const u64 tail = len & 15, tb = 16 * nblk;
    if (tail > 8) {
        u64 k2 = 0;
        for (u64 i = tail; i > 8; --i) k2 = (k2 << 8) | d[tb + i - 1];
        k2 *= SMB_C2; k2 = smb_rotl64(k2, 33); k2 *= SMB_C1; h2 ^= k2;
    }
    if (tail > 0) {
        u64 k1 = 0;
        for (u64 i = tail < 8 ? tail : 8; i > 0; --i) k1 = (k1 << 8) | d[tb + i - 1];
        k1 *= SMB_C1; k1 = smb_rotl64(k1, 31); k1 *= SMB_C2; h1 ^= k1;
    }
    h1 ^= len; h2 ^= len;
    h1 += h2; h2 += h1;
    h1 = smb_fmix64(h1); h2 = smb_fmix64(h2);
    *out = h1 + h2;
}
void launch_murmur_bytes(const u8* data, u64 len, u64 seed, u64* d_out, cudaStream_t s) {
    murmur_bytes_kernel<<<1, 1, 0, s>>>(data, len, seed, d_out); count_launches(1);
}

// angular similarity terms -- single block; rows are sketches with abundances
__global__ void __launch_bounds__(1024) angular_terms_kernel(
    const u64* __restrict__ a, const u64* __restrict__ aa, u64 na, const u64* __restrict__ b,
    const u64* __restrict__ ba, u64 nb, unsigned long long* __restrict__ out) {
    unsigned long long prod = 0, asq = 0, bsq = 0;
    for (u64 i = threadIdx.x; i < na; i += blockDim.x) {
        u64 x = a[i], ab = aa[i];
        asq += ab * ab;
        u64 lo = 0, hi = nb;
        while (lo < hi) { u64 mid = (lo + hi) >> 1; if (b[mid] < x) lo = mid + 1; else hi = mid; }
        if (lo < nb && b[lo] == x) prod += ab * ba[lo];
    }
    for (u64 j = threadIdx.x; j < nb; j += blockDim.x) bsq += ba[j] * ba[j];
    for (int d = 16; d; d >>= 1) {
        prod += __shfl_xor_sync(0xffffffffu, prod, d);
        asq += __shfl_xor_sync(0xffffffffu, asq, d);
        bsq += __shfl_xor_sync(0xffffffffu, bsq, d);
    }
    if (lane_id() == 0) { atomicAdd(out + 0, prod); atomicAdd(out + 1, asq); atomicAdd(out + 2, bsq); }
}
void launch_angular_terms(const u64* a, const u64* aa, u64 na, const u64* b, const u64* ba, u64 nb,
                          unsigned long long* d_out, cudaStream_t s) {
    cudaMemsetAsync(d_out, 0, 3 * sizeof(unsigned long long), s);
    angular_terms_kernel<<<1, 1024, 0, s>>>(a, aa, na, b, ba, nb, d_out); count_launches(1);
}

__global__ void __launch_bounds__(256) row_prefix_counts_kernel(const u64* __restrict__ h,
                                                               const u64* __restrict__ off, int n_rows,
                                                               u64 max_hash, u32* __restrict__ out) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const u64* row = h + off[r];
    u64 lo = 0, hi = off[r + 1] - off[r];
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (row[mid] <= max_hash) lo = mid + 1; else hi = mid; }
    out[r] = (u32)lo;
}
void launch_row_prefix_counts(const u64* h, const u64* off, int n_rows, u64 max_hash, u32* out_cnt,
                              cudaStream_t s) {
    if (n_rows <= 0) return;
    row_prefix_counts_kernel<<<(n_rows + 255) / 256, 256, 0, s>>>(h, off, n_rows, max_hash, out_cnt); count_launches(1);
}

void launch_sort_unique_small(u64* cand, const u64* cand_off, const u32* cand_cnt, int n_rows,
                              u32* out_cnt, u64* abund, cudaStream_t s) {
    if (n_rows <= 0) return;
    size_t smem = (size_t)SORT_MAX * 8 + (size_t)SORT_MAX * 4;
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(sort_unique_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        configured = true;
    }
    sort_unique_small_kernel<<<n_rows, SORT_THREADS, smem, s>>>(cand, cand_off, cand_cnt, out_cnt, abund); count_launches(1);
}

// Big row: CUB radix sort into scratch, then unique back into the row.  scratch must hold
// 2*n u64 (+ CUB temp, allocated here with cudaMallocAsync).
cudaError_t sort_unique_big_row(u64* row, u64 n, u64* scratch_sorted, u64* scratch_heads,
                                u64* abund_row, u32* d_out_cnt, cudaStream_t s) {
    size_t temp_bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, row, scratch_sorted, (long long)n, 0, 64, s);
    void* temp = nullptr;
    cudaError_t e = cudaMallocAsync(&temp, temp_bytes ? temp_bytes : 16, s);
    if (e != cudaSuccess) return e;
    cub::DeviceRadixSort::SortKeys(temp, temp_bytes, row, scratch_sorted, (long long)n, 0, 64, s);
    unique_sorted_row_kernel<<<1, SORT_THREADS, 0, s>>>(scratch_sorted, n, row, abund_row, scratch_heads, d_out_cnt); count_launches(1);
    cudaFreeAsync(temp, s);
    return cudaGetLastError();
}

// gather rows into a dense CSR buffer: dst[dst_off[r] + i] = src[src_off[r] + i], i < cnt[r]
__global__ void __launch_bounds__(256) compact_rows_kernel(const u64* __restrict__ src,
                                                          const u64* __restrict__ src_off,
                                                          const u32* __restrict__ cnt,
                                                          const u64* __restrict__ dst_off,
                                                          u64* __restrict__ dst) {
    const int r = blockIdx.x;
    const u64 so = src_off[r], d0 = dst_off[r];
    const u32 n = cnt[r];
    for (u32 i = threadIdx.x + blockIdx.y * blockDim.x; i < n; i += blockDim.x * gridDim.y)
        dst[d0 + i] = src[so + i];
}

void launch_compact_rows(const u64* src, const u64* src_off, const u32* cnt, const u64* dst_off,
                         u64* dst, int n_rows, cudaStream_t s) {
    if (n_rows <= 0) return;
    dim3 grid(n_rows, 4);
    compact_rows_kernel<<<grid, 256, 0, s>>>(src, src_off, cnt, dst_off, dst); count_launches(1);
}

}  // namespace smb
