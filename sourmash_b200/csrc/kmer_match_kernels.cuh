// kmer_match_kernels.cuh -- `sig kmers` on the device: hash every window of every record, keep the windows whose hash
// is in a query hash set Q, and emit (key = record << 32 | ordinal, hash) for each of them.  Included from
// sketch_kernels.cu, which keeps the launchers (launch_kmer_match, ...).
//
// Replaces the per-record loop of the reference's `sig kmers` (src/sourmash/sig/__main__.py:1206-1256): a fresh sketch
// per record, add_sequence / add_protein, intersection with the merged query, kmers_and_hashes + a set lookup per k-mer.
//
// Work mapping.  The sketch kernels give every CTA a tile of ONE stream; on 150 bp reads that leaves most of a CTA
// idle.  Here a record is cut into chunks of W windows (DNA) or W window starts (protein family), chunk_start[] is the
// prefix of the chunks of all records, and thread t of a block of chunks owns chunk blockbase + t, whichever record
// it falls in (one binary search over chunk_start per chunk).  A chunk never leaves its record, so no window straddles
// two records.  The grid is persistent: each CTA builds the probe table once and then walks blocks of chunks.
//
// Hashing is the sketch path's: the register-rolling kmer_roll.cuh kernels for k = 21, 31, 51 (hash_thread_windows),
// dna_window_hash (sketch_kernels.cu) for any other k, the aa_kmers.cuh functions for residues and for six-frame
// translation.  A DNA window counts when its k bases are all valid (add_sequence(seq, force=True)).
//
// Probe.  Only windows with 0 < h <= max_hash are probed (about 1/scaled of them; a num sketch probes every valid
// window).  Q sorted-unique; UINT64_MAX is answered by a flag, keys above the largest other key by a compare.  Small Q:
// a shared-memory split table per CTA (split_table.cuh).  Larger Q: the global bucket directory + L2 occupancy bitmap of
// the one-vs-many search (search_kernels.cuh, built by launch_build_global_dir / launch_build_query_bitmap).
//
// Output.  Matches are staged per CTA in shared memory and flushed with one global atomicAdd per CTA and block of
// chunks; when the staging is full a thread appends directly.  The global count always advances, so a run whose
// matches overflow the buffer tells the host the exact size for the second run.
#pragma once
#include "common.cuh"
#include "kmer_roll.cuh"
#include "aa_kmers.cuh"
#include "split_table.cuh"
#include "sketch_device.cuh"
#include "kernels.h"

namespace smb {

static constexpr int MATCH_THREADS = 256;
static constexpr int MATCH_STAGE = 512;         // staged matches per CTA (key + hash: 8 KB)

__host__ __device__ __forceinline__ size_t match_split_smem(u64 nq, u64 nb) {
    return (size_t)(nq + 2) * 8 + (size_t)(nb + 2) * 2;
}

__device__ __forceinline__ bool match_probe(const KmerMatchArgs& a, const SplitTable& t, u64 h) {
    if (h == SMB_U64_MAX) return a.q_has_max != 0;
    if (a.nq == 0 || h > a.q_top) return false;        // (h >> shift) < nb from here on
    if (a.split) return (split_probe_verify(t, h, a.shift) | split_probe_rest(t, h, a.shift)) != 0u;
    const u32 bm_shift = a.shift >= (u32)a.fine_log2 ? a.shift - (u32)a.fine_log2 : 0u;
    const u64 bit = h >> bm_shift;
    if (!((__ldg(a.bitmap + (bit >> 5)) >> (bit & 31)) & 1u)) return false;
    const u64 b = h >> a.shift;
    for (u64 p = a.gdir[b], pe = a.gdir[b + 1]; p < pe; ++p) {
        const u64 k = ld_nc_u64(a.q + p);
        if (k >= h) return k == h;
    }
    return false;
}

__device__ __forceinline__ int match_find_record(const u64* __restrict__ chunk_start, int n_rec, u64 c) {
    int lo = 0, hi = n_rec;                            // last record with chunk_start <= c
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (chunk_start[mid] <= c) lo = mid; else hi = mid; }
    return lo;
}

// any DNA k, one window: the bytes straight from global / L1 (defined in sketch_kernels.cu)
__device__ __forceinline__ u64 dna_window_hash(const u8* __restrict__ base, u64 w, u32 K, u64 seed, bool& valid);

// residue of the forward (rev = false) or reverse-complement codon at DNA position pos (aa_translate_at, one strand)
__device__ __forceinline__ u32 match_codon(const AaTables& T, const u8* __restrict__ seq, u64 L, u64 pos, bool rev) {
    const u32 c0 = pos < L ? T.base_code[seq[pos]] : 5u;
    const u32 c1 = pos + 1 < L ? T.base_code[seq[pos + 1]] : 5u;
    const u32 c2 = pos + 2 < L ? T.base_code[seq[pos + 2]] : 5u;
    return rev ? T.codon[aa_comp_code(c2) * 36u + aa_comp_code(c1) * 6u + aa_comp_code(c0)] : T.codon[c0 * 36u + c1 * 6u + c2];
}

// aa_raw_index (seq_to_hashes order of translated windows) with the frame sizes computed in place: an AaFrames table
// indexed by frame would live in local memory.  q = window start on its own strand, L >= 3 * kaa.
__device__ __forceinline__ u64 match_aa_ordinal(u64 L, u32 kaa, u64 q, bool reverse) {
    auto nwin = [&](u32 f) -> u64 { const u64 na = (L - f) / 3; return na >= kaa ? na - kaa + 1 : 0; };
    const u32 f = (u32)(q % 3);
    const u64 n0 = nwin(0), n1 = nwin(1);
    const u64 base = f == 0 ? 0 : f == 1 ? 2 * n0 : 2 * (n0 + n1);
    return base + (reverse ? (f == 0 ? n0 : f == 1 ? n1 : nwin(2)) : 0) + q / 3;
}

template <int MODE, int K>
__global__ void __launch_bounds__(MATCH_THREADS) kmer_match_kernel(KmerMatchArgs a) {
    SMB_DYN_SHARED(unsigned char, smem_raw);
    SMB_SHARED u64 s_key[MATCH_STAGE];
    SMB_SHARED u64 s_hash[MATCH_STAGE];
    SMB_SHARED u32 s_cnt;
    SMB_SHARED unsigned long long s_base;
    const int tid = threadIdx.x;
    // dynamic shared memory: the split table of Q (when Q is small), then the AA tables (protein family)
    u32* lo_w = reinterpret_cast<u32*>(smem_raw);
    const int kstride = a.split ? (int)a.nq + 2 : 0;
    u32* hi_w = lo_w + kstride;
    u16* dir = reinterpret_cast<u16*>(smem_raw + (size_t)kstride * 8);
    SplitTable tab;
    tab.lo = lo_w; tab.hi = hi_w; tab.dir = dir;
    AaTables* T = nullptr;
    if constexpr (MODE >= 2) {
        const size_t t_off = a.split ? (match_split_smem(a.nq, a.nb) + 15) & ~(size_t)15 : 0;
        T = reinterpret_cast<AaTables*>(smem_raw + t_off);
        for (u32 i = tid; i < sizeof(AaTables) / 4; i += MATCH_THREADS)
            reinterpret_cast<u32*>(T)[i] = reinterpret_cast<const u32*>(a.tabs)[i];
    }
    if (a.split) {
        split_table_load(lo_w, hi_w, dir, a.q, (int)a.nq, (int)a.nb, tid, MATCH_THREADS);
        __syncthreads();
        split_table_heads(lo_w, hi_w, dir, (int)a.nq, a.shift, tid, MATCH_THREADS);
        __syncthreads();
        split_table_flags(dir, (int)a.nb, tid, MATCH_THREADS);
    }
    if (tid == 0) s_cnt = 0;
    __syncthreads();

    for (u64 blk = blockIdx.x; blk * MATCH_THREADS < a.n_chunks; blk += gridDim.x) {
        const u64 c = blk * MATCH_THREADS + tid;
        if (c < a.n_chunks) {
            const int r = match_find_record(a.chunk_start, a.n_rec, c);
            const u64 s0 = a.rec_off[r], L = a.rec_len[r];
            const u64 first = (c - a.chunk_start[r]) * (u64)a.W;
            auto emit = [&](u64 ordinal, u64 h) {
                if (h == 0ull || h > a.max_hash || !match_probe(a, tab, h)) return;
                a.rec_hit[r] = 1;
                const u64 key = ((u64)r << 32) | ordinal;
                const u32 slot = atomicAdd(&s_cnt, 1u);
                if (slot < MATCH_STAGE) {
                    s_key[slot] = key; s_hash[slot] = h;
                } else {                                   // staging full: append directly
                    const unsigned long long g = atomicAdd(a.count, 1ull);
                    if (g < a.cap) { a.keys[g] = key; a.hashes[g] = h; }
                }
            };
            if constexpr (MODE == 0) {
                // aligned coordinates, as in hash_kmers_kernel: the stream starts `lead` bytes into its 16-byte line
                const u64 b0 = s0 & ~15ull;
                const u32 lead = (u32)(s0 - b0);
                const u64 Lp = (u64)lead + L;
                hash_thread_windows<K>(a.bases + b0, Lp, lead, first, a.W, a.seed, [&](u64 w, bool valid, u64 h) {
                    if (w < lead || w + K > Lp) return;
                    if (!valid) { if (a.rec_invalid) a.rec_invalid[r] = 1; return; }
                    emit(w - lead, h);
                });
            } else if constexpr (MODE == 1) {
                const u64 nwin = L >= a.K ? L - a.K + 1 : 0;
                const u64 end = first + (u64)a.W < nwin ? first + (u64)a.W : nwin;
                for (u64 w = first; w < end; ++w) {
                    bool valid;
                    const u64 h = dna_window_hash(a.bases + s0, w, a.K, a.seed, valid);
                    if (!valid) { if (a.rec_invalid) a.rec_invalid[r] = 1; continue; }
                    emit(w, h);
                }
            } else {
                const u8* __restrict__ seq = a.bases + s0;
                const u32 kaa = a.K, stride = MODE == 3 ? 3u : 1u;
                const u64 span = (u64)kaa * stride;
                const u64 nstart = L >= span ? L - span + 1 : 0;
                const u64 end = first + (u64)a.W < nstart ? first + (u64)a.W : nstart;
                for (u64 p = first; p < end; ++p) {
                    if constexpr (MODE == 2) {
                        emit(p, murmur_at(kaa, a.seed, [&](u32 t) -> u32 { return T->residue[seq[p + t]]; }));
                    } else {
                        for (int rev = 0; rev < 2; ++rev) {    // one call site of emit: it stays inlined
                            const u64 h = murmur_at(kaa, a.seed, [&](u32 t) -> u32 {
                                return match_codon(*T, seq, L, p + 3ull * (rev ? kaa - 1u - t : t), rev != 0); });
                            emit(match_aa_ordinal(L, kaa, rev ? L - p - span : p, rev != 0), h);
                        }
                    }
                }
            }
        }
        __syncthreads();
        const u32 n = min(s_cnt, (u32)MATCH_STAGE);
        if (n) {
            if (tid == 0) s_base = atomicAdd(a.count, (unsigned long long)n);
            __syncthreads();
            for (u32 i = tid; i < n; i += MATCH_THREADS) {
                const u64 g = (u64)s_base + i;
                if (g < a.cap) { a.keys[g] = s_key[i]; a.hashes[g] = s_hash[i]; }
            }
        }
        __syncthreads();
        if (tid == 0) s_cnt = 0;
        __syncthreads();
    }
}

// Found hashes of a scaled query: flag[i] = 1 for every Q key some match holds, matches of skipped records
// (skip[record] != 0, nullable) left out.
__global__ void __launch_bounds__(256) match_mark_found_kernel(const u64* __restrict__ keys, const u64* __restrict__ hashes,
                                                              u64 n, const u8* __restrict__ skip,
                                                              const u64* __restrict__ q, u64 nq, u8* __restrict__ flag) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (u64)gridDim.x * blockDim.x) {
        if (skip && skip[keys[e] >> 32]) continue;
        const u64 x = hashes[e];
        u64 lo = 0, hi = nq;
        while (lo < hi) { const u64 mid = (lo + hi) >> 1; if (ld_nc_u64(q + mid) < x) lo = mid + 1; else hi = mid; }
        if (lo < nq && ld_nc_u64(q + lo) == x) flag[lo] = 1;
    }
}

// Num sketches (kmerminhash_intersection, minhash.rs:560-589): the common hashes of a record are those of its
// bottom-num sketch B that are in Q and among the first `num` of B ∪ Q.  One thread per record with a probe hit merges
// B and Q in ascending order; the record passes when a common hash has union rank < num.  flag[i] = 1 for every Q key
// that is common for some passing record that is not skipped (found_mh += seq_mh.intersection(query_mh)).
__global__ void __launch_bounds__(256) match_num_common_kernel(const u64* __restrict__ bh, const u64* __restrict__ boff,
                                                              const u32* __restrict__ recs, int n,
                                                              const u64* __restrict__ q, u64 nq, u32 num,
                                                              const u8* __restrict__ skip, u8* __restrict__ rec_hit,
                                                              u8* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u64* b = bh + boff[i];
    const u64 nbk = boff[i + 1] - boff[i];
    u64 x = 0, y = 0, rank = 0;
    bool pass = false;
    const bool keep = !(skip && skip[recs[i]]);
    while (rank < num && (x < nbk || y < nq)) {
        const u64 vb = x < nbk ? b[x] : SMB_U64_MAX, vq = y < nq ? ld_nc_u64(q + y) : SMB_U64_MAX;
        if (x < nbk && y < nq && vb == vq) { pass = true; if (keep) flag[y] = 1; ++x; ++y; }
        else if (y >= nq || (x < nbk && vb < vq)) ++x;
        else ++y;
        ++rank;
    }
    rec_hit[recs[i]] = pass ? 1 : 0;
}

}  // namespace smb
