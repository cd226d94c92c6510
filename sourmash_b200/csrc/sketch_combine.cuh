// sketch_combine.cuh -- union, intersection and difference of all rows of a resident set in one sorted pass
// (`sig merge`, `sig intersect`, `sig subtract`).  compare_kernels.cu launches them (sketchset_combine).
//
// The reference merges n sketches with one KmerMinHash::merge per sketch (src/core/src/sketch/minhash.rs:432-516),
// each a fresh vector of the running union: O(n |union|) element moves.  `sig intersect` / `sig subtract` build
// Python sets of every hash (src/sourmash/sig/__main__.py:526-712).  Here the (hash, element index) pairs of the
// whole set are radix-sorted once, stably, so that every distinct hash h is one run of m(h) elements with its rows
// ascending (rows are sets: m(h) = the number of rows holding h).  One thread per run head then decides the run and
// sums its abundances, and an exclusive scan of the keep flags compacts the kept runs in hash order.
//
//   op           keeps h when                          value
//   UNION        always                                sum of the run's abundances (sets with abundances)
//   ALL          m(h) = n_rows                         -
//   FIRST_ONLY   m(h) = 1 and the element is in row 0  -
//
// A run is walked by its head thread alone.  Runs are as long as the number of rows holding the hash (10^4 for
// 10^4 copies of one genome); the walk is sequential but correct at any length.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace smb {

__global__ void __launch_bounds__(256) combine_iota_kernel(u32* __restrict__ idx, u64 T) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (u64)gridDim.x * blockDim.x) idx[i] = (u32)i;
}

// keys / idx: the sorted (hash, element index) stream of T elements.  For every run head i: flag[i] = 1 when the op
// keeps the run, and (abund != null) val[i] = the sum of abund[idx[j]] over the run.  Every other flag is 0.
// row0_end = offsets[1]: element indices below it lie in row 0, and the stable sort puts row 0's element first.
__global__ void __launch_bounds__(256) combine_runs_kernel(const u64* __restrict__ keys, const u32* __restrict__ idx,
                                                           u64 T, const u64* __restrict__ abund, u32 op, u64 n_rows,
                                                           u64 row0_end, u32* __restrict__ flag, u64* __restrict__ val) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (u64)gridDim.x * blockDim.x) {
        const u64 k = keys[i];
        if (i > 0 && keys[i - 1] == k) { flag[i] = 0; continue; }
        u64 j = i + 1;
        u64 sum = abund ? abund[idx[i]] : 0;
        while (j < T && keys[j] == k) {
            if (abund) sum += abund[idx[j]];
            ++j;
        }
        const u64 m = j - i;
        bool keep = true;
        if (op == COMBINE_ALL) keep = m == n_rows;
        else if (op == COMBINE_FIRST_ONLY) keep = m == 1 && idx[i] < row0_end;
        flag[i] = keep ? 1u : 0u;
        if (val) val[i] = sum;
    }
}

// pos = exclusive scan of flag: kept run heads go to out_h[pos[i]] (and out_v from val); *count = the number kept
__global__ void __launch_bounds__(256) combine_scatter_kernel(const u64* __restrict__ keys, const u64* __restrict__ val,
                                                              const u32* __restrict__ flag, const u32* __restrict__ pos,
                                                              u64 T, u64* __restrict__ out_h, u64* __restrict__ out_v,
                                                              unsigned long long* __restrict__ count) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (u64)gridDim.x * blockDim.x) {
        if (flag[i]) {
            out_h[pos[i]] = keys[i];
            if (out_v) out_v[pos[i]] = val[i];
        }
        if (i == T - 1) *count = (unsigned long long)pos[i] + flag[i];
    }
}

}  // namespace smb
