// lca_kernels.cuh -- the lowest common ancestor of every database hash, and per-query counts of those ancestors
// (`sourmash lca classify` / `lca summarize`).  compare_kernels.cu launches them (lca_table_build, lca_counts).
//
// The reference finds, for every query hash, the lineages of every database holding it (gather_assignments,
// src/sourmash/lca/lca_utils.py:186-199), builds a dictionary tree of them and walks it down to the first node with
// several children or to its only leaf (count_lca_for_assignments, :202-225): one Python tree per query hash.  That
// answer depends on the databases alone, so here it is computed once per command for every database hash:
//
//   table build  the (hash, trie node) pairs of all databases are radix-sorted by hash; one thread per run of equal
//                hashes folds the run's nodes into its LCA node (lca_fold_kernel); a scan and a scatter compact the
//                distinct hashes into a sorted hash[] with a parallel lca[].
//   counts       one thread per query element binary-searches the table; a hit becomes the key (query << 32 | lca)
//                with its element index as the value, a miss the key (n_queries << 32), which sorts after every hit.
//                A stable sort of those pairs makes every (query, node) one run with its elements ascending; one
//                thread per run head sums the run's weights and takes its first element (lca_count_runs_kernel).
//
// The fold follows the tree walk, not the textbook LCA: the walk descends while a node has exactly one child, so
// lineages that lie on one root path (a;b and a;b;c) give the deepest of them, and only lineages that branch give
// the branch point.  The state of a fold is a node and whether the lineages seen so far branch; a node that is an
// ancestor or a descendant of the state's node keeps a branched state as it is.  Trie depth is at most 8 ranks, so
// every ancestor test is a climb of at most 8 steps.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace smb {

__device__ __forceinline__ u32 lca_climb(const u32* __restrict__ parent, const u8* __restrict__ depth, u32 a, u32 d) {
    while (depth[a] > d) a = parent[a];
    return a;
}

// the common ancestor of trie nodes a and b (the root, node 0, is everyone's)
__device__ __forceinline__ u32 lca_pair(const u32* __restrict__ parent, const u8* __restrict__ depth, u32 a, u32 b) {
    const u32 da = depth[a], db = depth[b];
    if (da > db) a = lca_climb(parent, depth, a, db);
    else b = lca_climb(parent, depth, b, da);
    while (a != b) { a = parent[a]; b = parent[b]; }
    return a;
}

// keys / nodes: the (hash, node) pairs sorted by hash.  For every run head i whose hash is <= max_hash and whose run
// holds a node other than LCA_NO_NODE: flag[i] = 1 and lca[i] = the run's LCA node.  Every other flag is 0.
__global__ void __launch_bounds__(256) lca_fold_kernel(const u64* __restrict__ keys, const u32* __restrict__ nodes,
                                                       u64 T, u64 max_hash, const u32* __restrict__ parent,
                                                       const u8* __restrict__ depth, u32* __restrict__ flag,
                                                       u32* __restrict__ lca) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (u64)gridDim.x * blockDim.x) {
        const u64 k = keys[i];
        flag[i] = 0;
        if ((i > 0 && keys[i - 1] == k) || k > max_hash) continue;
        u32 cur = LCA_NO_NODE;
        bool branched = false;
        for (u64 j = i; j < T && keys[j] == k; ++j) {
            const u32 y = nodes[j];
            if (y == LCA_NO_NODE) continue;
            if (cur == LCA_NO_NODE) { cur = y; continue; }
            const u32 l = lca_pair(parent, depth, cur, y);
            if (l == y) continue;                             // y lies above cur: nothing changes
            if (l == cur) { if (!branched) cur = y; continue; }   // y lies below: a chain goes deeper
            cur = l;                                          // y branches off
            branched = true;
        }
        if (cur != LCA_NO_NODE) { flag[i] = 1; lca[i] = cur; }
    }
}

// pos = exclusive scan of flag: kept run heads go to out_h[pos[i]] / out_lca[pos[i]]; *count = the number kept
__global__ void __launch_bounds__(256) lca_scatter_kernel(const u64* __restrict__ keys, const u32* __restrict__ lca,
                                                          const u32* __restrict__ flag, const u32* __restrict__ pos,
                                                          u64 T, u64* __restrict__ out_h, u32* __restrict__ out_lca,
                                                          unsigned long long* __restrict__ count) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (u64)gridDim.x * blockDim.x) {
        if (flag[i]) {
            out_h[pos[i]] = keys[i];
            out_lca[pos[i]] = lca[i];
        }
        if (i == T - 1) *count = (unsigned long long)pos[i] + flag[i];
    }
}

// One thread per query element e of the CSR (q_off: n_q + 1 offsets): key[e] = (query << 32) | lca of its hash when
// the table holds the hash, else n_q << 32; idx[e] = e.  The table is searched by exact comparison, so any hash value,
// UINT64_MAX included, is found or missed on its own.
__global__ void __launch_bounds__(256) lca_probe_kernel(const u64* __restrict__ qh, const u64* __restrict__ q_off,
                                                        u32 n_q, u64 Tq, const u64* __restrict__ t_h,
                                                        const u32* __restrict__ t_lca, u64 n_t, u64* __restrict__ key,
                                                        u32* __restrict__ idx) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < Tq; e += (u64)gridDim.x * blockDim.x) {
        u32 lo = 0, hi = n_q;                                  // the query: last q with q_off[q] <= e
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (q_off[mid] <= e) lo = mid; else hi = mid;
        }
        const u64 h = qh[e];
        u64 a = 0, b = n_t;                                    // first table entry >= h
        while (a < b) {
            const u64 mid = (a + b) >> 1;
            if (t_h[mid] < h) a = mid + 1; else b = mid;
        }
        key[e] = (a < n_t && t_h[a] == h) ? ((u64)lo << 32 | t_lca[a]) : ((u64)n_q << 32);
        idx[e] = (u32)e;
    }
}

// keys / idx: the probe's pairs sorted by key, stably.  For every run head i of a hit: flag[i] = 1, weight[i] = the
// sum over the run of abund[idx] (1 per element without abund), and the run's first element is idx[i].
__global__ void __launch_bounds__(256) lca_count_runs_kernel(const u64* __restrict__ keys, const u32* __restrict__ idx,
                                                             u64 Tq, u64 miss_key, const u64* __restrict__ abund,
                                                             u32* __restrict__ flag, u64* __restrict__ weight) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < Tq; i += (u64)gridDim.x * blockDim.x) {
        const u64 k = keys[i];
        flag[i] = 0;
        if ((i > 0 && keys[i - 1] == k) || k == miss_key) continue;
        u64 sum = 0;
        for (u64 j = i; j < Tq && keys[j] == k; ++j) sum += abund ? abund[idx[j]] : 1;
        flag[i] = 1;
        weight[i] = sum;
    }
}

// pos = exclusive scan of flag: row pos[i] = (query, node, weight, first element - the query's first offset)
__global__ void __launch_bounds__(256) lca_count_scatter_kernel(const u64* __restrict__ keys, const u32* __restrict__ idx,
                                                                const u64* __restrict__ weight,
                                                                const u32* __restrict__ flag, const u32* __restrict__ pos,
                                                                u64 Tq, const u64* __restrict__ q_off,
                                                                u32* __restrict__ out_q, u32* __restrict__ out_node,
                                                                u64* __restrict__ out_w, u64* __restrict__ out_first,
                                                                unsigned long long* __restrict__ count) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < Tq; i += (u64)gridDim.x * blockDim.x) {
        if (flag[i]) {
            const u32 q = (u32)(keys[i] >> 32);
            const u32 p = pos[i];
            out_q[p] = q;
            out_node[p] = (u32)keys[i];
            out_w[p] = weight[i];
            out_first[p] = idx[i] - q_off[q];
        }
        if (i == Tq - 1) *count = (unsigned long long)pos[i] + flag[i];
    }
}

}  // namespace smb
