// lca_kernels.cuh -- the lowest common ancestor of every database hash, and per-query counts of those ancestors
// (`sourmash lca classify` / `lca summarize`), and the database build (`lca index`, below).  compare_kernels.cu
// launches them (lca_table_build, lca_counts, lca_index_build).
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

// ------------------------------------------------------------------------------------------------------------------
// The database build (`sourmash lca index`, lca_index_build in compare_kernels.cu).  The reference inserts one
// (hash, idx) pair at a time into a dict of sets (LCA_Database.insert, src/sourmash/lca/lca_db.py:145-205) and
// json.dumps the dict (save_to_json, :420-465).  Here the input is the resident, downsampled set whose row r is idx r:
//
//   group   a stable radix sort of (hash, flat position) pairs: every run of equal hashes holds its positions
//           ascending, hence its idx ascending (lcx_head_kernel marks the run heads, a scan numbers the runs).
//   order   the dict's keys come out in first-insertion order, which is the flat order of the run heads: every head
//           writes its run id at its flat position (lcx_runs_kernel), a flagged compaction in flat order lists the
//           runs in key order, and lcx_keys_kernel inverts that list and takes each key's hash and size.
//   format  json.dump's text of the member, {"<hash>": [i0, i1, ...], ...}, with every byte owned by one element:
//           an element writes its idx and the ", " before it; the first of a key also the key's ", " separator and
//           "<hash>": [; the last also "]".  Sizes per element (lcx_elems_kernel), one scan, then any key range is
//           written by one thread per element (lcx_text_kernel), so a hash held by every genome costs what as many
//           hashes of one genome each cost.
// ------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ u32 lcx_digits(u64 v) {
    u32 d = 1;
    while (v >= 10) { v /= 10; ++d; }
    return d;
}

// v in decimal into [p, p + lcx_digits(v))
__device__ __forceinline__ void lcx_put_decimal(char* p, u64 v, u32 n) {
    for (u32 i = n; i-- > 0;) { p[i] = (char)('0' + v % 10); v /= 10; }
}

__global__ void __launch_bounds__(256) lcx_iota_kernel(u32* __restrict__ out, u64 T) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < T; e += (u64)gridDim.x * blockDim.x) out[e] = (u32)e;
}

// keys: the hashes sorted; head[e] = 1 where a run of equal hashes starts
__global__ void __launch_bounds__(256) lcx_head_kernel(const u64* __restrict__ keys, u64 T, u32* __restrict__ head) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < T; e += (u64)gridDim.x * blockDim.x)
        head[e] = (e == 0 || keys[e - 1] != keys[e]) ? 1u : 0u;
}

// rid = exclusive scan of head, so element e is in run rid[e] + head[e] - 1.  Run heads record where their run starts;
// at flat position pos[e] go the run id and whether e heads its run; the last element closes run_start and counts.
__global__ void __launch_bounds__(256) lcx_runs_kernel(const u32* __restrict__ pos, const u32* __restrict__ head,
                                                       const u32* __restrict__ rid, u64 T, u32* __restrict__ run_start,
                                                       u32* __restrict__ flat_run, u32* __restrict__ flat_head,
                                                       unsigned long long* __restrict__ n_runs) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < T; e += (u64)gridDim.x * blockDim.x) {
        const u32 h = head[e];
        const u32 r = rid[e] + h - 1;
        if (h) run_start[r] = (u32)e;
        flat_run[pos[e]] = r;
        flat_head[pos[e]] = h;
        if (e == T - 1) { run_start[r + 1] = (u32)T; *n_runs = (unsigned long long)r + 1; }
    }
}

// key_run: the run of every key in key order.  key_rank inverts it; size[k] and hash[k] are key k's
__global__ void __launch_bounds__(256) lcx_keys_kernel(const u32* __restrict__ key_run, u64 K,
                                                       const u32* __restrict__ run_start, const u64* __restrict__ keys,
                                                       u32* __restrict__ key_rank, u32* __restrict__ size,
                                                       u64* __restrict__ hash) {
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < K; k += (u64)gridDim.x * blockDim.x) {
        const u32 r = key_run[k];
        key_rank[r] = (u32)k;
        size[k] = run_start[r + 1] - run_start[r];
        hash[k] = keys[run_start[r]];
    }
}

// One thread per sorted element e: its place d in key order (koff = exclusive scan of the key sizes), its idx (the
// row whose offsets hold its flat position) and the bytes it owns in the text.
__global__ void __launch_bounds__(256) lcx_elems_kernel(const u64* __restrict__ hash, const u32* __restrict__ pos,
                                                        const u32* __restrict__ head, const u32* __restrict__ rid,
                                                        u64 T, const u32* __restrict__ run_start,
                                                        const u32* __restrict__ key_rank, const u32* __restrict__ koff,
                                                        const u64* __restrict__ row_off, u32 n_rows,
                                                        u32* __restrict__ idx, u32* __restrict__ key_of,
                                                        u64* __restrict__ bytes) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < T; e += (u64)gridDim.x * blockDim.x) {
        const u32 h = head[e];
        const u32 r = rid[e] + h - 1;
        const u32 k = key_rank[r];
        const u64 d = (u64)koff[k] + (e - run_start[r]);
        const u64 p = pos[e];
        u32 lo = 0, hi = n_rows;                               // the row: last r with row_off[r] <= p
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (row_off[mid] <= p) lo = mid; else hi = mid;
        }
        idx[d] = lo;
        key_of[d] = k;
        u64 b = lcx_digits(lo);
        b += h ? (k ? 2 : 0) + 1 + lcx_digits(hash[k]) + 4 : 2;    // ", " "\"" hash "\": [" or ", "
        if (e + 1 == run_start[r + 1]) b += 1;                     // "]"
        bytes[d] = b;
    }
}

// The key range [k0, k1): at is the exclusive scan of the element bytes (T + 1 entries).  k1 is the largest key whose
// range fits max_bytes with its braces counted (the opening one when k0 is 0, the closing one when k1 is K), at least
// k0 + 1.  The size grows with k1, so a binary search finds it.  out: k1, the range's bytes without braces, and its
// elements [koff[k0], koff[k1]).  One thread.
__global__ void lcx_plan_kernel(const u64* __restrict__ at, const u32* __restrict__ koff, u64 K, u64 k0, u64 max_bytes,
                                unsigned long long* __restrict__ out) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const u64 base = at[koff[k0]];
    const u64 lead = k0 == 0 ? 1 : 0;
    u64 lo = k0 + 1, hi = K;                                   // last k1 in [k0 + 1, K] within the budget, or k0 + 1
    while (lo < hi) {
        const u64 mid = (lo + hi + 1) >> 1;
        if (at[koff[mid]] - base + lead + (mid == K ? 1 : 0) <= max_bytes) lo = mid; else hi = mid - 1;
    }
    out[0] = lo;
    out[1] = at[koff[lo]] - base;
    out[2] = koff[k0];
    out[3] = koff[lo];
}

// The text of elements [d0, d1) (the keys of one range) into out, element d at out[at[d] - at[d0]]
__global__ void __launch_bounds__(256) lcx_text_kernel(const u64* __restrict__ hash, const u32* __restrict__ koff,
                                                       const u32* __restrict__ idx, const u32* __restrict__ key_of,
                                                       const u64* __restrict__ at, u64 d0, u64 d1,
                                                       char* __restrict__ out) {
    const u64 base = at[d0];
    for (u64 d = d0 + (u64)blockIdx.x * blockDim.x + threadIdx.x; d < d1; d += (u64)gridDim.x * blockDim.x) {
        const u32 k = key_of[d];
        char* p = out + (at[d] - base);
        if (d == koff[k]) {
            if (k) { *p++ = ','; *p++ = ' '; }
            const u64 hv = hash[k];
            const u32 n = lcx_digits(hv);
            *p++ = '"';
            lcx_put_decimal(p, hv, n);
            p += n;
            *p++ = '"'; *p++ = ':'; *p++ = ' '; *p++ = '[';
        } else {
            *p++ = ','; *p++ = ' ';
        }
        const u32 v = idx[d];
        const u32 n = lcx_digits(v);
        lcx_put_decimal(p, v, n);
        p += n;
        if (d + 1 == koff[k + 1]) *p = ']';
    }
}

}  // namespace smb
