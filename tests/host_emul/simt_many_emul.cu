// simt_many_emul.cu -- the many-query range-major pass of sourmash_b200/csrc/range_kernels.cuh on the CPU through the
// SIMT emulator of simt.h, built as range_major_build / many_vs_many_range_major build it (compare_kernels.cu): the
// range-major copy, the query ids (rm_query_ids_kernel), a stable host sort standing in for cub::DeviceRadixSort::
// SortPairs, then one_vs_many_range_major_kernel with the id array.  Test infrastructure for the CPU-only suite.
//   simt_many_emul <P> <bitmap log2> <threads> <ids 1 | 0: null id array, one query> <queries.u64> <query offsets.u64>
//                  <hashes.u64> <offsets.u64> <out.u32 G x n>
#define SMB_SIMT_EMUL 1
#include "simt.h"

#include <numeric>

#include "../../sourmash_b200/csrc/range_kernels.cuh"

using namespace smb;

template <class T>
static std::vector<T> slurp(const char* path) {
    std::vector<T> v;
    FILE* f = fopen(path, "rb");
    if (!f) return v;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    v.resize((size_t)n / sizeof(T));
    if (n && fread(v.data(), 1, (size_t)n, f) != (size_t)n) v.clear();
    fclose(f);
    return v;
}

int main(int argc, char** argv) {
    if (argc != 10) { fprintf(stderr, "usage: see the head of simt_many_emul.cu\n"); return 2; }
    const int P = atoi(argv[1]), bm_log2 = atoi(argv[2]), threads = atoi(argv[3]), use_ids = atoi(argv[4]);
    std::vector<u64> q = slurp<u64>(argv[5]), qoff = slurp<u64>(argv[6]), h = slurp<u64>(argv[7]), off = slurp<u64>(argv[8]);
    const int n = (int)off.size() - 1, G = (int)qoff.size() - 1;
    const u64 T = h.size(), nq = q.size();
    if (G < 1 || qoff[G] != nq || (!use_ids && G != 1)) return 2;
    // the range-major copy
    u64 max_key = 0;
    for (u64 v : h) max_key = std::max(max_key, v);
    const u64 width = range_width(max_key, P);
    const size_t cells = (size_t)n * P;
    std::vector<u32> bounds(cells + n + 1), cnt(cells + 2), slice(cells + 2);
    h.push_back(0);
    smb_emu::launch(3, 64, 0, [&] { rm_bounds_kernel(h.data(), off.data(), n, width, P, bounds.data()); });
    smb_emu::launch(2, 96, 0, [&] { rm_counts_kernel(bounds.data(), n, P, cnt.data()); });
    u32 run = 0;
    for (size_t i = 0; i <= cells; ++i) { slice[i] = run; run += cnt[i]; }          // cub::DeviceScan::ExclusiveSum
    if (slice[cells] != (u32)T) return 3;
    std::vector<u64> rm(T + 64, 0);
    smb_emu::launch(3, 64, 0, [&] { rm_scatter_kernel(h.data(), off.data(), bounds.data(), slice.data(), n, P, rm.data()); });
    const int nc = (n >> RM_COARSE_LOG2) + 2;
    std::vector<u32> coarse((size_t)P * nc + 1);
    smb_emu::launch(2, 64, 0, [&] { rm_coarse_kernel(slice.data(), n, P, nc, coarse.data()); });
    // the group's key stream: ids, statistics, the stable pair sort
    std::vector<u32> ids_in(nq + 1), ids(nq + 1);
    unsigned long long stat[2] = {0, 0};
    q.push_back(0);
    smb_emu::launch(3, 64, 0, [&] { rm_query_ids_kernel(q.data(), qoff.data(), G, ids_in.data(), stat); });
    if (stat[1]) return 4;                                                           // a query not sorted and unique
    u64 want_max = 0;
    for (int g = 0; g < G; ++g) if (qoff[g + 1] > qoff[g]) want_max = std::max(want_max, q[qoff[g + 1] - 1]);
    if (stat[0] != want_max) return 5;
    std::vector<size_t> perm(nq);
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](size_t a, size_t b) { return q[a] < q[b]; });
    std::vector<u64> keys(nq + 1);
    for (u64 i = 0; i < nq; ++i) { keys[i] = q[perm[i]]; ids[i] = ids_in[perm[i]]; }
    for (u64 i = 0; i < nq; ++i)
        if (ids_in[i] != (u32)(std::upper_bound(qoff.begin(), qoff.end(), i) - qoff.begin() - 1)) return 6;
    std::vector<u32> out((size_t)G * n + 1, 0);
    RangeMajorArgs a{keys.data(), nq, rm.data(), slice.data(), coarse.data(), nc, n, P, width, (u32)bm_log2,
                     range_bitmap_shift(width, 1ull << bm_log2), out.data(), use_ids ? ids.data() : nullptr};
    const size_t smem = (bm_log2 > 5 ? ((size_t)1 << (bm_log2 - 3)) : 4) + (size_t)(threads / 32) * RM_QUEUE * sizeof(u32);
    if (nq && n) smb_emu::launch(P, threads, smem, [&] { one_vs_many_range_major_kernel(a); });
    FILE* f = fopen(argv[9], "wb");
    fwrite(out.data(), sizeof(u32), (size_t)G * n, f);
    fclose(f);
    return 0;
}
