// simt_stream_emul.cu -- the stream construction of the stripe join (sourmash_b200/csrc/join_stripe.cuh) on the CPU through
// the SIMT emulator of simt.h (CTAs as cooperative fibers, real __syncthreads / shared memory / atomics), kernel by kernel
// as join_stripe_create_shard (compare_kernels.cu) launches it, for the whole set or one key-range shard; a stable host
// sort stands in for cub::DeviceRadixSort::SortPairs.  The windows of pos[] follow the product's rule, or
// SMB_STRIPE_POS_WINDOW (elements) -- small windows split a test set into many.  Test infrastructure for the CPU-only suite.
//   simt_stream_emul <tag bits 16|32> <sort-key bits> <key-range shards> <shard> <hashes.u64> <offsets.u64> <out.u32 tags, pos>
// writes tags[0, T + STRIPE_TAG_PAD) as u32, then pos[0, T_all) (elements outside the stream: 0xffffffff).
#define SMB_SIMT_EMUL 1
#include "simt.h"

#include <numeric>

#include "../../sourmash_b200/csrc/join_kernels.cuh"
#include "../../sourmash_b200/csrc/join_stripe.cuh"

using namespace smb;

template <class T>
static std::vector<T> slurp(const char* path) {
    FILE* f = fopen(path, "rb");
    std::vector<T> v;
    if (!f) return v;
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    v.resize((size_t)n / sizeof(T));
    if (n && fread(v.data(), 1, (size_t)n, f) != (size_t)n) v.clear();
    fclose(f);
    return v;
}
template <class T>
static void dump(const char* path, const std::vector<T>& v) {
    FILE* f = fopen(path, "wb");
    fwrite(v.data(), sizeof(T), v.size(), f);
    fclose(f);
}

// The stream construction of join_stripe_create_shard (compare_kernels.cu) from the sorted keys on: row block table,
// window offsets, tags + position buckets, the window pass, the repair of runs that mix hashes.  The stream holds the
// elements [ebeg[r], eend[r]) of every row, doff[r] of them in rows < r; `pays` is the sort's input buffer (the
// buckets, then the repaired runs' ordered payloads).  One window: the tag kernel stores pos[] itself.
template <typename TagT>
static void stripe_stream(const std::vector<u32>& key32s, const std::vector<u64>& payss, std::vector<u64>& pays,
                          const std::vector<u64>& off, const u64* ebeg, const u64* eend, const u64* doff, u64 T, int low_bits,
                          u32 swz, std::vector<TagT>& tags, std::vector<u32>& pos, u32& count) {
    const int n = (int)off.size() - 1;
    const u64 T_all = off[n];
    const u64 nblk = (T_all >> STRIPE_EBLK_LOG2) + 1;
    std::vector<u32> eblk(nblk + 1), worklist(T + 1);
    smb_emu::launch(2, 64, 0, [&] { stripe_eblk_kernel(off.data(), n, T_all, eblk.data()); });
    const char* w = getenv("SMB_STRIPE_POS_WINDOW");
    const int lg = stripe_pos_window_log2(SMB_L2_BYTES, w ? strtoull(w, nullptr, 10) : 0ull, T_all);
    const u32 nw = T_all ? (u32)(((T_all - 1) >> lg) + 1) : 0u;
    std::vector<u32> boff(nw + 1), cur(nw + 1);
    const bool windows = nw > 1;
    if (windows) {
        smb_emu::launch(2, 64, 0, [&] { stripe_window_offsets_kernel(off.data(), n, ebeg, eend, doff, T_all, T, lg, nw, boff.data(), cur.data()); });
        if (boff[nw] != (u32)T) { fprintf(stderr, "window offsets end at %u, not %llu\n", boff[nw], (unsigned long long)T); exit(9); }
    }
    count = 0;
    u32* wl = low_bits ? worklist.data() : nullptr;
    smb_emu::launch(2, 96, 0, [&] { stripe_tag_kernel<TagT>(key32s.data(), payss.data(), off.data(), eblk.data(), T, tags.data(), pos.data(), wl,
                                                            &count, swz, windows ? pays.data() : nullptr, cur.data(), lg, nw); });
    if (windows) {
        for (u32 i = 0; i < nw; ++i)                 // every bucket filled exactly
            if (cur[i] != boff[i + 1]) { fprintf(stderr, "bucket %u ends at %u, not %u\n", i, cur[i], boff[i + 1]); exit(9); }
        smb_emu::launch((unsigned)((T + 64 * STRIPE_POS_UNROLL - 1) / (64 * STRIPE_POS_UNROLL)), 64, 0,
                        [&] { stripe_pos_window_kernel(pays.data(), T, pos.data()); });
    }
    if (getenv("SMB_EMUL_REPORT")) fprintf(stderr, "windows: %u\n", nw);
    if (low_bits)
        smb_emu::launch(2, 64, 0, [&] { stripe_fix_kernel<TagT>(key32s.data(), payss.data(), T, worklist.data(), &count, off.data(), n, pays.data(), tags.data(), pos.data(), swz); });
    if (getenv("SMB_EMUL_REPORT")) fprintf(stderr, "mixed runs repaired: %u\n", count);
}

// `sort_bits` < 64 shortens the sort key below the 32 bits the product uses, so that runs mixing different hashes --
// rare with 32-bit keys -- occur in every small test set and the descent detection of the tag kernel / the fix kernel
// are exercised.
static int stripe_low_bits_for_test(const std::vector<u64>& h, int sort_bits) {
    u64 max_key = 0;
    for (u64 v : h) max_key = std::max(max_key, v);
    int key_bits = 1;
    while (key_bits < 64 && (max_key >> key_bits)) ++key_bits;
    int low_bits = stripe_low_bits(max_key);
    if (sort_bits < 32 && key_bits > sort_bits) low_bits = std::min(32, key_bits - sort_bits);   // coarser keys (the payload holds at most 32 low bits)
    return low_bits;
}

// stable host sort by key (stands in for cub::DeviceRadixSort::SortPairs)
static void sort_stream(const std::vector<u32>& key32, const std::vector<u64>& pays, u64 T, std::vector<u32>& key32s, std::vector<u64>& payss) {
    std::vector<u32> perm(T);
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](u32 a, u32 b) { return key32[a] < key32[b]; });
    for (u64 q = 0; q < T; ++q) { key32s[q] = key32[perm[q]]; payss[q] = pays[perm[q]]; }
}

// The stream of the whole set (shards = 1) or of key range `shard` of `shards` (the rows' slices, as
// join_stripe_create_shard builds it), swizzle of the product for n columns.
template <typename TagT>
static int stream_run(int sort_bits, int shards, int shard, std::vector<u64>& h, const std::vector<u64>& off, const char* fout) {
    const int n = (int)off.size() - 1;
    const u64 T_all = h.size();
    const int low_bits = stripe_low_bits_for_test(h, sort_bits);
    u64 max_key = 0;
    for (u64 v : h) max_key = std::max(max_key, v);
    h.push_back(0);
    const size_t nn = (size_t)n + 1;
    std::vector<u64> beg(nn + 1, 0), cnt(nn + 1, 0), doff(nn + 1, 0), ebeg(nn + 1), eend(nn + 1);
    u64 lo = 0, hi = 0;
    bool bounded = false;
    join_shard_range(max_key, shard, shards, lo, hi, bounded);
    if (shards > 1) {
        smb_emu::launch((unsigned)((nn + 63) / 64), 64, 0, [&] { join_row_range_kernel(h.data(), off.data(), n, lo, hi, bounded ? 1 : 0, beg.data(), cnt.data()); });
        for (size_t r = 0; r < nn; ++r) doff[r + 1] = doff[r] + cnt[r];                 // cub::DeviceScan::ExclusiveSum
        smb_emu::launch((n + 63) / 64 + 1, 64, 0, [&] { stripe_slice_ranges_kernel(off.data(), beg.data(), cnt.data(), n, ebeg.data(), eend.data()); });
    } else {
        for (int r = 0; r <= n; ++r) { doff[r] = off[r]; ebeg[r] = off[r]; eend[r] = r < n ? off[r + 1] : off[r]; }
    }
    const u64 T = shards > 1 ? doff[n] : T_all;
    std::vector<u32> key32(T + 1), key32s(T + 1), pos(T_all + 1, 0xffffffffu);
    std::vector<u64> pays(T + 1), payss(T + 1);
    if (shards > 1) smb_emu::launch(3, 64, 0, [&] { stripe_keys_slice_kernel(h.data(), ebeg.data(), doff.data(), n, low_bits, key32.data(), pays.data()); });
    else smb_emu::launch(3, 64, 0, [&] { stripe_keys_kernel(h.data(), T, low_bits, key32.data(), pays.data()); });
    sort_stream(key32, pays, T, key32s, payss);
    std::vector<TagT> tags(T + STRIPE_TAG_PAD + 1);
    u32 count = 0;
    stripe_stream<TagT>(key32s, payss, pays, off, ebeg.data(), eend.data(), doff.data(), T, low_bits, (u32)n & ~31u, tags, pos, count);
    std::vector<u32> out(T + STRIPE_TAG_PAD + T_all);
    for (u64 q = 0; q < T + STRIPE_TAG_PAD; ++q) out[q] = (u32)tags[q];
    for (u64 e = 0; e < T_all; ++e) out[T + STRIPE_TAG_PAD + e] = pos[e];
    dump(fout, out);
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 8) { fprintf(stderr, "usage: see the head of simt_stream_emul.cu\n"); return 2; }
    std::vector<u64> h = slurp<u64>(argv[5]), off = slurp<u64>(argv[6]);
    return atoi(argv[1]) == 16 ? stream_run<u16>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), h, off, argv[7])
                               : stream_run<u32>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), h, off, argv[7]);
}
