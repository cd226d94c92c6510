// simt_order_emul.cu -- the row order of the stripe join's count kernel (sourmash_b200/csrc/join_stripe.cuh) on the CPU
// through the SIMT emulator of simt.h: the stream of the whole set or of one key-range shard, built kernel by kernel as
// join_stripe_create_shard (compare_kernels.cu) builds a set whose pos[] is one window; then the labels
// (stripe_label_kernel) and a stable host sort by label standing in for cub::DeviceRadixSort (stripe_make_order); then the
// count kernel in that order over two ranges of rows, each range's rows selected from the order by
// stripe_select_rows_kernel, upper triangle + mirror as join_stripe_rows / join_stripe_counts launch it.  Test
// infrastructure for the CPU-only suite.
//   simt_order_emul <tag bits 16|32> <swizzle 0|1> <key-range shards> <shard> <R> <hashes.u64> <offsets.u64> <out>
// writes the labels (u32 n) to <out>.lab and the matrix to <out>.mat: float64 Jaccard (whole set) or u32 counts (shard).
#define SMB_SIMT_EMUL 1
#include "simt.h"

#include <numeric>
#include <string>

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
static void dump(const std::string& path, const std::vector<T>& v) {
    FILE* f = fopen(path.c_str(), "wb");
    fwrite(v.data(), sizeof(T), v.size(), f);
    fclose(f);
}

template <typename TagT>
static int order_run(int swizzle, int shards, int shard, int R, std::vector<u64>& h, const std::vector<u64>& off, const char* fout) {
    const int n = (int)off.size() - 1;
    const u64 T_all = h.size();
    u64 max_key = 0;
    for (u64 v : h) max_key = std::max(max_key, v);
    const int low_bits = stripe_low_bits(max_key);
    h.push_back(0);
    const size_t nn = (size_t)n + 1;
    // the rows' elements in the stream: whole rows, or their slices of key range `shard`
    std::vector<u64> beg(nn + 1, 0), cnt(nn + 1, 0), doff(nn + 1, 0), ebeg(nn + 1), eend(nn + 1);
    if (shards > 1) {
        u64 lo = 0, hi = 0;
        bool bounded = false;
        join_shard_range(max_key, shard, shards, lo, hi, bounded);
        smb_emu::launch((unsigned)((nn + 63) / 64), 64, 0, [&] { join_row_range_kernel(h.data(), off.data(), n, lo, hi, bounded ? 1 : 0, beg.data(), cnt.data()); });
        for (size_t r = 0; r < nn; ++r) doff[r + 1] = doff[r] + cnt[r];                 // cub::DeviceScan::ExclusiveSum
        smb_emu::launch((n + 63) / 64 + 1, 64, 0, [&] { stripe_slice_ranges_kernel(off.data(), beg.data(), cnt.data(), n, ebeg.data(), eend.data()); });
    } else {
        for (int r = 0; r <= n; ++r) { ebeg[r] = off[r]; eend[r] = r < n ? off[r + 1] : off[r]; }
    }
    const u64 T = shards > 1 ? doff[n] : T_all;
    // the stream: keys, stable host sort, tags + positions (one window), the repair of runs that mix hashes
    std::vector<u32> key32(T + 1), key32s(T + 1), worklist(T + 1), pos(T_all + 1, 0xffffffffu), sizes(nn);
    std::vector<u64> pays(T + 1), payss(T + 1);
    if (shards > 1) smb_emu::launch(3, 64, 0, [&] { stripe_keys_slice_kernel(h.data(), ebeg.data(), doff.data(), n, low_bits, key32.data(), pays.data()); });
    else smb_emu::launch(3, 64, 0, [&] { stripe_keys_kernel(h.data(), T, low_bits, key32.data(), pays.data()); });
    std::vector<u32> perm(T);
    std::iota(perm.begin(), perm.end(), 0u);
    std::stable_sort(perm.begin(), perm.end(), [&](u32 a, u32 b) { return key32[a] < key32[b]; });
    for (u64 q = 0; q < T; ++q) { key32s[q] = key32[perm[q]]; payss[q] = pays[perm[q]]; }
    std::vector<u32> eblk((T_all >> STRIPE_EBLK_LOG2) + 2);
    smb_emu::launch(2, 64, 0, [&] { stripe_eblk_kernel(off.data(), n, T_all, eblk.data()); });
    smb_emu::launch((n + 63) / 64 + 1, 64, 0, [&] { stripe_sizes_kernel(off.data(), n, sizes.data()); });
    const u32 swz = swizzle ? ((u32)n & ~31u) : 0u;
    std::vector<TagT> tags(T + STRIPE_TAG_PAD + 1);
    u32 count = 0;
    u32* wl = low_bits ? worklist.data() : nullptr;
    smb_emu::launch(2, 96, 0, [&] { stripe_tag_kernel<TagT>(key32s.data(), payss.data(), off.data(), eblk.data(), T, tags.data(), pos.data(), wl, &count, swz); });
    if (low_bits)
        smb_emu::launch(2, 64, 0, [&] { stripe_fix_kernel<TagT>(key32s.data(), payss.data(), T, worklist.data(), &count, off.data(), n, pays.data(), tags.data(), pos.data(), swz); });
    // the order
    std::vector<u32> label(nn), rowid(nn), order(nn), sel(nn);
    smb_emu::launch(3, 64, 0, [&] { stripe_label_kernel<TagT>(tags.data(), pos.data(), ebeg.data(), eend.data(), n, swz, label.data(), rowid.data()); });
    for (int r = 0; r < n; ++r) if (rowid[r] != (u32)r) return 3;
    std::iota(order.begin(), order.begin() + n, 0u);
    std::stable_sort(order.begin(), order.begin() + n, [&](u32 a, u32 b) { return label[a] < label[b]; });
    // the count kernel in that order, two ranges of rows
    const size_t cells = (size_t)n * n;
    std::vector<double> out(cells + 1, -1.0);
    std::vector<u32> counts(cells + 1, 0xdeadbeefu);
    const size_t smem = (size_t)STRIPE_HEADER + (size_t)R * n * sizeof(u32);
    const int cut = n / 3;
    for (int c = 0; c < 2; ++c) {
        const int r0 = c ? cut : 0, r1 = c ? n : cut;
        if (r1 <= r0) continue;
        smb_emu::launch(1, 128, 0, [&] { stripe_select_rows_kernel(order.data(), n, r0, r1, sel.data() + r0); });
        StripeArgs a{tags.data(), pos.data(), ebeg.data(), eend.data(), sizes.data(), T, n, R, r0, r1,
                     shards > 1 ? nullptr : out.data() + (size_t)r0 * n, shards > 1 ? counts.data() + (size_t)r0 * n : nullptr, nullptr, swz,
                     sel.data() + r0};
        smb_emu::launch((r1 - r0 + R - 1) / R, 64, smem, [&] { join_stripe_kernel<TagT, true, 2>(a); });
        const int t0 = r0 / STRIPE_MIRROR_TILE, t1 = (r1 + STRIPE_MIRROR_TILE - 1) / STRIPE_MIRROR_TILE;
        if (shards > 1) smb_emu::launch(smb_emu::Dim3(t1, t1 - t0), 1024, 0, [&] { stripe_mirror_kernel<u32>(counts.data(), n, r0, r1); });
        else smb_emu::launch(smb_emu::Dim3(t1, t1 - t0), 1024, 0, [&] { stripe_mirror_kernel<double>(out.data(), n, r0, r1); });
    }
    label.resize(n);
    dump(std::string(fout) + ".lab", label);
    if (shards > 1) { counts.resize(cells); dump(std::string(fout) + ".mat", counts); }
    else { out.resize(cells); dump(std::string(fout) + ".mat", out); }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 9) { fprintf(stderr, "usage: see the head of simt_order_emul.cu\n"); return 2; }
    std::vector<u64> h = slurp<u64>(argv[6]), off = slurp<u64>(argv[7]);
    const int R = atoi(argv[5]);
    if (R < 1 || R > STRIPE_MAX_ROWS) return 6;
    return atoi(argv[1]) == 16 ? order_run<u16>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), R, h, off, argv[8])
                               : order_run<u32>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), R, h, off, argv[8]);
}
