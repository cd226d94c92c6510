// simt_hash_sort_emul.cu -- the stream construction of the stripe join from the sorted hashes themselves
// (sourmash_b200/csrc/join_stripe.cuh: stripe_iota_kernel / stripe_gather_slice_kernel, stripe_hash_tag_kernel,
// stripe_hash_fix_kernel) on the CPU through the SIMT emulator of simt.h, kernel by kernel as join_stripe_create_shard
// (compare_kernels.cu) launches it, for the whole set or one key-range shard; a stable host sort on the bit window
// stands in for cub::DeviceRadixSort::SortPairs.  A window narrower than the product's 32 bits makes runs that mix
// hashes in every small set.
// Windows and sub-windows of pos[] follow the product's rules, or SMB_STRIPE_POS_WINDOW / SMB_STRIPE_POS_SUBWINDOW
// (elements): small ones split a test set into hundreds.  Then the count kernel reads the bits (StripeArgs::succ) over
// all rows, upper triangle + mirror.  Test infrastructure for the CPU-only suite.
//   simt_hash_sort_emul <tag bits 16|32> <sort window bits> <key-range shards> <shard> <R> <hashes.u64> <offsets.u64> <out>
// writes <out>.tags (u32, T + STRIPE_TAG_PAD), <out>.pos (u32, T_all), <out>.succ (u32 words, ceil(T_all / 32)) and
// <out>.mat: float64 Jaccard (whole set) or u32 counts (shard).
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
static u64 env_u64(const char* name) {
    const char* v = getenv(name);
    return v ? strtoull(v, nullptr, 10) : 0ull;
}

template <typename TagT>
static int hash_sort_run(int sort_bits, int shards, int shard, int R, std::vector<u64>& h, const std::vector<u64>& off, const char* fout) {
    const int n = (int)off.size() - 1;
    const u64 T_all = h.size();
    u64 max_key = 0;
    for (u64 v : h) max_key = std::max(max_key, v);
    h.push_back(0);
    const size_t nn = (size_t)n + 1;
    std::vector<u64> beg(nn + 1, 0), cnt(nn + 1, 0), doff(nn + 1, 0), ebeg(nn + 1), eend(nn + 1);
    u64 lo = 0, max_rel = max_key;
    if (shards > 1) {
        u64 hi = 0;
        bool bounded = false;
        join_shard_range(max_key, shard, shards, lo, hi, bounded);
        max_rel = bounded ? hi - lo - 1 : max_key - lo;
        smb_emu::launch((unsigned)((nn + 63) / 64), 64, 0, [&] { join_row_range_kernel(h.data(), off.data(), n, lo, hi, bounded ? 1 : 0, beg.data(), cnt.data()); });
        for (size_t r = 0; r < nn; ++r) doff[r + 1] = doff[r] + cnt[r];                 // cub::DeviceScan::ExclusiveSum
        smb_emu::launch((n + 63) / 64 + 1, 64, 0, [&] { stripe_slice_ranges_kernel(off.data(), beg.data(), cnt.data(), n, ebeg.data(), eend.data()); });
    } else {
        for (int r = 0; r <= n; ++r) { doff[r] = off[r]; ebeg[r] = off[r]; eend[r] = r < n ? off[r + 1] : off[r]; }
    }
    int begin_bit = 0, end_bit = 0;
    stripe_sort_window(max_rel, begin_bit, end_bit);
    if (sort_bits < 32 && end_bit > sort_bits) begin_bit = end_bit - sort_bits;
    const u64 T = shards > 1 ? doff[n] : T_all;
    // the sort's input (the hashes themselves + an iota, or a shard's gathered slices), stable host sort on the window
    std::vector<u32> es_in(T + 1), es(T + 1), pos(T_all + 1, 0xffffffffu), sizes(nn);
    std::vector<u64> hs_in(T + 1), hs(T + 1), bucket(T + 1), sub(T + 1);
    if (shards > 1) smb_emu::launch(3, 64, 0, [&] { stripe_gather_slice_kernel(h.data(), ebeg.data(), doff.data(), n, lo, hs_in.data(), es_in.data()); });
    else {
        smb_emu::launch(3, 64, 0, [&] { stripe_iota_kernel(T, es_in.data()); });
        std::copy(h.begin(), h.begin() + T, hs_in.begin());
    }
    const u64 wmask = end_bit - begin_bit >= 64 ? ~0ull : ((1ull << (end_bit - begin_bit)) - 1ull);
    std::vector<u32> perm(T);
    std::iota(perm.begin(), perm.end(), 0u);
    std::stable_sort(perm.begin(), perm.end(), [&](u32 a, u32 b) { return ((hs_in[a] >> begin_bit) & wmask) < ((hs_in[b] >> begin_bit) & wmask); });
    for (u64 q = 0; q < T; ++q) { hs[q] = hs_in[perm[q]]; es[q] = es_in[perm[q]]; }
    // tags, positions and successor bits, as join_stripe_create_shard builds them
    const u64 nblk = (T_all >> STRIPE_EBLK_LOG2) + 1;
    std::vector<u32> eblk(nblk + 1);
    smb_emu::launch(2, 64, 0, [&] { stripe_eblk_kernel(off.data(), n, T_all, eblk.data()); });
    smb_emu::launch((n + 63) / 64 + 1, 64, 0, [&] { stripe_sizes_kernel(off.data(), n, sizes.data()); });
    int lg = 0, slg = 0;
    stripe_pos_levels(SMB_L2_BYTES, env_u64("SMB_STRIPE_POS_WINDOW"), env_u64("SMB_STRIPE_POS_SUBWINDOW"), T_all, lg, slg);
    const u32 nw = (u32)(((T_all - 1) >> lg) + 1), nsub = (u32)(((T_all - 1) >> slg) + 1);
    const bool windows = nw > 1;
    std::vector<u32> boff(nw + 1), cur(nw + 1), sboff(nsub + 1), scur(nsub + 1), succ((T_all + 31) / 32 + 1, 0xdeadbeefu);
    if (windows) {
        smb_emu::launch(2, 64, 0, [&] { stripe_window_offsets_kernel(off.data(), n, ebeg.data(), eend.data(), doff.data(), T_all, T, lg, nw, boff.data(), cur.data()); });
        smb_emu::launch(2, 64, 0, [&] { stripe_window_offsets_kernel(off.data(), n, ebeg.data(), eend.data(), doff.data(), T_all, T, slg, nsub, sboff.data(), scur.data()); });
    } else {
        std::fill(succ.begin(), succ.end(), 0u);                                         // cudaMemsetAsync
    }
    const u32 swz = (u32)n & ~31u;
    std::vector<TagT> tags(T + STRIPE_TAG_PAD + 1);
    u32 count = 0;
    u32* wl = begin_bit ? es_in.data() : nullptr;                                     // the iota is free after the sort
    smb_emu::launch(2, 96, 0, [&] { stripe_hash_tag_kernel<TagT>(hs.data(), es.data(), begin_bit, off.data(), eblk.data(), T, tags.data(), pos.data(),
                                                                 wl, &count, swz, windows ? bucket.data() : nullptr, cur.data(), lg, nw, succ.data()); });
    if (windows) {
        for (u32 i = 0; i < nw; ++i)                 // every bucket filled exactly
            if (cur[i] != boff[i + 1]) { fprintf(stderr, "bucket %u ends at %u, not %u\n", i, cur[i], boff[i + 1]); return 9; }
        smb_emu::launch(smb_emu::Dim3(2, nw), 64, (size_t)STRIPE_SUB_U * 64 * sizeof(u64), [&] { stripe_sub_partition_kernel(bucket.data(), boff.data(), lg, slg, scur.data(), sub.data()); });
        for (u32 i = 0; i < nsub; ++i)
            if (scur[i] != sboff[i + 1]) { fprintf(stderr, "sub-bucket %u ends at %u, not %u\n", i, scur[i], sboff[i + 1]); return 9; }
        const size_t smem = ((size_t)4 << slg) + ((size_t)1 << slg) / 8;
        smb_emu::launch(nsub, 64, smem, [&] { stripe_pos_sub_kernel(sub.data(), sboff.data(), T_all, slg, pos.data(), succ.data()); });
    }
    if (begin_bit) {
        u32* tmp = reinterpret_cast<u32*>(bucket.data());                              // the buckets are free again
        smb_emu::launch(2, 64, 0, [&] { stripe_hash_fix_kernel<TagT>(hs.data(), es.data(), begin_bit, T, wl, &count, off.data(), n, tmp, tags.data(),
                                                                     pos.data(), swz, succ.data()); });
    }
    fprintf(stderr, "windows: %u\nsub-windows: %u\nmixed runs repaired: %u\nsort window bits: %d\n", windows ? nw : 1u, windows ? nsub : 0u, count,
            end_bit - begin_bit);
    // the count kernel with the bits, all rows in index order, then the mirror
    const size_t cells = (size_t)n * n;
    std::vector<double> out(cells + 1, -1.0);
    std::vector<u32> counts(cells + 1, 0xdeadbeefu);
    const size_t smem = (size_t)STRIPE_HEADER + (size_t)R * n * sizeof(u32);
    StripeArgs a{tags.data(), pos.data(), ebeg.data(), eend.data(), sizes.data(), T, n, R, 0, n,
                 shards > 1 ? nullptr : out.data(), shards > 1 ? counts.data() : nullptr, nullptr, swz, nullptr, succ.data()};
    smb_emu::launch((n + R - 1) / R, 64, smem, [&] { join_stripe_kernel<TagT, true, 2>(a); });
    const int t = (n + STRIPE_MIRROR_TILE - 1) / STRIPE_MIRROR_TILE;
    if (shards > 1) smb_emu::launch(smb_emu::Dim3(t, t), 1024, 0, [&] { stripe_mirror_kernel<u32>(counts.data(), n, 0, n); });
    else smb_emu::launch(smb_emu::Dim3(t, t), 1024, 0, [&] { stripe_mirror_kernel<double>(out.data(), n, 0, n); });
    std::vector<u32> tg(T + STRIPE_TAG_PAD);
    for (u64 q = 0; q < T + STRIPE_TAG_PAD; ++q) tg[q] = (u32)tags[q];
    pos.resize(T_all);
    succ.resize((T_all + 31) / 32);
    dump(std::string(fout) + ".tags", tg);
    dump(std::string(fout) + ".pos", pos);
    dump(std::string(fout) + ".succ", succ);
    if (shards > 1) { counts.resize(cells); dump(std::string(fout) + ".mat", counts); }
    else { out.resize(cells); dump(std::string(fout) + ".mat", out); }
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 9) { fprintf(stderr, "usage: see the head of simt_hash_sort_emul.cu\n"); return 2; }
    std::vector<u64> h = slurp<u64>(argv[6]), off = slurp<u64>(argv[7]);
    const int R = atoi(argv[5]);
    if (R < 1 || R > STRIPE_MAX_ROWS || h.empty()) return 6;
    return atoi(argv[1]) == 16 ? hash_sort_run<u16>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), R, h, off, argv[8])
                               : hash_sort_run<u32>(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), R, h, off, argv[8]);
}
