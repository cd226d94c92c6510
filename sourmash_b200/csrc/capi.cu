// capi.cu -- the C ABI of libsourmash_b200.so (see include/sourmash_b200.h).
//
// Host-side object model (KmerMinHash, Signature, ComputeParameters: sorted containers,
// parameter checks, error protocol) written in C++ against the behaviour of the reference's
// Rust core, with every hashing / set-intersection computation dispatched to the sm_90a
// kernels in sketch_kernels.cu / compare_kernels.cu.  There is no CPU implementation of
// those computations in this library: without a CUDA device the calls fail with
// SOURMASH_ERROR_CODE_CUDA.
//
// Reference behaviour cited per function (paths relative to sourmash/).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <zlib.h>

#include "../../include/sourmash_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "ingest.h"
#include "md5.h"
#include "range_search.cuh"
#include "zipread.h"

namespace smb {
static std::atomic<uint64_t> g_launches{0};
void count_launches(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
}  // namespace smb

namespace {

// ------------------------------------------------------------------------------------------
// error protocol: src/core/src/ffi/utils.rs:17-19 (TLS LAST_ERROR), :195-208 (landingpad)
// ------------------------------------------------------------------------------------------
struct SmbError {
    uint32_t code;
    std::string msg;
};
thread_local bool t_has_error = false;
thread_local SmbError t_error;

void set_error(uint32_t code, const std::string& msg) {
    t_has_error = true;
    t_error.code = code;
    t_error.msg = msg;
}

[[noreturn]] void fail(uint32_t code, const std::string& msg) { throw SmbError{code, msg}; }

// messages: src/core/src/errors.rs:10-59
[[noreturn]] void fail_ksize() { fail(SOURMASH_ERROR_CODE_MISMATCH_K_SIZES, "different ksizes cannot be compared"); }
[[noreturn]] void fail_dnaprot() { fail(SOURMASH_ERROR_CODE_MISMATCH_DNA_PROT, "DNA/prot minhashes cannot be compared"); }
[[noreturn]] void fail_scaled() { fail(SOURMASH_ERROR_CODE_MISMATCH_SCALED, "mismatch in scaled; comparison fail"); }
[[noreturn]] void fail_seed() { fail(SOURMASH_ERROR_CODE_MISMATCH_SEED, "mismatch in seed; comparison fail"); }

template <typename R, typename F>
R guarded(F&& f) {
    try {
        return f();
    } catch (const SmbError& e) {
        set_error(e.code, e.msg);
    } catch (const std::bad_alloc&) {
        set_error(SOURMASH_ERROR_CODE_PANIC, "out of host memory");
    } catch (const std::exception& e) {
        set_error(SOURMASH_ERROR_CODE_PANIC, std::string("panic: ") + e.what());
    }
    return R{};
}
template <typename F>
void guarded_void(F&& f) {
    try {
        f();
    } catch (const SmbError& e) {
        set_error(e.code, e.msg);
    } catch (const std::bad_alloc&) {
        set_error(SOURMASH_ERROR_CODE_PANIC, "out of host memory");
    } catch (const std::exception& e) {
        set_error(SOURMASH_ERROR_CODE_PANIC, std::string("panic: ") + e.what());
    }
}

SourmashStr make_str(const std::string& s) {
    SourmashStr r;
    r.len = s.size();
    r.data = (char*)malloc(s.size() + 1);
    memcpy(r.data, s.data(), s.size());
    r.data[s.size()] = 0;
    r.owned = true;
    return r;
}

// ------------------------------------------------------------------------------------------
// CUDA context
// ------------------------------------------------------------------------------------------
thread_local int t_device = -1;
thread_local cudaStream_t t_stream = 0;
std::once_flag g_probe_once;
int g_device_count = 0;
std::string g_probe_error;

void probe_devices() {
    std::call_once(g_probe_once, [] {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess) {
            g_probe_error = cudaGetErrorString(e);
            n = 0;
            cudaGetLastError();
        }
        g_device_count = n;
    });
}

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) {
        std::string m = std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e);
        cudaGetLastError();
        fail(SOURMASH_ERROR_CODE_CUDA, m);
    }
}
#define CK(x) cuda_check((x), #x)

cudaStream_t need_gpu() {
    probe_devices();
    if (g_device_count <= 0)
        fail(SOURMASH_ERROR_CODE_CUDA,
             "no usable CUDA device (" + (g_probe_error.empty() ? std::string("device count 0") : g_probe_error) +
                 "); sourmash_b200 has no CPU fallback for hashing / intersection");
    if (t_device >= 0) CK(cudaSetDevice(t_device));
    // keep freed stream-ordered allocations cached in the pool (default threshold 0 returns
    // them to the driver at every synchronisation, i.e. a fresh cudaMalloc per call)
    thread_local int t_pool_ready_for = -2;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    if (t_pool_ready_for != dev) {
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            unsigned long long keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
        t_pool_ready_for = dev;
    }
    return t_stream;
}

// stream-ordered device buffer
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaStream_t s = 0;
    DevBuf() {}
    DevBuf(size_t count, cudaStream_t st) { alloc(count, st); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), s(o.s) { o.p = nullptr; o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p = o.p; n = o.n; s = o.s; o.p = nullptr; o.n = 0; }
        return *this;
    }
    void alloc(size_t count, cudaStream_t st) {
        release();
        n = count; s = st;
        size_t bytes = std::max<size_t>(count * sizeof(T), 16);
        bytes = (bytes + 15) & ~size_t(15);
        CK(cudaMallocAsync((void**)&p, bytes, st));
    }
    void release() {
        if (p) { cudaFreeAsync(p, s); p = nullptr; n = 0; }
    }
    ~DevBuf() { release(); }
    void upload(const T* h, size_t count) {
        if (count) CK(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
    }
    void download(T* h, size_t count) const {
        if (count) CK(cudaMemcpyAsync(h, p, count * sizeof(T), cudaMemcpyDeviceToHost, s));
    }
    void zero() { CK(cudaMemsetAsync(p, 0, std::max<size_t>(n * sizeof(T), 16), s)); }
};

void sync(cudaStream_t s) { CK(cudaStreamSynchronize(s)); }

// optional CUDA-event timing of the dominant kernels (smb_set_profiling / smb_last_kernel_ms)
struct KernelTimer {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool armed = false;
    void begin(cudaStream_t s) {
        if (!e0) { CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); }
        CK(cudaEventRecord(e0, s));
    }
    void end(cudaStream_t s) { CK(cudaEventRecord(e1, s)); armed = true; }
    double ms() {
        if (!armed) return -1.0;
        float t = 0.f;
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&t, e0, e1));
        return (double)t;
    }
};
// second stream for uploads that overlap with kernels, and a small pool of timing-less events
thread_local cudaStream_t t_copy_stream = nullptr;
thread_local std::vector<cudaEvent_t> t_events;
thread_local size_t t_event_next = 0;
cudaStream_t copy_stream() {
    if (!t_copy_stream) CK(cudaStreamCreateWithFlags(&t_copy_stream, cudaStreamNonBlocking));
    return t_copy_stream;
}
cudaEvent_t pool_event() {
    if (t_events.size() < 64) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        t_events.push_back(e);
        return e;
    }
    return t_events[t_event_next++ % t_events.size()];
}
thread_local bool t_profiling = false;
thread_local KernelTimer t_timer_pairwise, t_timer_hash;

// max_hash_for_scaled / scaled_for_max_hash: src/core/src/sketch/minhash.rs:21-34
uint64_t max_hash_for_scaled(uint64_t scaled) {
    if (scaled == 0) return 0;
    if (scaled == 1) return UINT64_MAX;
    double v = 18446744073709551616.0 / (double)scaled;   // u64::MAX as f64 == 2^64
    return (uint64_t)v;
}
uint64_t scaled_for_max_hash(uint64_t max_hash) {
    if (max_hash == 0) return 0;
    double v = 18446744073709551616.0 / (double)max_hash;
    if (v >= 18446744073709551616.0) return UINT64_MAX;
    return (uint64_t)v;
}

}  // namespace

// ==========================================================================================
// device-resident CSR sketch set
// ==========================================================================================
struct SmbSketchSet {
    size_t n_rows = 0;
    std::vector<uint64_t> h_off;          // host copy of offsets (n_rows + 1)
    DevBuf<uint64_t> own_hashes, own_off, own_abunds;
    const uint64_t* d_hashes = nullptr;   // either own_* or borrowed
    const uint64_t* d_off = nullptr;
    const uint64_t* d_abunds = nullptr;
    uint64_t max_len = 0;
    mutable uint64_t max_key = 0;         // largest hash of any row (lazily computed on the device)
    mutable bool max_key_known = false;
    // range-major copy of the set (range_kernels.cuh), built at the first search with a query too large for shared
    // memory and kept with the resident set: the streaming one-vs-many pass reads it instead of the rows
    mutable smb::RangeMajor* range_major = nullptr;
    mutable bool range_major_tried = false;
    // inverted index (hash -> rows), built on request by smb_sketchset_build_index: the one-vs-many
    // counts of search / prefetch / gather then cost work proportional to the query (db_index.cuh)
    smb::DbIndex* index = nullptr;
    ~SmbSketchSet() {
        if (index) smb::db_index_destroy(index);
        if (range_major) smb::range_major_destroy(range_major);
    }
    uint64_t total() const { return h_off.empty() ? 0 : h_off.back(); }
    void finish_offsets() {
        max_len = 0;
        for (size_t i = 0; i < n_rows; ++i) max_len = std::max(max_len, h_off[i + 1] - h_off[i]);
    }
};

namespace {

// ------------------------------------------------------------------------------------------
// sketching core: streams in HBM -> CSR rows in HBM
// ------------------------------------------------------------------------------------------
struct StreamList {
    const uint8_t* d_bases = nullptr;        // 16-byte aligned, padded allocation
    const uint8_t* h_bases = nullptr;        // if set: host copy still to be uploaded to d_bases
    uint64_t total_bytes = 0;                //         (done in groups, overlapped with hashing)
    std::vector<uint64_t> off, len;          // per stream
    std::vector<uint32_t> row;               // per stream -> sketch index (empty: identity)
    size_t n_sketches = 0;
};

struct SketchParams {
    std::vector<uint32_t> ksizes;
    uint64_t max_hash = 0;                   // scaled mode threshold (0 in num mode)
    uint32_t num = 0;
    uint64_t seed = 42;
    bool track = false;
    // protein-family sketches: ksizes hold the ABI value (3 x residues, signature.rs:200-203);
    // input_is_protein: streams are residues (add_protein) instead of DNA to translate
    HashFunctions hash_function = HASH_FUNCTIONS_MURMUR64_DNA;
    bool input_is_protein = false;
    bool aa_mode() const { return hash_function != HASH_FUNCTIONS_MURMUR64_DNA; }
};

// expected survivors -> capacity with slack
uint64_t cap_for(uint64_t nwin, uint64_t thr) {
    if (thr == UINT64_MAX) return nwin;
    long double frac = ((long double)thr + 1.0L) / 18446744073709551616.0L;
    long double e = (long double)nwin * frac;
    uint64_t c = (uint64_t)(e * 1.25L + 8.0L * sqrtl(e + 1.0L) + 64.0L);
    return std::min<uint64_t>(nwin, c);
}

std::unique_ptr<SmbSketchSet> sketch_streams(const StreamList& in, const SketchParams& P,
                                             cudaStream_t s, uint64_t* n_kmers_out) {
    const size_t ns = in.off.size();
    const size_t nk = P.ksizes.size();
    const size_t n_sk = in.n_sketches;
    const size_t n_rows = n_sk * nk;
    auto set = std::make_unique<SmbSketchSet>();
    set->n_rows = n_rows;
    set->h_off.assign(n_rows + 1, 0);
    uint64_t n_kmers = 0;

    // per-sketch byte totals and per-row window counts
    std::vector<uint64_t> row_windows(n_rows, 0);
    uint64_t total_bytes = 0, longest = 0;
    for (size_t i = 0; i < ns; ++i) {
        size_t sk = in.row.empty() ? i : in.row[i];
        total_bytes += in.len[i];
        longest = std::max(longest, in.len[i]);
        for (size_t j = 0; j < nk; ++j) {
            uint64_t k = P.ksizes[j];
            uint64_t nw = (k > 0 && in.len[i] >= k) ? in.len[i] - k + 1 : 0;
            if (P.aa_mode()) {
                // residues: windows of k/3; DNA: every window of 3*(k/3) bases is hashed on both
                // strands (signature.rs:307-345)
                const uint64_t kaa = k / 3, span = P.input_is_protein ? kaa : 3 * kaa;
                nw = (kaa > 0 && in.len[i] >= span) ? (in.len[i] - span + 1) * (P.input_is_protein ? 1 : 2) : 0;
            }
            row_windows[sk * nk + j] += nw;
            n_kmers += nw;
        }
    }
    if (n_kmers_out) *n_kmers_out = n_kmers;
    bool never_stores = (P.num == 0 && P.max_hash == 0);     // minhash.rs:324-327
    if (n_rows == 0 || n_kmers == 0 || never_stores) {
        set->own_off.alloc(n_rows + 1, s);
        set->own_off.zero();
        set->own_hashes.alloc(1, s);
        if (P.track) set->own_abunds.alloc(1, s);
        set->d_off = set->own_off.p; set->d_hashes = set->own_hashes.p;
        set->d_abunds = P.track ? set->own_abunds.p : nullptr;
        set->finish_offsets();
        return set;
    }

    // windows per thread: keep >= ~8 CTAs per SM in flight when the input allows it
    const int threads = smb::hash_threads();
    int W = 128;
    while (W > 16 && total_bytes / ((uint64_t)threads * W) < (uint64_t)SMB_SMS * 8) W -= 16;

    std::vector<uint32_t> tile_r(ns + 1, 0), tile_g(ns + 1, 0);
    for (size_t i = 0; i < ns; ++i) {
        uint64_t lp = (in.off[i] & 15) + in.len[i];
        uint64_t per = (uint64_t)threads * W;
        tile_r[i + 1] = tile_r[i] + (uint32_t)((lp + per - 1) / per);
        tile_g[i + 1] = tile_g[i] + (uint32_t)((in.len[i] + 255) / 256);
    }
    DevBuf<uint64_t> d_soff(ns, s), d_slen(ns, s);
    DevBuf<uint32_t> d_tile_r(ns + 1, s), d_tile_g(ns + 1, s), d_srow;
    d_soff.upload(in.off.data(), ns);
    d_slen.upload(in.len.data(), ns);
    d_tile_r.upload(tile_r.data(), ns + 1);
    d_tile_g.upload(tile_g.data(), ns + 1);
    if (!in.row.empty()) { d_srow.alloc(ns, s); d_srow.upload(in.row.data(), ns); }

    // num mode keeps the `num` smallest distinct hashes: hash with a threshold that keeps a
    // few times `num` survivors, widen to "everything" if a row comes back short.
    std::vector<uint64_t> thr(n_rows, P.max_hash);
    if (P.num > 0) {
        for (size_t r = 0; r < n_rows; ++r) {
            long double want = 4.0L * P.num + 1024.0L;
            long double nw = (long double)std::max<uint64_t>(row_windows[r], 1);
            thr[r] = want >= nw ? UINT64_MAX : (uint64_t)(want / nw * 18446744073709551615.0L);
        }
    }
    // one threshold per launch: use the widest of the rows handled by the launch (per k)
    std::vector<uint64_t> cap(n_rows, 0);
    std::vector<uint32_t> cnt(n_rows, 0), ucnt(n_rows, 0);
    DevBuf<uint64_t> d_cand, d_cand_off(n_rows + 1, s), d_abund;
    DevBuf<uint32_t> d_cnt(n_rows, s), d_ucnt(n_rows, s);
    std::vector<uint64_t> cand_off(n_rows + 1, 0);
    std::vector<uint64_t> kthr(nk, 0);
    for (size_t j = 0; j < nk; ++j) {
        uint64_t t = 0;
        for (size_t sk = 0; sk < n_sk; ++sk) t = std::max(t, thr[sk * nk + j]);
        kthr[j] = t;
    }
    for (size_t r = 0; r < n_rows; ++r) cap[r] = cap_for(row_windows[r], kthr[r % nk]);

    DevBuf<uint8_t> d_aa_tables;
    if (P.aa_mode()) {
        for (uint32_t k : P.ksizes)
            if (k / 3 > smb::aa_max_k(!P.input_is_protein))
                fail(SOURMASH_ERROR_CODE_INTERNAL, "protein-family ksize too large for the shared-memory tile");
        const smb::AaTables T = smb::build_aa_tables((int)P.hash_function);
        d_aa_tables.alloc(sizeof T, s);
        d_aa_tables.upload((const uint8_t*)&T, sizeof T);
        sync(s);                                           // T is a stack temporary
    }
    const smb::AaTables* d_tabs = (const smb::AaTables*)d_aa_tables.p;
    auto launch_k = [&](smb::HashLaunch& L, size_t j, uint32_t r0, uint32_t r1, uint32_t g0, uint32_t g1) {
        if (P.aa_mode())
            smb::launch_hash_aa_range(L, d_tabs, P.ksizes[j] / 3, !P.input_is_protein, (int)j, g0, g1, s);
        else
            smb::launch_hash_kmers_range(L, P.ksizes[j], (int)j, r0, r1, g0, g1, s);
    };

    // experimental: the default dna parameter string k=21,31,51 hashed in one pass (SMB_SKETCH_FUSED)
    int fused_rows[3] = {-1, -1, -1};
    bool fused = smb::sketch_fused_enabled() && !P.aa_mode() && nk == 3;
    if (fused) {
        for (size_t j = 0; j < nk; ++j) {
            const int slot = P.ksizes[j] == 21 ? 0 : P.ksizes[j] == 31 ? 1 : P.ksizes[j] == 51 ? 2 : -1;
            if (slot >= 0) fused_rows[slot] = (int)j;
        }
        fused = fused_rows[0] >= 0 && fused_rows[1] >= 0 && fused_rows[2] >= 0;
    }
    auto launch_all_k = [&](smb::HashLaunch& L, uint32_t r0, uint32_t r1, uint32_t g0, uint32_t g1) {
        if (fused) {
            const uint64_t thr3[3] = {kthr[fused_rows[0]], kthr[fused_rows[1]], kthr[fused_rows[2]]};
            smb::launch_hash_kmers_fused_range(L, fused_rows, thr3, r0, r1, s);
            return;
        }
        for (size_t j = 0; j < nk; ++j) {
            L.max_hash = kthr[j];
            launch_k(L, j, r0, r1, g0, g1);
        }
    };

    bool uploaded = false;
    for (int attempt = 0; attempt < 4; ++attempt) {
        for (size_t r = 0; r < n_rows; ++r) cand_off[r + 1] = cand_off[r] + cap[r];
        d_cand.alloc(cand_off[n_rows], s);
        if (P.track) d_abund.alloc(cand_off[n_rows], s);
        d_cand_off.upload(cand_off.data(), n_rows + 1);
        d_cnt.zero();
        smb::HashLaunch L{};
        L.bases = in.d_bases; L.stream_off = d_soff.p; L.stream_len = d_slen.p;
        L.stream_row = in.row.empty() ? nullptr : d_srow.p;
        L.n_streams = (int)ns;
        L.tile_start_rolled = d_tile_r.p; L.total_tiles_rolled = tile_r[ns];
        L.tile_start_generic = d_tile_g.p; L.total_tiles_generic = tile_g[ns];
        L.W = W; L.seed = P.seed;
        L.cand = d_cand.p; L.cand_off = d_cand_off.p; L.cand_cnt = d_cnt.p;
        L.row_stride = (int)nk;
        if (t_profiling) t_timer_hash.begin(s);
        if (in.h_bases && !uploaded) {
            // pipeline: copy a group of streams on the copy stream, hash it on `s` as soon as it
            // has landed, while the next group is in flight
            cudaStream_t cs = copy_stream();
            cudaEvent_t ready = pool_event();
            CK(cudaEventRecord(ready, s));                  // d_bases allocation is ordered on s
            CK(cudaStreamWaitEvent(cs, ready, 0));
            // groups ramp up (8, 16, 32, 48, 48, ... MB): hashing starts after the first few MB have
            // landed instead of after a full-size group
            uint64_t group_bytes = 8ull << 20;
            size_t g0 = 0;
            while (g0 < ns) {
                size_t g1 = g0;
                uint64_t lo = in.off[g0], hi = lo;
                while (g1 < ns && (hi - lo < group_bytes || g1 == g0)) { hi = in.off[g1] + in.len[g1]; ++g1; }
                group_bytes = std::min<uint64_t>(group_bytes * 2, 48ull << 20);
                if (g1 == ns) hi = in.total_bytes;
                CK(cudaMemcpyAsync((void*)(in.d_bases + lo), in.h_bases + lo, hi - lo, cudaMemcpyHostToDevice, cs));
                cudaEvent_t ev = pool_event();
                CK(cudaEventRecord(ev, cs));
                CK(cudaStreamWaitEvent(s, ev, 0));
                launch_all_k(L, tile_r[g0], tile_r[g1], tile_g[g0], tile_g[g1]);
                g0 = g1;
            }
            uploaded = true;
        } else {
            launch_all_k(L, 0, tile_r[ns], 0, tile_g[ns]);
        }
        if (t_profiling) t_timer_hash.end(s);
        CK(cudaGetLastError());
        d_cnt.download(cnt.data(), n_rows);
        sync(s);
        bool overflow = false;
        for (size_t r = 0; r < n_rows; ++r)
            if (cnt[r] > cap[r]) { overflow = true; cap[r] = std::min<uint64_t>(row_windows[r], (uint64_t)cnt[r] + 64); }
        if (overflow) continue;                      // rerun with exact capacities

        // sort + unique
        smb::launch_sort_unique_small(d_cand.p, d_cand_off.p, d_cnt.p, (int)n_rows, d_ucnt.p,
                                      P.track ? d_abund.p : nullptr, s);
        const uint32_t small_max = (uint32_t)smb::sort_small_max();
        for (size_t r = 0; r < n_rows; ++r) {
            if (cnt[r] > small_max) {
                DevBuf<uint64_t> sorted(cnt[r], s), heads(cnt[r], s);
                CK(smb::sort_unique_big_row(d_cand.p + cand_off[r], cnt[r], sorted.p, heads.p,
                                            P.track ? d_abund.p + cand_off[r] : nullptr,
                                            d_ucnt.p + r, s));
            }
        }
        CK(cudaGetLastError());
        d_ucnt.download(ucnt.data(), n_rows);
        sync(s);
        if (P.num > 0) {
            bool shortfall = false;
            for (size_t j = 0; j < nk; ++j) {
                if (kthr[j] == UINT64_MAX) continue;
                for (size_t sk = 0; sk < n_sk; ++sk)
                    if (ucnt[sk * nk + j] < P.num) { shortfall = true; kthr[j] = UINT64_MAX; break; }
            }
            if (shortfall) {
                for (size_t r = 0; r < n_rows; ++r) cap[r] = cap_for(row_windows[r], kthr[r % nk]);
                continue;
            }
            for (size_t r = 0; r < n_rows; ++r) ucnt[r] = std::min(ucnt[r], P.num);
        }
        // dense CSR
        for (size_t r = 0; r < n_rows; ++r) set->h_off[r + 1] = set->h_off[r] + ucnt[r];
        DevBuf<uint32_t> d_final_cnt(n_rows, s);
        d_final_cnt.upload(ucnt.data(), n_rows);
        set->own_off.alloc(n_rows + 1, s);
        set->own_off.upload(set->h_off.data(), n_rows + 1);
        set->own_hashes.alloc(set->total(), s);
        smb::launch_compact_rows(d_cand.p, d_cand_off.p, d_final_cnt.p, set->own_off.p,
                                 set->own_hashes.p, (int)n_rows, s);
        if (P.track) {
            set->own_abunds.alloc(set->total(), s);
            smb::launch_compact_rows(d_abund.p, d_cand_off.p, d_final_cnt.p, set->own_off.p,
                                     set->own_abunds.p, (int)n_rows, s);
        }
        CK(cudaGetLastError());
        sync(s);      // h_off vector / ucnt are host temporaries used by the async uploads
        set->d_off = set->own_off.p; set->d_hashes = set->own_hashes.p;
        set->d_abunds = P.track ? set->own_abunds.p : nullptr;
        set->finish_offsets();
        return set;
    }
    fail(SOURMASH_ERROR_CODE_INTERNAL, "sketch candidate buffers kept overflowing");
}

// ------------------------------------------------------------------------------------------
// pairwise counts core (device in, device out)
// ------------------------------------------------------------------------------------------
struct CountsDev {
    DevBuf<uint32_t> common, usize;
    size_t ldo = 0;
};

// largest key of a set: one tiny reduction kernel + an 8-byte readback, cached on the set
uint64_t set_max_key(const SmbSketchSet& A, cudaStream_t s) {
    if (!A.max_key_known) {
        uint64_t m = 0;
        if (A.n_rows && A.total()) {
            DevBuf<unsigned long long> d_max(1, s);
            d_max.zero();
            smb::launch_max_last(A.d_hashes, A.d_off, (int)A.n_rows, nullptr, nullptr, 0, d_max.p, s);
            unsigned long long v = 0;
            d_max.download(&v, 1);
            sync(s);
            m = v;
        }
        A.max_key = m;
        A.max_key_known = true;
    }
    return A.max_key;
}

// Which algorithm computes the symmetric (all-vs-all) scaled count matrix?  The inverted join
// (compare_kernels.cu) costs one sort plus one increment per shared hash per pair; the tile kernel
// costs |A_i| probes per pair.  Decided from a deterministic 1/64 key-range sample of the set, so
// every rank holding the same set decides alike.  SMB_COMPARE_ALGO=join|tile overrides.
struct JoinDecision { bool use = false; double increments = 0, elements = 0; unsigned long long max_group = 0; };
thread_local JoinDecision t_last_join;

JoinDecision plan_join(const SmbSketchSet& A, uint64_t max_key, cudaStream_t s) {
    JoinDecision d;
    const char* env = getenv("SMB_COMPARE_ALGO");
    if (env && !strcmp(env, "tile")) return d;
    const size_t n = A.n_rows;
    if (n < 64 || A.total() == 0) return d;
    DevBuf<unsigned long long> scratch(2, s);
    CK(smb::join_estimate(A.d_hashes, A.d_off, (int)n, max_key, scratch.p, &d.increments, &d.elements,
                          &d.max_group, s));
    // cost model (ms): per-element cost of the stream build and sort, per-increment cost of the counting (with a
    // margin: hot cells serialise), per-hash cost of the tile kernel's pair walk.  The constants were fitted on the
    // previous target GPU and have not been refitted on the H100.  There they rank the two paths correctly for the
    // benchmark's 10 000 x 5 000-hash set (10.5 ms by the join, 218 ms by the tile kernel), but the crossover for
    // sets of near-duplicate sketches, where the join does the most work, has not been re-checked on the H100.  The
    // choice affects only speed: both paths give the same counts.
    const double join_ms = d.elements * 7e-8 + d.increments * 1.8e-8 + 0.5;
    const double pairs = 0.5 * (double)n * (double)(n - 1);
    const double avg_len = (double)A.total() / (double)n;
    const double tile_ms = pairs * avg_len * 7.4e-10 + 0.05;
    d.use = (env && !strcmp(env, "join")) || join_ms < tile_ms;
    return d;
}

void pairwise_counts_dev(const SmbSketchSet& A, const SmbSketchSet* Bp, uint32_t num, uint32_t* d_common,
                         uint32_t* d_usize, size_t ldo, cudaStream_t s,
                         smb::TileShard tiles = smb::TileShard{0, 1}) {
    const bool symmetric = (Bp == nullptr);
    const SmbSketchSet& B = symmetric ? A : *Bp;
    const int nA = (int)A.n_rows, nB = (int)B.n_rows;
    if (nA == 0 || nB == 0) return;
    if (symmetric && num == 0 && tiles.count < 0) {
        const uint64_t mk = set_max_key(A, s);
        t_last_join = plan_join(A, mk, s);
        if (t_last_join.use) {
            if (t_profiling) t_timer_pairwise.begin(s);
            CK(cudaMemsetAsync(d_common, 0, (size_t)nA * ldo * sizeof(uint32_t), s));
            CK(smb::join_counts(A.d_hashes, A.d_off, nA, mk, tiles.shard, tiles.n_shards, d_common, ldo, s));
            if (t_profiling) t_timer_pairwise.end(s);
            return;
        }
    }
    if (num > 0) {
        smb::launch_pairwise_num(A.d_hashes, A.d_off, nA, B.d_hashes, B.d_off, nB, num, d_common,
                                 d_usize, ldo, symmetric, s);
        return;
    }
    const uint64_t max_key = std::max(set_max_key(A, s), symmetric ? 0 : set_max_key(B, s));
    smb::PairwisePlan plan = smb::plan_pairwise(A.max_len, max_key, nB);
    if (plan.tables_per_cta == 0) {
        // rows too large for shared memory; a shard takes the rows i % n_shards == shard
        smb::launch_pairwise_generic(A.d_hashes, A.d_off, nA, B.d_hashes, B.d_off, nB, d_common, ldo,
                                     symmetric, tiles, s);
        return;
    }
    if (t_profiling) t_timer_pairwise.begin(s);
    smb::launch_pairwise_tile(plan, A.d_hashes, A.d_off, nA, B.d_hashes, B.d_off, nB, d_common, ldo,
                              symmetric, tiles, s);
    if (t_profiling) t_timer_pairwise.end(s);
}

// upload one sorted row as a 1-row set
std::unique_ptr<SmbSketchSet> single_row_set(const uint64_t* h, size_t n, const uint64_t* ab,
                                             cudaStream_t s) {
    auto set = std::make_unique<SmbSketchSet>();
    set->n_rows = 1;
    set->h_off = {0, (uint64_t)n};
    set->own_off.alloc(2, s);
    set->own_off.upload(set->h_off.data(), 2);
    set->own_hashes.alloc(n, s);
    set->own_hashes.upload(h, n);
    if (ab) { set->own_abunds.alloc(n, s); set->own_abunds.upload(ab, n); }
    set->d_off = set->own_off.p; set->d_hashes = set->own_hashes.p;
    set->d_abunds = ab ? set->own_abunds.p : nullptr;
    set->finish_offsets();
    return set;
}

}  // namespace

struct SmbGatherState {
    const SmbSketchSet* db = nullptr;        // the set the rounds run on (== sub.get() when compacted)
    std::unique_ptr<SmbSketchSet> sub;       // rows of the caller's database with overlap >= min_count
    std::vector<uint32_t> rowmap;            // compact row -> caller's row (empty: identity)
    DevBuf<uint64_t> q, isect;               // the original query stays in place ...
    DevBuf<uint8_t> alive;                   // ... consumed hashes are flagged, not removed
    DevBuf<uint32_t> counts, delta, d_n;
    DevBuf<unsigned long long> d_best;
    size_t nq = 0, remaining = 0;
    bool delta_pending = false;
};

// ==========================================================================================
// KmerMinHash host object: src/core/src/sketch/minhash.rs:41-64
// ==========================================================================================
// u64 -> decimal digits (no locale, no format parsing); returns the number of characters
inline int u64_to_dec(uint64_t v, char* out) {
    char tmp[24];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (int i = 0; i < n; ++i) out[i] = tmp[n - 1 - i];
    return n;
}

struct SourmashKmerMinHash {
    uint32_t num = 0, ksize = 0;
    HashFunctions hash_function = HASH_FUNCTIONS_MURMUR64_DNA;
    uint64_t seed = 42, max_hash = 0;
    bool track = false;
    std::vector<uint64_t> mins, abunds;     // abunds parallel to mins when track

    uint64_t scaled() const { return scaled_for_max_hash(max_hash); }   // minhash.rs:233-235

    // minhash.rs:886-912
    void check_compatible(const SourmashKmerMinHash& o) const {
        if (ksize != o.ksize) fail_ksize();
        if (hash_function != o.hash_function) fail_dnaprot();
        if (max_hash != o.max_hash) fail_scaled();
        if (seed != o.seed) fail_seed();
    }
    void remove_hash(uint64_t h) {          // minhash.rs:406-416
        auto it = std::lower_bound(mins.begin(), mins.end(), h);
        if (it != mins.end() && *it == h) {
            size_t p = it - mins.begin();
            mins.erase(it);
            if (track) abunds.erase(abunds.begin() + p);
        }
    }
    void add_hash_with_abundance(uint64_t h, uint64_t abundance) {   // minhash.rs:313-383
        uint64_t current_max = mins.empty() ? UINT64_MAX : mins.back();
        if (h > max_hash && max_hash != 0) return;
        if (num == 0 && max_hash == 0) return;
        if (abundance == 0) { remove_hash(h); return; }
        if (mins.empty()) { mins.push_back(h); if (track) abunds.push_back(abundance); return; }
        if (h <= max_hash || h <= current_max || mins.size() < (size_t)num) {
            auto it = std::lower_bound(mins.begin(), mins.end(), h);
            size_t pos = it - mins.begin();
            if (it == mins.end()) {
                mins.push_back(h);
                if (track) abunds.push_back(abundance);
            } else if (*it != h) {
                mins.insert(it, h);
                if (track) abunds.insert(abunds.begin() + pos, abundance);
                if (num != 0 && mins.size() > (size_t)num) { mins.pop_back(); if (track) abunds.pop_back(); }
            } else if (track) {
                abunds[pos] += abundance;
            }
        }
    }
    // bulk union with a sorted-unique batch (same result as add_hash_with_abundance per item)
    void absorb_sorted(const uint64_t* h, const uint64_t* ab, size_t n) {
        if (num == 0 && max_hash == 0) return;
        std::vector<uint64_t> m, a;
        m.reserve(mins.size() + n);
        if (track) a.reserve(mins.size() + n);
        size_t i = 0, j = 0;
        while (i < mins.size() || j < n) {
            if (j < n && max_hash != 0 && h[j] > max_hash) { ++j; continue; }
            bool take_i = j >= n || (i < mins.size() && mins[i] <= h[j]);
            bool take_j = i >= mins.size() || (j < n && h[j] <= mins[i]);
            uint64_t v = take_i ? mins[i] : h[j];
            uint64_t c = 0;
            if (track) c = (take_i ? abunds[i] : 0) + (take_j ? (ab ? ab[j] : 1) : 0);
            m.push_back(v);
            if (track) a.push_back(c);
            if (take_i) ++i;
            if (take_j) ++j;
        }
        if (num != 0 && m.size() > (size_t)num) { m.resize(num); if (track) a.resize(num); }
        mins.swap(m);
        if (track) abunds.swap(a);
    }
    // minhash.rs:432-516
    void merge(const SourmashKmerMinHash& o) {
        check_compatible(o);
        const bool both = track && o.track;
        std::vector<uint64_t> m, a;
        m.reserve(mins.size() + o.mins.size());
        size_t i = 0, j = 0;
        while (i < mins.size() && j < o.mins.size()) {
            if (o.mins[j] < mins[i]) { m.push_back(o.mins[j]); if (both) a.push_back(o.abunds[j]); ++j; }
            else if (o.mins[j] == mins[i]) { m.push_back(mins[i]); if (both) a.push_back(abunds[i] + o.abunds[j]); ++i; ++j; }
            else { m.push_back(mins[i]); if (both) a.push_back(abunds[i]); ++i; }
        }
        for (; i < mins.size(); ++i) { m.push_back(mins[i]); if (both) a.push_back(abunds[i]); }
        for (; j < o.mins.size(); ++j) { m.push_back(o.mins[j]); if (both) a.push_back(o.abunds[j]); }
        if (num != 0 && m.size() > (size_t)num) { m.resize(num); if (both) a.resize(num); }
        mins.swap(m);
        abunds.swap(a);
        track = both;            // merged_abunds = None unless both sides track
    }
    // minhash.rs:777-798 (errors on upsampling; identity when scaled() equal or num sketch)
    SourmashKmerMinHash downsample_scaled(uint64_t new_scaled) const {
        if (scaled() == new_scaled || scaled() == 0) return *this;
        if (scaled() > new_scaled)
            fail(SOURMASH_ERROR_CODE_CANNOT_UPSAMPLE_SCALED, "new scaled smaller than previous; cannot upsample");
        SourmashKmerMinHash r;
        r.num = num; r.ksize = ksize; r.hash_function = hash_function; r.seed = seed;
        r.track = track; r.max_hash = max_hash_for_scaled(new_scaled);
        size_t keep = std::upper_bound(mins.begin(), mins.end(), r.max_hash) - mins.begin();
        r.mins.assign(mins.begin(), mins.begin() + keep);
        if (track) r.abunds.assign(abunds.begin(), abunds.begin() + keep);
        return r;
    }
    std::string md5sum() const {   // minhash.rs:290-307
        smb::Md5 ctx;
        char buf[4096];
        size_t fill = (size_t)u64_to_dec(ksize, buf);
        for (uint64_t v : mins) {
            if (fill > sizeof buf - 24) { ctx.update((const uint8_t*)buf, fill); fill = 0; }
            fill += (size_t)u64_to_dec(v, buf + fill);
        }
        ctx.update((const uint8_t*)buf, fill);
        return ctx.hexdigest();
    }
};

namespace {

typedef SourmashKmerMinHash MH;

// hash one sequence on the GPU and fold the survivors into the sketch.
// signature.rs:38-58 (+ :271-279 for the !force error, raised after earlier windows were added)
// protein-family sketch fed residues (add_protein, signature.rs:60-80) or DNA to translate in six
// frames (add_sequence on such a sketch, signature.rs:307-357; no validity check, `force` unused)
void mh_add_aa(MH& mh, const uint8_t* seq, size_t len, bool input_is_protein) {
    const size_t kaa = mh.ksize / 3;                     // signature.rs:200-203
    if (len < kaa) return;                               // max_index == 0: the iterator ends at once
    if (mh.hash_function == HASH_FUNCTIONS_MURMUR64_DNA) // only reachable with input_is_protein
        fail(SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION, "Invalid hash function: \"DNA\"");   // :376-380
    if (kaa == 0 || (!input_is_protein && len < 3 * kaa)) return;       // signature.rs:259-262
    cudaStream_t s = need_gpu();
    DevBuf<uint8_t> d_seq(len + 32, s);
    d_seq.upload(seq, len);
    StreamList in;
    in.d_bases = d_seq.p;
    in.off = {0}; in.len = {len}; in.n_sketches = 1;
    SketchParams P;
    P.ksizes = {mh.ksize}; P.max_hash = mh.max_hash; P.num = mh.num; P.seed = mh.seed;
    P.track = mh.track; P.hash_function = mh.hash_function; P.input_is_protein = input_is_protein;
    auto set = sketch_streams(in, P, s, nullptr);
    const size_t n = set->total();
    std::vector<uint64_t> h(n), ab(mh.track ? n : 0);
    if (n) {
        CK(cudaMemcpyAsync(h.data(), set->d_hashes, n * 8, cudaMemcpyDeviceToHost, s));
        if (mh.track) CK(cudaMemcpyAsync(ab.data(), set->d_abunds, n * 8, cudaMemcpyDeviceToHost, s));
        sync(s);
    }
    mh.absorb_sorted(h.data(), mh.track ? ab.data() : nullptr, n);
}

void mh_add_sequence(MH& mh, const uint8_t* seq, size_t len, bool force) {
    if (mh.hash_function != HASH_FUNCTIONS_MURMUR64_DNA) { mh_add_aa(mh, seq, len, false); return; }
    const size_t k = mh.ksize;
    if (k == 0 || len < k) return;                       // signature.rs:206-210
    cudaStream_t s = need_gpu();
    DevBuf<uint8_t> d_seq(len + 32, s);
    d_seq.upload(seq, len);
    size_t use_len = len;
    int64_t bad_window = -1;
    if (!force) {
        DevBuf<unsigned long long> d_pos(1, s);
        smb::launch_first_invalid(d_seq.p, len, d_pos.p, s);
        unsigned long long pos = 0;
        d_pos.download(&pos, 1);
        sync(s);
        if (pos != ~0ull) {
            bad_window = pos + 1 >= k ? (int64_t)(pos - k + 1) : 0;
            use_len = (size_t)bad_window + k - 1;         // windows [0, bad_window) only
        }
    }
    if (use_len >= k) {
        StreamList in;
        in.d_bases = d_seq.p;
        in.off = {0}; in.len = {use_len}; in.n_sketches = 1;
        SketchParams P;
        P.ksizes = {mh.ksize}; P.max_hash = mh.max_hash; P.num = mh.num; P.seed = mh.seed;
        P.track = mh.track;
        auto set = sketch_streams(in, P, s, nullptr);
        size_t n = set->total();
        std::vector<uint64_t> h(n), ab(mh.track ? n : 0);
        if (n) {
            CK(cudaMemcpyAsync(h.data(), set->d_hashes, n * 8, cudaMemcpyDeviceToHost, s));
            if (mh.track) CK(cudaMemcpyAsync(ab.data(), set->d_abunds, n * 8, cudaMemcpyDeviceToHost, s));
            sync(s);
        }
        mh.absorb_sorted(h.data(), mh.track ? ab.data() : nullptr, n);
    }
    if (bad_window >= 0) {
        std::string km((const char*)seq + bad_window, k);
        for (auto& c : km) if (c >= 'a' && c <= 'z') c -= 32;
        fail(SOURMASH_ERROR_CODE_INVALID_DNA, "invalid DNA character in input k-mer: " + km);
    }
}

// force=True over several sketches that differ only in ksize (the `sketch dna -p k=21,k=31,k=51`
// case, signature.rs:661-677): one upload, one hash launch per ksize, one sort pass.
void add_sequence_group(std::vector<MH*>& group, const uint8_t* seq, size_t len) {
    cudaStream_t s = need_gpu();
    DevBuf<uint8_t> d_seq(len + 32, s);
    d_seq.upload(seq, len);
    StreamList in;
    in.d_bases = d_seq.p;
    in.off = {0}; in.len = {len}; in.n_sketches = 1;
    SketchParams P;
    for (MH* m : group) P.ksizes.push_back(m->ksize);
    const MH& f = *group[0];
    P.max_hash = f.max_hash; P.num = f.num; P.seed = f.seed; P.track = f.track;
    auto set = sketch_streams(in, P, s, nullptr);
    const size_t n = set->total();
    std::vector<uint64_t> h(n), ab(f.track ? n : 0);
    if (n) {
        CK(cudaMemcpyAsync(h.data(), set->d_hashes, n * 8, cudaMemcpyDeviceToHost, s));
        if (f.track) CK(cudaMemcpyAsync(ab.data(), set->d_abunds, n * 8, cudaMemcpyDeviceToHost, s));
        sync(s);
    }
    for (size_t j = 0; j < group.size(); ++j) {
        const size_t o = set->h_off[j], c = set->h_off[j + 1] - o;
        group[j]->absorb_sorted(h.data() + o, f.track ? ab.data() + o : nullptr, c);
    }
}

// seq_to_hashes for protein-family sketches (ffi/minhash.rs:63-99 over signature.rs:307-392):
// hashes in the reference's order; zeros dropped unless keep_zeros, in which case the translate
// iterator's two bookkeeping Ok(0) items (signature.rs:346,351) are part of the output too.
std::vector<uint64_t> aa_seq_to_hashes(const MH& mh, const uint8_t* seq, size_t len, bool is_protein,
                                       bool keep_zeros) {
    std::vector<uint64_t> out;
    const size_t kaa = mh.ksize / 3;
    if (len < kaa) return out;
    if (is_protein && mh.hash_function == HASH_FUNCTIONS_MURMUR64_DNA)
        fail(SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION, "Invalid hash function: \"DNA\"");
    const bool translate = !is_protein;
    if (kaa == 0 || (translate && len < 3 * kaa)) return out;
    if (kaa > smb::aa_max_k(translate))
        fail(SOURMASH_ERROR_CODE_INTERNAL, "protein-family ksize too large for the shared-memory tile");
    cudaStream_t s = need_gpu();
    const size_t span = translate ? 3 * kaa : kaa;
    const size_t nraw = (len - span + 1) * (translate ? 2 : 1);
    DevBuf<uint8_t> d_seq(len + 32, s), d_tabs(sizeof(smb::AaTables), s);
    d_seq.upload(seq, len);
    const smb::AaTables T = smb::build_aa_tables((int)mh.hash_function);
    d_tabs.upload((const uint8_t*)&T, sizeof T);
    DevBuf<uint64_t> d_raw(nraw, s);
    uint64_t off = 0, ln = len;
    uint32_t tg[2] = {0, (uint32_t)((len + 255) / 256)};
    DevBuf<uint64_t> d_off(1, s), d_len(1, s);
    DevBuf<uint32_t> d_tg(2, s);
    d_off.upload(&off, 1); d_len.upload(&ln, 1); d_tg.upload(tg, 2);
    smb::HashLaunch L{};
    L.bases = d_seq.p; L.stream_off = d_off.p; L.stream_len = d_len.p; L.stream_row = nullptr;
    L.n_streams = 1; L.tile_start_rolled = d_tg.p; L.total_tiles_rolled = 0;
    L.tile_start_generic = d_tg.p; L.total_tiles_generic = tg[1];
    L.W = 16; L.seed = mh.seed; L.max_hash = UINT64_MAX;
    smb::launch_aa_window_hashes(L, (const smb::AaTables*)d_tabs.p, (uint32_t)kaa, translate, len, d_raw.p, s);
    CK(cudaGetLastError());
    std::vector<uint64_t> raw(nraw);
    d_raw.download(raw.data(), nraw);
    sync(s);
    out.reserve(nraw + 2);
    if (translate && keep_zeros) out.push_back(0);
    for (uint64_t h : raw) if (h != 0 || keep_zeros) out.push_back(h);
    if (translate && keep_zeros) out.push_back(0);
    return out;
}

struct PairCounts { uint64_t common, usize; };

// |A ∩ B| (and |M| for num sketches) of two host sketches, computed on the GPU
PairCounts mh_pair_counts(const MH& a, const MH& b, bool num_semantics) {
    cudaStream_t s = need_gpu();
    auto sa = single_row_set(a.mins.data(), a.mins.size(), nullptr, s);
    auto sb = single_row_set(b.mins.data(), b.mins.size(), nullptr, s);
    DevBuf<uint32_t> d_out(2, s);
    d_out.zero();
    uint32_t num = num_semantics ? a.num : 0;
    pairwise_counts_dev(*sa, sb.get(), num, d_out.p, d_out.p + 1, 1, s);
    CK(cudaGetLastError());
    uint32_t out[2] = {0, 0};
    d_out.download(out, 2);
    sync(s);
    PairCounts r;
    r.common = out[0];
    r.usize = num ? out[1] : (uint64_t)a.mins.size() + b.mins.size() - out[0];
    return r;
}

// minhash.rs:593-621
PairCounts mh_intersection_size(const MH& a, const MH& b) {
    a.check_compatible(b);
    return mh_pair_counts(a, b, a.num != 0);
}

double mh_jaccard(const MH& a, const MH& b) {       // minhash.rs:624-631
    a.check_compatible(b);
    PairCounts c = mh_intersection_size(a, b);
    return (double)c.common / (double)std::max<uint64_t>(1, c.usize);
}

// the tail of minhash.rs:635-680: the score from the dot product and the two sums of squares (u64, wrapped), on the
// host with libm -- mh_angular and smb_search_angular share it, so the two give the same bits
double angular_from_terms(uint64_t prod, uint64_t a_sq, uint64_t b_sq) {
    const double norm_a = std::sqrt((double)a_sq), norm_b = std::sqrt((double)b_sq);
    if (norm_a == 0. || norm_b == 0.) return 0.0;
    const double p = std::min((double)prod / (norm_a * norm_b), 1.0);
    const double distance = 2. * std::acos(p) / 3.14159265358979323846264338327950288;
    return 1. - distance;
}

double mh_angular(const MH& a, const MH& b) {       // minhash.rs:635-680
    a.check_compatible(b);
    if (!a.track || !b.track)
        fail(SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING, "sketch needs abundance for this operation");
    cudaStream_t s = need_gpu();
    auto sa = single_row_set(a.mins.data(), a.mins.size(), a.abunds.data(), s);
    auto sb = single_row_set(b.mins.data(), b.mins.size(), b.abunds.data(), s);
    DevBuf<unsigned long long> d_out(3, s);
    smb::launch_angular_terms(sa->d_hashes, sa->d_abunds, a.mins.size(), sb->d_hashes, sb->d_abunds,
                              b.mins.size(), d_out.p, s);
    unsigned long long t[3];
    d_out.download(t, 3);
    sync(s);
    return angular_from_terms(t[0], t[1], t[2]);
}

double mh_similarity(const MH& a, const MH& b, bool ignore_abundance, bool downsample) {
    // minhash.rs:682-702
    if (downsample && a.scaled() != b.scaled()) {
        const MH& first = a.scaled() > b.scaled() ? a : b;
        const MH& second = a.scaled() > b.scaled() ? b : a;
        MH ds = second.downsample_scaled(first.scaled());
        return mh_similarity(first, ds, ignore_abundance, false);
    }
    if (ignore_abundance || !a.track || !b.track) return mh_jaccard(a, b);
    return mh_angular(a, b);
}

uint64_t mh_count_common(const MH& a, const MH& b, bool downsample) {   // minhash.rs:539-558
    if (downsample && a.scaled() != b.scaled()) {
        const MH& first = a.scaled() > b.scaled() ? a : b;
        const MH& second = a.scaled() > b.scaled() ? b : a;
        MH ds = second.downsample_scaled(first.scaled());
        return mh_count_common(first, ds, false);
    }
    a.check_compatible(b);
    return mh_pair_counts(a, b, false).common;
}

// minhash.rs:560-589 + ffi/minhash.rs:428-441
MH* mh_intersection(const MH& a, const MH& b) {
    a.check_compatible(b);
    cudaStream_t s = need_gpu();
    auto sa = single_row_set(a.mins.data(), a.mins.size(), nullptr, s);
    auto sb = single_row_set(b.mins.data(), b.mins.size(), nullptr, s);
    DevBuf<uint64_t> d_out(std::min(a.mins.size(), b.mins.size()) + 1, s);
    DevBuf<uint32_t> d_n(1, s);
    smb::launch_intersect_rows(sa->d_hashes, a.mins.size(), sb->d_hashes, b.mins.size(), d_out.p, d_n.p, s);
    uint32_t n = 0;
    d_n.download(&n, 1);
    sync(s);
    size_t keep = n;
    if (a.num != 0) keep = std::min<size_t>(keep, mh_pair_counts(a, b, true).common);
    std::vector<uint64_t> common(keep);
    if (keep) { CK(cudaMemcpyAsync(common.data(), d_out.p, keep * 8, cudaMemcpyDeviceToHost, s)); sync(s); }
    MH* r = new MH(a);
    r->mins.clear();
    r->abunds.clear();
    for (uint64_t h : common) r->add_hash_with_abundance(h, 1);
    return r;
}

uint64_t murmur_on_gpu(const uint8_t* data, size_t len, uint64_t seed) {
    cudaStream_t s = need_gpu();
    DevBuf<uint8_t> d(len + 16, s);
    d.upload(data, len);
    DevBuf<uint64_t> d_out(1, s);
    smb::launch_murmur_bytes(d.p, len, seed, d_out.p, s);
    uint64_t h = 0;
    d_out.download(&h, 1);
    sync(s);
    return h;
}

uint64_t* to_boxed(const std::vector<uint64_t>& v, uintptr_t* size) {
    uint64_t* p = (uint64_t*)malloc(std::max<size_t>(v.size(), 1) * 8);
    if (!v.empty()) memcpy(p, v.data(), v.size() * 8);
    *size = v.size();
    return p;
}

}  // namespace
// ==========================================================================================
// Signature / ComputeParameters: src/core/src/signature.rs:401-445, cmd.rs:22-188
// ==========================================================================================
struct SourmashComputeParameters {
    std::vector<uint32_t> ksizes{21, 31, 51};    // cmd.rs:60-84 defaults
    bool dna = true, protein = false, dayhoff = false, hp = false, track_abundance = false;
    uint32_t num_hashes = 500;
    uint64_t scaled = 0, seed = 42;
};
struct SourmashSignature {                 // signature.rs:401-445
    std::string name, filename;
    std::string license = "CC0";
    std::string email, klass = "sourmash_signature", hash_function = "0.murmur64";
    double version = 0.4;
    std::vector<MH> sketches;
};
struct SmbRecords { smb::RecordBatch b; };
struct SmbSigs { smb::SigBatch b; };
struct SourmashZipStorage {
    smb::ZipArchive zip;
    std::string path, subdir;
    bool has_subdir = false;
};

namespace {

// ------------------------------------------------------------------------------------------
// .sig JSON writer (serde field order of signature.rs:401-445 and sketch/minhash.rs:103-131)
// ------------------------------------------------------------------------------------------
void json_escape(std::string& out, const std::string& s) {
    out.push_back('"');
    for (unsigned char c : s) {
        switch (c) {
            case '"': out += "\\\""; break;
            case '\\': out += "\\\\"; break;
            case '\n': out += "\\n"; break;
            case '\r': out += "\\r"; break;
            case '\t': out += "\\t"; break;
            case '\b': out += "\\b"; break;
            case '\f': out += "\\f"; break;
            default:
                if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); out += b; }
                else out.push_back((char)c);
        }
    }
    out.push_back('"');
}
void json_u64_array(std::string& out, const std::vector<uint64_t>& v) {
    out.push_back('[');
    const size_t base = out.size();
    out.resize(base + v.size() * 21 + 1);
    char* w = &out[base];
    for (size_t i = 0; i < v.size(); ++i) {
        if (i) *w++ = ',';
        w += u64_to_dec(v[i], w);
    }
    out.resize((size_t)(w - out.data()));
    out.push_back(']');
}
const char* molecule_name(HashFunctions hf) {          // encodings.rs:55-69 (Display)
    return hf == HASH_FUNCTIONS_MURMUR64_PROTEIN ? "protein" : hf == HASH_FUNCTIONS_MURMUR64_DAYHOFF ? "dayhoff"
         : hf == HASH_FUNCTIONS_MURMUR64_HP ? "hp" : "DNA";
}
void json_signature(std::string& out, const SourmashSignature& sig) {
    out += "{\"class\":"; json_escape(out, sig.klass);
    out += ",\"email\":"; json_escape(out, sig.email);
    out += ",\"hash_function\":"; json_escape(out, sig.hash_function);
    out += ",\"filename\":";
    if (sig.filename.empty()) out += "null"; else json_escape(out, sig.filename);
    if (!sig.name.empty()) { out += ",\"name\":"; json_escape(out, sig.name); }
    out += ",\"license\":"; json_escape(out, sig.license);
    out += ",\"signatures\":[";
    for (size_t i = 0; i < sig.sketches.size(); ++i) {
        const MH& m = sig.sketches[i];
        if (i) out.push_back(',');
        out += "{\"num\":" + std::to_string(m.num) + ",\"ksize\":" + std::to_string(m.ksize) +
               ",\"seed\":" + std::to_string(m.seed) + ",\"max_hash\":" + std::to_string(m.max_hash) + ",\"mins\":";
        json_u64_array(out, m.mins);
        out += ",\"md5sum\":\"" + m.md5sum() + "\"";
        if (m.track) { out += ",\"abundances\":"; json_u64_array(out, m.abunds); }
        out += std::string(",\"molecule\":\"") + molecule_name(m.hash_function) + "\"}";
    }
    char vb[32];
    snprintf(vb, sizeof vb, "%.17g", sig.version);
    double back = strtod(vb, nullptr);
    for (int prec = 1; prec < 17; ++prec) {                // shortest representation that round-trips
        char t[32]; snprintf(t, sizeof t, "%.*g", prec, sig.version);
        if (strtod(t, nullptr) == sig.version) { memcpy(vb, t, sizeof t); break; }
    }
    (void)back;
    out += std::string("],\"version\":") + vb + "}";
}
std::string json_signatures(const SourmashSignature* const* sigs, size_t n) {
    // one string per signature, rendered by a few threads (digits + md5 are the whole cost)
    std::vector<std::string> parts(n);
    std::atomic<size_t> next{0};
    auto worker = [&] { for (;;) { size_t i = next.fetch_add(1); if (i >= n) return; json_signature(parts[i], *sigs[i]); } };
    const size_t nt = std::min<size_t>(n < 8 ? 1 : 16, std::max<unsigned>(std::thread::hardware_concurrency(), 1u));
    std::vector<std::thread> pool;
    for (size_t t = 1; t < nt; ++t) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
    size_t tot = 2 + n;
    for (auto& p : parts) tot += p.size();
    std::string out;
    out.reserve(tot);
    out.push_back('[');
    for (size_t i = 0; i < n; ++i) { if (i) out.push_back(','); out += parts[i]; }
    out.push_back(']');
    return out;
}
std::string gzip_bytes(const std::string& in, int level) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, level, Z_DEFLATED, 15 + 16, 8, Z_DEFAULT_STRATEGY) != Z_OK)
        fail(SOURMASH_ERROR_CODE_INTERNAL, "zlib deflateInit2 failed");
    std::string out(deflateBound(&zs, in.size()) + 32, '\0');
    zs.next_in = (Bytef*)in.data(); zs.avail_in = (uInt)in.size();
    zs.next_out = (Bytef*)&out[0]; zs.avail_out = (uInt)out.size();
    int r = deflate(&zs, Z_FINISH);
    deflateEnd(&zs);
    if (r != Z_STREAM_END) fail(SOURMASH_ERROR_CODE_INTERNAL, "zlib deflate failed");
    out.resize(zs.total_out);
    return out;
}
std::string gunzip_bytes(const uint8_t* p, size_t n) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 32) != Z_OK) fail(SOURMASH_ERROR_CODE_INTERNAL, "zlib inflateInit2 failed");
    std::string out;
    std::vector<char> buf(1 << 20);
    zs.next_in = (Bytef*)p; zs.avail_in = (uInt)n;
    int r;
    do {
        zs.next_out = (Bytef*)buf.data(); zs.avail_out = (uInt)buf.size();
        r = inflate(&zs, Z_NO_FLUSH);
        if (r != Z_OK && r != Z_STREAM_END) { inflateEnd(&zs); fail(SOURMASH_ERROR_CODE_NIFFLER_ERROR, "gzip stream is corrupt"); }
        out.append(buf.data(), buf.size() - zs.avail_out);
    } while (r != Z_STREAM_END);
    inflateEnd(&zs);
    return out;
}

// one host sketch object from row i of a parsed batch
MH mh_from_batch(const smb::SigBatch& B, size_t i) {
    const smb::SigSketch& sk = B.sketches[i];
    MH m;
    m.num = sk.num; m.ksize = sk.ksize; m.seed = sk.seed; m.max_hash = sk.max_hash;
    m.hash_function = (HashFunctions)sk.hash_function; m.track = sk.has_abund;
    m.mins.assign(B.mins.begin() + B.off[i], B.mins.begin() + B.off[i + 1]);
    if (sk.has_abund) m.abunds.assign(B.abunds.begin() + B.off[i], B.abunds.begin() + B.off[i + 1]);
    return m;
}
// sketch i with the metadata of the signature object it was stored in
SourmashSignature* sig_from_batch(const smb::SigBatch& B, size_t i) {
    const smb::SigRecord& r = B.sigs[B.sketches[i].sig_index];
    auto* sig = new SourmashSignature();
    sig->name = r.name; sig->filename = r.filename; sig->license = r.license; sig->email = r.email;
    sig->klass = r.klass; sig->hash_function = r.hash_function; sig->version = r.version;
    sig->sketches.push_back(mh_from_batch(B, i));
    return sig;
}
// Signature::load_signatures (signature.rs:583-658): one signature per sketch, filtered by ksize
// (as stored) and molecule type
SourmashSignature** sigs_from_batch(const smb::SigBatch& B, uintptr_t ksize, const char* select_moltype,
                                    uintptr_t* size) {
    int want_hf = 0;
    if (select_moltype) {
        std::string m(select_moltype);
        for (auto& c : m) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
        want_hf = m == "dna" ? 1 : m == "protein" ? 2 : m == "dayhoff" ? 3 : m == "hp" ? 4 : -1;
        if (want_hf < 0) fail(SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION, "Invalid hash function: \"" + std::string(select_moltype) + "\"");
    }
    std::vector<SourmashSignature*> out;
    for (size_t i = 0; i < B.sketches.size(); ++i) {
        const smb::SigSketch& sk = B.sketches[i];
        if (ksize != 0 && sk.ksize != ksize) continue;
        if (want_hf && (int)sk.hash_function != want_hf) continue;
        out.push_back(sig_from_batch(B, i));
    }
    *size = out.size();
    auto** arr = (SourmashSignature**)malloc(std::max<size_t>(out.size(), 1) * sizeof(void*));
    if (!out.empty()) memcpy(arr, out.data(), out.size() * sizeof(void*));
    return arr;
}
int default_threads() {
    unsigned n = std::thread::hardware_concurrency();
    return (int)std::min<unsigned>(std::max<unsigned>(n, 1u), 32u);
}

}  // namespace

extern "C" {


// ------------------------------------------------------------------------------------------
void sourmash_init(void) {}
void sourmash_err_clear(void) { t_has_error = false; }
SourmashErrorCode sourmash_err_get_last_code(void) { return t_has_error ? t_error.code : 0; }
SourmashStr sourmash_err_get_last_message(void) {
    if (t_has_error) return make_str(t_error.msg);
    SourmashStr r{nullptr, 0, false};
    return r;
}
SourmashStr sourmash_err_get_backtrace(void) { SourmashStr r{nullptr, 0, false}; return r; }
void sourmash_str_free(SourmashStr* s) {
    if (s && s->owned && s->data) { free(s->data); s->data = nullptr; s->len = 0; s->owned = false; }
}
SourmashStr sourmash_str_from_cstr(const char* s) { return make_str(s ? s : ""); }

uint64_t hash_murmur(const char* kmer, uint64_t seed) {
    return guarded<uint64_t>([&] { return murmur_on_gpu((const uint8_t*)kmer, strlen(kmer), seed); });
}

// residue encodings (ffi/minhash.rs:157-178): scalar table lookups on the tables the kernel uses
char sourmash_translate_codon(const char* codon) {
    return guarded<char>([&]() -> char {
        const size_t n = strlen(codon);
        if (n == 1) return 'X';                                            // encodings.rs:299-301
        if (n != 2 && n != 3)
            fail(SOURMASH_ERROR_CODE_INVALID_CODON_LENGTH, "Codon is invalid length: " + std::to_string(n));
        const smb::AaTables T = smb::build_aa_tables((int)HASH_FUNCTIONS_MURMUR64_PROTEIN);
        // no case folding here: translate_codon looks the bytes up as they are (encodings.rs:303-321)
        auto code = [&](char c) -> uint32_t { return (c >= 'a' && c <= 'z') ? 5u : T.base_code[(uint8_t)c]; };
        const uint32_t c2 = n == 3 ? code(codon[2]) : 4u;                  // two bases: third is 'N'
        return (char)T.codon[code(codon[0]) * 36 + code(codon[1]) * 6 + c2];
    });
}
char sourmash_aa_to_dayhoff(char aa) { return (char)smb::aa_reencode((uint8_t)aa, (int)HASH_FUNCTIONS_MURMUR64_DAYHOFF); }
char sourmash_aa_to_hp(char aa) { return (char)smb::aa_reencode((uint8_t)aa, (int)HASH_FUNCTIONS_MURMUR64_HP); }

// ------------------------------------------------------------------------------------------
SourmashKmerMinHash* kmerminhash_new(uint64_t scaled, uint32_t k, HashFunctions hash_function,
                                     uint64_t seed, bool track_abundance, uint32_t n) {
    MH* m = new MH();
    m->num = n; m->ksize = k; m->hash_function = hash_function; m->seed = seed;
    m->track = track_abundance; m->max_hash = max_hash_for_scaled(scaled);
    return m;
}
void kmerminhash_free(SourmashKmerMinHash* ptr) { delete ptr; }
void kmerminhash_slice_free(uint64_t* ptr, uintptr_t) { free(ptr); }

void kmerminhash_add_sequence(SourmashKmerMinHash* ptr, const char* sequence, bool force) {
    guarded_void([&] { mh_add_sequence(*ptr, (const uint8_t*)sequence, strlen(sequence), force); });
}
void kmerminhash_add_protein(SourmashKmerMinHash* ptr, const char* sequence) {
    guarded_void([&] { mh_add_aa(*ptr, (const uint8_t*)sequence, strlen(sequence), true); });
}

const uint64_t* kmerminhash_seq_to_hashes(SourmashKmerMinHash* ptr, const char* sequence,
                                          uintptr_t insize, bool force, bool bad_kmers_as_zeroes,
                                          bool is_protein, uintptr_t* size) {
    return guarded<const uint64_t*>([&]() -> const uint64_t* {
        // ffi/minhash.rs:63-99
        MH& mh = *ptr;
        if (is_protein || mh.hash_function != HASH_FUNCTIONS_MURMUR64_DNA) {
            std::vector<uint64_t> out = aa_seq_to_hashes(mh, (const uint8_t*)sequence, insize, is_protein,
                                                         force && bad_kmers_as_zeroes);
            return to_boxed(out, size);
        }
        std::vector<uint64_t> out;
        const size_t k = mh.ksize, len = insize;
        if (k > 0 && len >= k) {
            cudaStream_t s = need_gpu();
            const size_t nwin = len - k + 1;
            DevBuf<uint8_t> d_seq(len + 32, s);
            d_seq.upload((const uint8_t*)sequence, len);
            DevBuf<uint64_t> d_raw(nwin, s);
            uint64_t off = 0, ln = len;
            uint32_t tr[2] = {0, 0}, tg[2] = {0, 0};
            const int W = 64;
            tr[1] = (uint32_t)((len + (size_t)smb::hash_threads() * W - 1) / ((size_t)smb::hash_threads() * W));
            tg[1] = (uint32_t)((len + 255) / 256);
            DevBuf<uint64_t> d_off(1, s), d_len(1, s);
            DevBuf<uint32_t> d_tr(2, s), d_tg(2, s);
            d_off.upload(&off, 1); d_len.upload(&ln, 1); d_tr.upload(tr, 2); d_tg.upload(tg, 2);
            smb::HashLaunch L{};
            L.bases = d_seq.p; L.stream_off = d_off.p; L.stream_len = d_len.p; L.stream_row = nullptr;
            L.n_streams = 1; L.tile_start_rolled = d_tr.p; L.total_tiles_rolled = tr[1];
            L.tile_start_generic = d_tg.p; L.total_tiles_generic = tg[1];
            L.W = W; L.seed = mh.seed; L.max_hash = UINT64_MAX;
            smb::launch_window_hashes(L, mh.ksize, d_raw.p, s);
            CK(cudaGetLastError());
            std::vector<uint64_t> raw(nwin);
            d_raw.download(raw.data(), nwin);
            // validity needs the bases (a genuine hash of 0 is indistinguishable in `raw`)
            sync(s);
            const uint8_t* sq = (const uint8_t*)sequence;
            auto ok = [&](uint8_t c) { c &= 0xDF; return c == 'A' || c == 'C' || c == 'G' || c == 'T'; };
            size_t bad_until = 0;                       // windows < bad_until contain a bad base
            for (size_t p = 0; p + 1 < k; ++p) if (!ok(sq[p])) bad_until = p + 1;
            out.reserve(nwin);
            for (size_t w = 0; w < nwin; ++w) {
                if (!ok(sq[w + k - 1])) bad_until = w + k;
                if (w < bad_until) {
                    if (!force) {
                        std::string km((const char*)sq + w, k);
                        for (auto& c : km) if (c >= 'a' && c <= 'z') c -= 32;
                        fail(SOURMASH_ERROR_CODE_INVALID_DNA, "invalid DNA character in input k-mer: " + km);
                    }
                    if (bad_kmers_as_zeroes) out.push_back(0);
                } else if (raw[w] != 0 || (force && bad_kmers_as_zeroes)) {
                    out.push_back(raw[w]);
                }
            }
        }
        return to_boxed(out, size);
    });
}

void kmerminhash_clear(SourmashKmerMinHash* ptr) { ptr->mins.clear(); ptr->abunds.clear(); }
void kmerminhash_add_hash(SourmashKmerMinHash* ptr, uint64_t h) { ptr->add_hash_with_abundance(h, 1); }
void kmerminhash_add_hash_with_abundance(SourmashKmerMinHash* ptr, uint64_t h, uint64_t abundance) {
    ptr->add_hash_with_abundance(h, abundance);
}
void kmerminhash_add_word(SourmashKmerMinHash* ptr, const char* word) {
    guarded_void([&] {
        ptr->add_hash_with_abundance(murmur_on_gpu((const uint8_t*)word, strlen(word), ptr->seed), 1);
    });
}
void kmerminhash_add_many(SourmashKmerMinHash* ptr, const uint64_t* hashes_ptr, uintptr_t insize) {
    for (uintptr_t i = 0; i < insize; ++i) ptr->add_hash_with_abundance(hashes_ptr[i], 1);
}
void kmerminhash_add_from(SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other) {
    for (uint64_t h : other->mins) ptr->add_hash_with_abundance(h, 1);
}
void kmerminhash_remove_hash(SourmashKmerMinHash* ptr, uint64_t h) { ptr->remove_hash(h); }
void kmerminhash_remove_many(SourmashKmerMinHash* ptr, const uint64_t* hashes_ptr, uintptr_t insize) {
    for (uintptr_t i = 0; i < insize; ++i) ptr->remove_hash(hashes_ptr[i]);
}
void kmerminhash_remove_from(SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other) {
    for (uint64_t h : other->mins) ptr->remove_hash(h);
}
const uint64_t* kmerminhash_get_mins(const SourmashKmerMinHash* ptr, uintptr_t* size) {
    return to_boxed(ptr->mins, size);
}
uintptr_t kmerminhash_get_mins_size(const SourmashKmerMinHash* ptr) { return ptr->mins.size(); }
const uint64_t* kmerminhash_get_abunds(SourmashKmerMinHash* ptr, uintptr_t* size) {
    if (!ptr->track) {
        set_error(SOURMASH_ERROR_CODE_PANIC, "panic: not implemented (sketch does not track abundance)");
        *size = 0;
        return nullptr;
    }
    return to_boxed(ptr->abunds, size);
}
void kmerminhash_set_abundances(SourmashKmerMinHash* ptr, const uint64_t* hashes_ptr,
                                const uint64_t* abunds_ptr, uintptr_t insize, bool clear) {
    // ffi/minhash.rs:269-301: sort pairs, optional clear, add_many_with_abund
    std::vector<std::pair<uint64_t, uint64_t>> pairs(insize);
    for (uintptr_t i = 0; i < insize; ++i) pairs[i] = {hashes_ptr[i], abunds_ptr[i]};
    std::sort(pairs.begin(), pairs.end());
    if (clear) { ptr->mins.clear(); ptr->abunds.clear(); }
    for (auto& pr : pairs) ptr->add_hash_with_abundance(pr.first, pr.second);
}
SourmashStr kmerminhash_md5sum(const SourmashKmerMinHash* ptr) { return make_str(ptr->md5sum()); }
bool kmerminhash_is_protein(const SourmashKmerMinHash* ptr) { return ptr->hash_function == HASH_FUNCTIONS_MURMUR64_PROTEIN; }
bool kmerminhash_dayhoff(const SourmashKmerMinHash* ptr) { return ptr->hash_function == HASH_FUNCTIONS_MURMUR64_DAYHOFF; }
bool kmerminhash_hp(const SourmashKmerMinHash* ptr) { return ptr->hash_function == HASH_FUNCTIONS_MURMUR64_HP; }
uint64_t kmerminhash_seed(const SourmashKmerMinHash* ptr) { return ptr->seed; }
bool kmerminhash_track_abundance(const SourmashKmerMinHash* ptr) { return ptr->track; }
void kmerminhash_disable_abundance(SourmashKmerMinHash* ptr) { ptr->track = false; ptr->abunds.clear(); }
void kmerminhash_enable_abundance(SourmashKmerMinHash* ptr) {
    if (!ptr->mins.empty()) {     // minhash.rs:265-275
        set_error(SOURMASH_ERROR_CODE_NON_EMPTY_MIN_HASH, "Can only set \"track_abundance=True\" if the MinHash is empty");
        return;
    }
    ptr->track = true;
    ptr->abunds.clear();
}
uint32_t kmerminhash_num(const SourmashKmerMinHash* ptr) { return ptr->num; }
uint32_t kmerminhash_ksize(const SourmashKmerMinHash* ptr) { return ptr->ksize; }
uint64_t kmerminhash_max_hash(const SourmashKmerMinHash* ptr) { return ptr->max_hash; }
HashFunctions kmerminhash_hash_function(const SourmashKmerMinHash* ptr) { return ptr->hash_function; }
void kmerminhash_hash_function_set(SourmashKmerMinHash* ptr, HashFunctions hash_function) {
    if (ptr->hash_function == hash_function) return;      // minhash.rs:247-259
    if (!ptr->mins.empty()) {
        set_error(SOURMASH_ERROR_CODE_NON_EMPTY_MIN_HASH, "Can only set \"hash_function\" if the MinHash is empty");
        return;
    }
    ptr->hash_function = hash_function;
}
void kmerminhash_merge(SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other) {
    guarded_void([&] { ptr->merge(*other); });
}
bool kmerminhash_is_compatible(const SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other) {
    try { ptr->check_compatible(*other); return true; } catch (const SmbError&) { return false; }
}
uint64_t kmerminhash_count_common(const SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other,
                                  bool downsample) {
    return guarded<uint64_t>([&] { return mh_count_common(*ptr, *other, downsample); });
}
SourmashKmerMinHash* kmerminhash_intersection(const SourmashKmerMinHash* ptr,
                                              const SourmashKmerMinHash* other) {
    return guarded<SourmashKmerMinHash*>([&] { return mh_intersection(*ptr, *other); });
}
uint64_t kmerminhash_intersection_union_size(const SourmashKmerMinHash* ptr,
                                             const SourmashKmerMinHash* other, uint64_t* union_size) {
    // ffi/minhash.rs:443-457: incompatibility is swallowed -> (0, 0); GPU failures still raise
    *union_size = 0;
    try {
        ptr->check_compatible(*other);
    } catch (const SmbError&) {
        return 0;
    }
    return guarded<uint64_t>([&] {
        PairCounts c = mh_intersection_size(*ptr, *other);
        *union_size = c.usize;
        return c.common;
    });
}
double kmerminhash_jaccard(const SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other) {
    return guarded<double>([&] { return mh_jaccard(*ptr, *other); });
}
double kmerminhash_similarity(const SourmashKmerMinHash* ptr, const SourmashKmerMinHash* other,
                              bool ignore_abundance, bool downsample) {
    return guarded<double>([&] { return mh_similarity(*ptr, *other, ignore_abundance, downsample); });
}
double kmerminhash_angular_similarity(const SourmashKmerMinHash* ptr,
                                      const SourmashKmerMinHash* other) {
    return guarded<double>([&] { return mh_angular(*ptr, *other); });
}

// ------------------------------------------------------------------------------------------
// Signature subset (ffi/signature.rs:24-217)
// ------------------------------------------------------------------------------------------
SourmashSignature* signature_new(void) { return new SourmashSignature(); }
void signature_free(SourmashSignature* ptr) { delete ptr; }
SourmashSignature* signature_from_params(const SourmashComputeParameters* p) {
    // cmd.rs:109-188 build_template: one sketch per ksize for each enabled molecule type
    return guarded<SourmashSignature*>([&]() -> SourmashSignature* {
        auto* sig = new SourmashSignature();
        for (uint32_t k : p->ksizes) {                      // per ksize: protein, dayhoff, hp, dna
            const std::pair<bool, HashFunctions> kinds[4] = {
                {p->protein, HASH_FUNCTIONS_MURMUR64_PROTEIN}, {p->dayhoff, HASH_FUNCTIONS_MURMUR64_DAYHOFF},
                {p->hp, HASH_FUNCTIONS_MURMUR64_HP}, {p->dna, HASH_FUNCTIONS_MURMUR64_DNA}};
            for (const auto& kind : kinds) {
                if (!kind.first) continue;
                MH m;
                m.num = p->num_hashes; m.ksize = k; m.seed = p->seed; m.track = p->track_abundance;
                m.hash_function = kind.second;
                m.max_hash = max_hash_for_scaled(p->scaled);
                sig->sketches.push_back(m);
            }
        }
        return sig;
    });
}
uintptr_t signature_len(const SourmashSignature* ptr) { return ptr->sketches.size(); }
bool signature_eq(const SourmashSignature* a, const SourmashSignature* b) {
    // signature.rs:869-888 (PartialEq): class, email, hash_function, filename and name, and the FIRST sketch of each --
    // sketches compare by md5sum (sketch/minhash.rs:66-71: ksize + mins; abundances, seed and max_hash do not enter)
    const bool metadata = a->klass == b->klass && a->email == b->email && a->hash_function == b->hash_function &&
                          a->filename == b->filename && a->name == b->name;
    if (a->sketches.empty() || b->sketches.empty()) return metadata;     // (the reference indexes signatures[0] and panics here)
    return metadata && a->sketches[0].md5sum() == b->sketches[0].md5sum();
}
void signature_add_sequence(SourmashSignature* ptr, const char* sequence, bool force) {
    // signature.rs:661-677: every sketch of the signature sees the sequence.  One upload, one
    // hash launch per ksize.
    guarded_void([&] {
        size_t len = strlen(sequence);
        auto& sk = ptr->sketches;
        bool groupable = force && sk.size() > 1;
        for (auto& mh : sk)
            groupable = groupable && mh.hash_function == HASH_FUNCTIONS_MURMUR64_DNA && mh.num == sk[0].num &&
                        mh.max_hash == sk[0].max_hash && mh.seed == sk[0].seed && mh.track == sk[0].track &&
                        mh.ksize > 0;
        if (groupable) {
            std::vector<MH*> group;
            for (auto& mh : sk) if (len >= mh.ksize) group.push_back(&mh);
            if (!group.empty()) add_sequence_group(group, (const uint8_t*)sequence, len);
        } else {
            for (auto& mh : sk) mh_add_sequence(mh, (const uint8_t*)sequence, len, force);
        }
    });
}
void signature_add_protein(SourmashSignature* ptr, const char* sequence) {
    // signature.rs:679-697: every sketch of the signature sees the residues
    guarded_void([&] {
        const size_t len = strlen(sequence);
        for (auto& mh : ptr->sketches) mh_add_aa(mh, (const uint8_t*)sequence, len, true);
    });
}
SourmashKmerMinHash* signature_first_mh(const SourmashSignature* ptr) {
    // ffi/signature.rs:169-185 returns a clone
    if (ptr->sketches.empty()) {
        set_error(SOURMASH_ERROR_CODE_INTERNAL, "internal error: \"found unsupported sketch type\"");
        return nullptr;
    }
    return new MH(ptr->sketches[0]);
}
SourmashKmerMinHash** signature_get_mhs(const SourmashSignature* ptr, uintptr_t* size) {
    size_t n = ptr->sketches.size();
    SourmashKmerMinHash** arr = (SourmashKmerMinHash**)malloc(std::max<size_t>(n, 1) * sizeof(void*));
    for (size_t i = 0; i < n; ++i) arr[i] = new MH(ptr->sketches[i]);
    *size = n;
    return arr;
}
// frees the pointer ARRAY signature_get_mhs returned (the sketches it points at are owned by the caller)
void smb_mh_array_free(SourmashKmerMinHash** arr) { free(arr); }
void signature_set_mh(SourmashSignature* ptr, const SourmashKmerMinHash* other) {
    ptr->sketches.clear();
    ptr->sketches.push_back(*other);
}
void signature_push_mh(SourmashSignature* ptr, const SourmashKmerMinHash* other) {
    ptr->sketches.push_back(*other);
}
SourmashStr signature_get_name(const SourmashSignature* ptr) { return make_str(ptr->name); }
SourmashStr signature_get_filename(const SourmashSignature* ptr) { return make_str(ptr->filename); }
SourmashStr signature_get_license(const SourmashSignature* ptr) { return make_str(ptr->license); }
void signature_set_name(SourmashSignature* ptr, const char* name) { ptr->name = name ? name : ""; }
void signature_set_filename(SourmashSignature* ptr, const char* name) { ptr->filename = name ? name : ""; }

// ------------------------------------------------------------------------------------------
// ComputeParameters (ffi/cmd/compute.rs:14-170)
// ------------------------------------------------------------------------------------------
SourmashComputeParameters* computeparams_new(void) { return new SourmashComputeParameters(); }
void computeparams_free(SourmashComputeParameters* ptr) { delete ptr; }
const uint32_t* computeparams_ksizes(const SourmashComputeParameters* ptr, uintptr_t* size) {
    size_t n = ptr->ksizes.size();
    uint32_t* p = (uint32_t*)malloc(std::max<size_t>(n, 1) * 4);
    if (n) memcpy(p, ptr->ksizes.data(), n * 4);
    *size = n;
    return p;
}
void computeparams_ksizes_free(uint32_t* ptr, uintptr_t) { free(ptr); }
void computeparams_set_ksizes(SourmashComputeParameters* ptr, const uint32_t* ksizes_ptr, uintptr_t insize) {
    ptr->ksizes.assign(ksizes_ptr, ksizes_ptr + insize);
}
bool computeparams_dna(const SourmashComputeParameters* p) { return p->dna; }
bool computeparams_protein(const SourmashComputeParameters* p) { return p->protein; }
bool computeparams_dayhoff(const SourmashComputeParameters* p) { return p->dayhoff; }
bool computeparams_hp(const SourmashComputeParameters* p) { return p->hp; }
bool computeparams_track_abundance(const SourmashComputeParameters* p) { return p->track_abundance; }
uint32_t computeparams_num_hashes(const SourmashComputeParameters* p) { return p->num_hashes; }
uint64_t computeparams_scaled(const SourmashComputeParameters* p) { return p->scaled; }
uint64_t computeparams_seed(const SourmashComputeParameters* p) { return p->seed; }
void computeparams_set_dna(SourmashComputeParameters* p, bool v) { p->dna = v; }
void computeparams_set_protein(SourmashComputeParameters* p, bool v) { p->protein = v; }
void computeparams_set_dayhoff(SourmashComputeParameters* p, bool v) { p->dayhoff = v; }
void computeparams_set_hp(SourmashComputeParameters* p, bool v) { p->hp = v; }
void computeparams_set_track_abundance(SourmashComputeParameters* p, bool v) { p->track_abundance = v; }
void computeparams_set_num_hashes(SourmashComputeParameters* p, uint32_t num) { p->num_hashes = num; }
void computeparams_set_scaled(SourmashComputeParameters* p, uint64_t scaled) { p->scaled = scaled; }
void computeparams_set_seed(SourmashComputeParameters* p, uint64_t new_seed) { p->seed = new_seed; }

// ==========================================================================================
// Part 2: batched entry points
// ==========================================================================================
int32_t smb_device_count(void) { probe_devices(); return g_device_count; }
const char* smb_device_probe_error(void) { probe_devices(); return g_probe_error.c_str(); }
void smb_pow_f64(const double* x, double e, double* out, uintptr_t n) {     // host libm, element by element: what CPython's float_pow calls
    for (uintptr_t i = 0; i < n; ++i) out[i] = ::pow(x[i], e);
}
void smb_set_device(int32_t device) { t_device = device; }
void smb_set_stream(void* cuda_stream) { t_stream = (cudaStream_t)cuda_stream; }
void smb_synchronize(void) { guarded_void([&] { cudaStream_t s = need_gpu(); sync(s); }); }
uint64_t smb_kernel_launches(void) { return smb::g_launches.load(); }
void smb_set_profiling(bool on) { t_profiling = on; }
double smb_last_kernel_ms(int32_t which) {
    return guarded<double>([&] { return which == 0 ? t_timer_pairwise.ms() : t_timer_hash.ms(); });
}
void smb_last_compare_plan(double* out4) {
    out4[0] = t_last_join.use ? 1.0 : 0.0;
    out4[1] = t_last_join.increments;
    out4[2] = t_last_join.elements;
    out4[3] = (double)t_last_join.max_group;
}
void* smb_alloc_pinned(uintptr_t nbytes) {
    return guarded<void*>([&]() -> void* {
        need_gpu();
        void* p = nullptr;
        CK(cudaHostAlloc(&p, std::max<size_t>(nbytes, 16), cudaHostAllocDefault));
        return p;
    });
}
void smb_free_pinned(void* ptr) { if (ptr) cudaFreeHost(ptr); }
uint64_t smb_max_hash_for_scaled(uint64_t scaled) { return max_hash_for_scaled(scaled); }

SmbSketchSet* smb_sketchset_from_host(const uint64_t* hashes, const uint64_t* offsets,
                                      uintptr_t n_rows, const uint64_t* abunds) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        cudaStream_t s = need_gpu();
        auto set = std::make_unique<SmbSketchSet>();
        set->n_rows = n_rows;
        set->h_off.assign(offsets, offsets + n_rows + 1);
        uint64_t total = set->total();
        set->own_off.alloc(n_rows + 1, s);
        set->own_off.upload(offsets, n_rows + 1);
        set->own_hashes.alloc(total, s);
        set->own_hashes.upload(hashes, total);
        if (abunds) { set->own_abunds.alloc(total, s); set->own_abunds.upload(abunds, total); }
        sync(s);
        set->d_off = set->own_off.p; set->d_hashes = set->own_hashes.p;
        set->d_abunds = abunds ? set->own_abunds.p : nullptr;
        set->finish_offsets();
        return set.release();
    });
}
SmbSketchSet* smb_sketchset_from_device(const uint64_t* d_hashes, const uint64_t* d_offsets,
                                        const uint64_t* h_offsets, uintptr_t n_rows) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        need_gpu();
        auto set = std::make_unique<SmbSketchSet>();
        set->n_rows = n_rows;
        set->h_off.assign(h_offsets, h_offsets + n_rows + 1);
        set->d_hashes = d_hashes; set->d_off = d_offsets;
        set->finish_offsets();
        return set.release();
    });
}
void smb_sketchset_free(SmbSketchSet* set) { delete set; }
uintptr_t smb_sketchset_len(const SmbSketchSet* set) { return set->n_rows; }
uint64_t smb_sketchset_total_hashes(const SmbSketchSet* set) { return set->total(); }
bool smb_sketchset_has_abunds(const SmbSketchSet* set) { return set->d_abunds != nullptr; }
void smb_sketchset_offsets(const SmbSketchSet* set, uint64_t* offsets_out) {
    memcpy(offsets_out, set->h_off.data(), (set->n_rows + 1) * 8);
}
void smb_sketchset_to_host(const SmbSketchSet* set, uint64_t* hashes_out, uint64_t* abunds_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        uint64_t total = set->total();
        if (total && hashes_out) CK(cudaMemcpyAsync(hashes_out, set->d_hashes, total * 8, cudaMemcpyDeviceToHost, s));
        if (total && abunds_out && set->d_abunds)
            CK(cudaMemcpyAsync(abunds_out, set->d_abunds, total * 8, cudaMemcpyDeviceToHost, s));
        sync(s);
    });
}
void smb_sketchset_copy_to_device(const SmbSketchSet* set, uint64_t* d_hashes_out, uint64_t* d_offsets_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        uint64_t total = set->total();
        if (total && d_hashes_out)
            CK(cudaMemcpyAsync(d_hashes_out, set->d_hashes, total * 8, cudaMemcpyDeviceToDevice, s));
        if (d_offsets_out)
            CK(cudaMemcpyAsync(d_offsets_out, set->d_off, (set->n_rows + 1) * 8, cudaMemcpyDeviceToDevice, s));
    });
}
const uint64_t* smb_sketchset_device_hashes(const SmbSketchSet* set) { return set->d_hashes; }
const uint64_t* smb_sketchset_device_offsets(const SmbSketchSet* set) { return set->d_off; }

SmbSketchSet* smb_sketchset_downsample(const SmbSketchSet* set, uint64_t max_hash) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        auto out = std::make_unique<SmbSketchSet>();
        out->n_rows = n;
        out->h_off.assign(n + 1, 0);
        DevBuf<uint32_t> d_cnt(n, s);
        smb::launch_row_prefix_counts(set->d_hashes, set->d_off, (int)n, max_hash, d_cnt.p, s);
        std::vector<uint32_t> cnt(n);
        d_cnt.download(cnt.data(), n);
        sync(s);
        for (size_t r = 0; r < n; ++r) out->h_off[r + 1] = out->h_off[r] + cnt[r];
        out->own_off.alloc(n + 1, s);
        out->own_off.upload(out->h_off.data(), n + 1);
        out->own_hashes.alloc(out->total(), s);
        smb::launch_compact_rows(set->d_hashes, set->d_off, d_cnt.p, out->own_off.p, out->own_hashes.p, (int)n, s);
        if (set->d_abunds) {
            out->own_abunds.alloc(out->total(), s);
            smb::launch_compact_rows(set->d_abunds, set->d_off, d_cnt.p, out->own_off.p, out->own_abunds.p, (int)n, s);
        }
        CK(cudaGetLastError());
        sync(s);
        out->d_off = out->own_off.p; out->d_hashes = out->own_hashes.p;
        out->d_abunds = set->d_abunds ? out->own_abunds.p : nullptr;
        out->finish_offsets();
        return out.release();
    });
}

// rows `rows[0..n)` of a resident set (any order, repeats allowed) as a new resident set -- e.g. the few candidates of
// a sharded prefetch that are replicated on every rank for the gather rounds
SmbSketchSet* smb_sketchset_take_rows(const SmbSketchSet* set, const uint32_t* rows, uintptr_t n) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        cudaStream_t s = need_gpu();
        auto out = std::make_unique<SmbSketchSet>();
        out->n_rows = n;
        out->h_off.assign(n + 1, 0);
        std::vector<uint64_t> src_off(n + 1, 0);
        std::vector<uint32_t> len(n + 1, 0);
        for (size_t i = 0; i < n; ++i) {
            if (rows[i] >= set->n_rows) fail(SOURMASH_ERROR_CODE_MSG, "row index out of range");
            src_off[i] = set->h_off[rows[i]];
            len[i] = (uint32_t)(set->h_off[rows[i] + 1] - set->h_off[rows[i]]);
            out->h_off[i + 1] = out->h_off[i] + len[i];
        }
        DevBuf<uint64_t> d_src(n + 1, s);
        DevBuf<uint32_t> d_len(n + 1, s);
        d_src.upload(src_off.data(), n + 1);
        d_len.upload(len.data(), n + 1);
        out->own_off.alloc(n + 1, s);
        out->own_off.upload(out->h_off.data(), n + 1);
        out->own_hashes.alloc(std::max<uint64_t>(out->total(), 1), s);
        if (n) smb::launch_compact_rows(set->d_hashes, d_src.p, d_len.p, out->own_off.p, out->own_hashes.p, (int)n, s);
        if (set->d_abunds) {
            out->own_abunds.alloc(std::max<uint64_t>(out->total(), 1), s);
            if (n) smb::launch_compact_rows(set->d_abunds, d_src.p, d_len.p, out->own_off.p, out->own_abunds.p, (int)n, s);
        }
        CK(cudaGetLastError());
        sync(s);
        out->d_off = out->own_off.p; out->d_hashes = out->own_hashes.p;
        out->d_abunds = set->d_abunds ? out->own_abunds.p : nullptr;
        out->finish_offsets();
        return out.release();
    });
}

static SketchParams make_params(const uint32_t* ksizes, uintptr_t n_ksizes, uint64_t scaled,
                                uint32_t num, uint64_t seed, bool track) {
    SketchParams P;
    P.ksizes.assign(ksizes, ksizes + n_ksizes);
    P.max_hash = max_hash_for_scaled(scaled);
    P.num = num; P.seed = seed; P.track = track;
    return P;
}

SmbSketchSet* smb_sketch_sequences(const uint8_t* seqs, const uint64_t* seq_offsets,
                                   uintptr_t n_seqs, const uint32_t* seq_to_sketch,
                                   uintptr_t n_sketches, const uint32_t* ksizes,
                                   uintptr_t n_ksizes, uint64_t scaled, uint32_t num, uint64_t seed,
                                   bool track_abundance, uint64_t* n_kmers_out) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        cudaStream_t s = need_gpu();
        const uint64_t total = n_seqs ? seq_offsets[n_seqs] : 0;
        DevBuf<uint8_t> d_bases(total + 32, s);
        StreamList in;
        in.d_bases = d_bases.p;
        in.h_bases = seqs;                           // uploaded in groups, overlapped with hashing
        in.total_bytes = total;
        in.off.assign(seq_offsets, seq_offsets + n_seqs);
        in.len.resize(n_seqs);
        for (size_t i = 0; i < n_seqs; ++i) in.len[i] = seq_offsets[i + 1] - seq_offsets[i];
        if (seq_to_sketch) in.row.assign(seq_to_sketch, seq_to_sketch + n_seqs);
        in.n_sketches = seq_to_sketch ? n_sketches : n_seqs;
        SketchParams P = make_params(ksizes, n_ksizes, scaled, num, seed, track_abundance);
        return sketch_streams(in, P, s, n_kmers_out).release();
    });
}

SmbSketchSet* smb_sketch_sequences_aa(const uint8_t* seqs, const uint64_t* seq_offsets,
                                      uintptr_t n_seqs, const uint32_t* seq_to_sketch,
                                      uintptr_t n_sketches, const uint32_t* ksizes,
                                      uintptr_t n_ksizes, HashFunctions hash_function,
                                      bool input_is_protein, uint64_t scaled, uint32_t num,
                                      uint64_t seed, bool track_abundance, uint64_t* n_kmers_out) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        if (hash_function != HASH_FUNCTIONS_MURMUR64_PROTEIN && hash_function != HASH_FUNCTIONS_MURMUR64_DAYHOFF &&
            hash_function != HASH_FUNCTIONS_MURMUR64_HP)
            fail(SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION, "Invalid hash function: \"DNA\"");
        cudaStream_t s = need_gpu();
        const uint64_t total = n_seqs ? seq_offsets[n_seqs] : 0;
        DevBuf<uint8_t> d_bases(total + 32, s);
        StreamList in;
        in.d_bases = d_bases.p;
        in.h_bases = seqs;
        in.total_bytes = total;
        in.off.assign(seq_offsets, seq_offsets + n_seqs);
        in.len.resize(n_seqs);
        for (size_t i = 0; i < n_seqs; ++i) in.len[i] = seq_offsets[i + 1] - seq_offsets[i];
        if (seq_to_sketch) in.row.assign(seq_to_sketch, seq_to_sketch + n_seqs);
        in.n_sketches = seq_to_sketch ? n_sketches : n_seqs;
        SketchParams P = make_params(ksizes, n_ksizes, scaled, num, seed, track_abundance);
        P.hash_function = hash_function;
        P.input_is_protein = input_is_protein;
        return sketch_streams(in, P, s, n_kmers_out).release();
    });
}

SmbSketchSet* smb_sketch_streams_dev(const uint8_t* d_bases, const uint64_t* h_stream_offsets,
                                     const uint64_t* h_stream_lens, uintptr_t n_streams,
                                     const uint32_t* ksizes, uintptr_t n_ksizes, uint64_t scaled,
                                     uint32_t num, uint64_t seed, bool track_abundance,
                                     uint64_t* n_kmers_out) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        cudaStream_t s = need_gpu();
        StreamList in;
        in.d_bases = d_bases;
        in.off.assign(h_stream_offsets, h_stream_offsets + n_streams);
        in.len.assign(h_stream_lens, h_stream_lens + n_streams);
        in.n_sketches = n_streams;
        SketchParams P = make_params(ksizes, n_ksizes, scaled, num, seed, track_abundance);
        return sketch_streams(in, P, s, n_kmers_out).release();
    });
}

void smb_pairwise_common(const SmbSketchSet* a, const SmbSketchSet* b, uint32_t num,
                         uint32_t* common_out, uint32_t* usize_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t nA = a->n_rows, nB = b ? b->n_rows : a->n_rows;
        if (nA == 0 || nB == 0) return;
        DevBuf<uint32_t> d_c(nA * nB, s), d_u;
        d_c.zero();
        if (num) { d_u.alloc(nA * nB, s); d_u.zero(); }
        pairwise_counts_dev(*a, b, num, d_c.p, num ? d_u.p : nullptr, nB, s);
        CK(cudaGetLastError());
        d_c.download(common_out, nA * nB);
        if (num && usize_out) d_u.download(usize_out, nA * nB);
        sync(s);
        if (!b) {   // mirror the strict upper triangle; diagonal = |A_i| (num: min(num,|A_i|))
            for (size_t i = 0; i < nA; ++i) {
                uint64_t li = a->h_off[i + 1] - a->h_off[i];
                if (num && li > num) li = num;
                common_out[i * nB + i] = (uint32_t)li;
                if (num && usize_out) usize_out[i * nB + i] = (uint32_t)li;
                for (size_t j = i + 1; j < nB; ++j) {
                    common_out[j * nB + i] = common_out[i * nB + j];
                    if (num && usize_out) usize_out[j * nB + i] = usize_out[i * nB + j];
                }
            }
        }
    });
}

void smb_pairwise_counts_shard_dev(const SmbSketchSet* set, uint32_t shard, uint32_t n_shards,
                                   uint32_t* d_common) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        if (set->n_rows == 0) return;
        if (n_shards == 0 || shard >= n_shards) fail(SOURMASH_ERROR_CODE_MSG, "bad shard index");
        pairwise_counts_dev(*set, nullptr, 0, d_common, nullptr, set->n_rows, s,
                            smb::TileShard{(int)shard, (int)n_shards});
        CK(cudaGetLastError());
    });
}

void smb_compare_counts_shard_dev(const SmbSketchSet* set, uint32_t shard, uint32_t n_shards, void* d_counts, uint32_t bits) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (n == 0) return;
        if (n_shards == 0 || shard >= n_shards) fail(SOURMASH_ERROR_CODE_MSG, "bad shard index");
        if (bits != 32 && bits != 16) fail(SOURMASH_ERROR_CODE_MSG, "counter width must be 32 or 16 bits");
        if (bits == 16 && set->max_len >= 65536) fail(SOURMASH_ERROR_CODE_MSG, "16-bit counters need rows shorter than 65536 hashes");
        const uint64_t mk = set_max_key(*set, s);
        if (smb::join_stripe_enabled() && set->total()) {
            t_last_join = plan_join(*set, mk, s);
            if (t_last_join.use) {
                smb::JoinStripe* js = nullptr;
                if (t_profiling) t_timer_pairwise.begin(s);
                CK(smb::join_stripe_create_shard(set->d_hashes, set->d_off, (int)n, set->total(), mk, (int)shard, (int)n_shards, &js, s));
                if (js) {
                    std::unique_ptr<smb::JoinStripe, void (*)(smb::JoinStripe*)> guard(js, smb::join_stripe_destroy);
                    CK(smb::join_stripe_counts(js, d_counts, (int)bits, s));
                    if (t_profiling) t_timer_pairwise.end(s);
                    return;
                }
                if (t_profiling) t_timer_pairwise.end(s);
            }
        }
        // tile kernel / global-reduction join: upper-triangle shards (u32), completed to whole rows, narrowed if asked
        DevBuf<uint32_t> wide;
        uint32_t* d32 = (uint32_t*)d_counts;
        if (bits == 16) { wide.alloc(n * n, s); d32 = wide.p; }
        CK(cudaMemsetAsync(d32, 0, n * n * sizeof(uint32_t), s));
        pairwise_counts_dev(*set, nullptr, 0, d32, nullptr, n, s, smb::TileShard{(int)shard, (int)n_shards});
        smb::launch_mirror_counts(d32, 32, (int)n, s);
        if (bits == 16) smb::launch_narrow_counts(d32, (uint64_t)n * n, (uint16_t*)d_counts, s);
        CK(cudaGetLastError());
        if (bits == 16) sync(s);                           // `wide` is released when this scope ends
    });
}

void smb_finalize_counts_rows_dev(const SmbSketchSet* set, const void* d_counts_rows, uint32_t bits, uint64_t row_begin,
                                  uint64_t row_end, double* d_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (row_end > n) row_end = n;
        if (row_begin >= row_end) return;
        smb::launch_finalize_counts_rows(d_counts_rows, (int)bits, set->d_off, (int)n, (int)row_begin, (int)row_end, d_out, s);
        CK(cudaGetLastError());
    });
}

void smb_finalize_jaccard_rows_dev(const SmbSketchSet* set, const uint32_t* d_common, uint64_t row_begin,
                                   uint64_t row_end, double* d_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (row_end > n) row_end = n;
        if (row_begin >= row_end) return;
        smb::launch_finalize_rows(d_common, n, set->d_off, (int)n, (int)row_begin, (int)row_end, d_out, s);
        CK(cudaGetLastError());
    });
}

// Stripe layout of the join (join_stripe.cuh, the default; SMB_JOIN_LAYOUT=plain switches it off): float64
// rows come straight out of the count kernel, block of rows by block of rows; with `host_out` every
// finished block is downloaded on the copy stream while the next one is counted.  Returns false when the
// layout does not apply (the caller continues with the global-reduction join).
static bool compare_jaccard_stripe(const SmbSketchSet* set, uint64_t max_key, double* d_out, double* host_out,
                                   cudaStream_t s) {
    const size_t n = set->n_rows;
    smb::JoinStripe* js = nullptr;
    if (t_profiling) t_timer_pairwise.begin(s);
    CK(smb::join_stripe_create(set->d_hashes, set->d_off, (int)n, set->total(), max_key, &js, s));
    if (!js) { if (t_profiling) t_timer_pairwise.end(s); return false; }
    std::unique_ptr<smb::JoinStripe, void (*)(smb::JoinStripe*)> guard(js, smb::join_stripe_destroy);
    if (!host_out) {
        CK(smb::join_stripe_rows(js, set->d_off, 0, (int)n, d_out, s));
        CK(smb::join_stripe_mirror(js, 0, (int)n, d_out, s));
        if (t_profiling) t_timer_pairwise.end(s);
        return true;
    }
    cudaStream_t cs = copy_stream();
    // the download (PCIe) takes several times longer than the counting: a small first block starts it early,
    // the later blocks are large enough to fill the GPU for a few waves of CTAs each
    const size_t per = std::max<size_t>((n + 7) / 8, 1);
    for (size_t r0 = 0; r0 < n; r0 += per) {
        const size_t r1 = std::min(n, r0 + per);
        CK(smb::join_stripe_rows(js, set->d_off, (int)r0, (int)r1, d_out + r0 * n, s));
        CK(smb::join_stripe_mirror(js, (int)r0, (int)r1, d_out, s));
        cudaEvent_t ev = pool_event();
        CK(cudaEventRecord(ev, s));
        CK(cudaStreamWaitEvent(cs, ev, 0));
        CK(cudaMemcpyAsync(host_out + r0 * n, d_out + r0 * n, (r1 - r0) * n * sizeof(double), cudaMemcpyDeviceToHost, cs));
    }
    if (t_profiling) t_timer_pairwise.end(s);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(cs));
    sync(s);
    return true;
}

static void compare_jaccard_impl(const SmbSketchSet* set, uint32_t num, double* d_out, cudaStream_t s) {
    const size_t n = set->n_rows;
    if (n == 0) return;
    if (num == 0 && smb::join_stripe_enabled()) {
        const uint64_t mk = set_max_key(*set, s);
        t_last_join = plan_join(*set, mk, s);
        if (t_last_join.use && compare_jaccard_stripe(set, mk, d_out, nullptr, s)) return;
    }
    DevBuf<uint32_t> d_c(n * n, s), d_u;
    if (num) d_u.alloc(n * n, s);
    pairwise_counts_dev(*set, nullptr, num, d_c.p, num ? d_u.p : nullptr, n, s);
    smb::launch_finalize_matrix(d_c.p, num ? d_u.p : nullptr, n, set->d_off, set->d_off, (int)n, (int)n,
                                num ? 1 : 0, true, d_out, s);
    CK(cudaGetLastError());
}

void smb_compare_jaccard_rows_dev(const SmbSketchSet* set, uint64_t row_begin, uint64_t row_end, double* d_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (row_end > n) row_end = n;
        if (row_begin >= row_end) return;
        const uint64_t mk = set_max_key(*set, s);
        if (smb::join_stripe_enabled() && set->total()) {
            // stripe layout: only the requested rows are counted (a rank of a multi-GPU compare takes
            // a block of rows and exchanges no counts)
            smb::JoinStripe* js = nullptr;
            if (t_profiling) t_timer_pairwise.begin(s);
            CK(smb::join_stripe_create(set->d_hashes, set->d_off, (int)n, set->total(), mk, &js, s));
            if (js) {
                std::unique_ptr<smb::JoinStripe, void (*)(smb::JoinStripe*)> guard(js, smb::join_stripe_destroy);
                smb::join_stripe_two_directions(js);           // a block of rows on its own has no rows above to mirror
                CK(smb::join_stripe_rows(js, set->d_off, (int)row_begin, (int)row_end, d_out, s));
                if (t_profiling) t_timer_pairwise.end(s);
                return;
            }
            if (t_profiling) t_timer_pairwise.end(s);
        }
        DevBuf<uint32_t> d_c(n * n, s);
        pairwise_counts_dev(*set, nullptr, 0, d_c.p, nullptr, n, s);
        smb::launch_finalize_rows(d_c.p, n, set->d_off, (int)n, (int)row_begin, (int)row_end, d_out, s);
        CK(cudaGetLastError());
    });
}

void smb_compare_jaccard_dev(const SmbSketchSet* set, uint32_t num, double* d_out) {
    guarded_void([&] { cudaStream_t s = need_gpu(); compare_jaccard_impl(set, num, d_out, s); });
}

void smb_compare_jaccard(const SmbSketchSet* set, uint32_t num, double* out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (n == 0) return;
        DevBuf<double> d_out(n * n, s);
        smb::PairwisePlan plan{};
        if (num == 0 && n >= 1024) {
            const uint64_t mk = set_max_key(*set, s);
            t_last_join = plan_join(*set, mk, s);
            if (t_last_join.use) {
                // counts by inverted join, then finalise blocks of rows and download each block on
                // the copy stream while the next one is being finalised
                if (smb::join_stripe_enabled() && compare_jaccard_stripe(set, mk, d_out.p, out, s)) return;
                DevBuf<uint32_t> d_c(n * n, s);
                cudaStream_t cs = copy_stream();
                if (t_profiling) t_timer_pairwise.begin(s);
                CK(cudaMemsetAsync(d_c.p, 0, n * n * sizeof(uint32_t), s));
                CK(smb::join_counts(set->d_hashes, set->d_off, (int)n, mk, 0, 1, d_c.p, n, s));
                if (t_profiling) t_timer_pairwise.end(s);
                const size_t per = (n + 7) / 8;
                for (size_t r0 = 0; r0 < n; r0 += per) {
                    const size_t r1 = std::min(n, r0 + per);
                    smb::launch_finalize_rows(d_c.p, n, set->d_off, (int)n, (int)r0, (int)r1, d_out.p + r0 * n, s);
                    cudaEvent_t ev = pool_event();
                    CK(cudaEventRecord(ev, s));
                    CK(cudaStreamWaitEvent(cs, ev, 0));
                    CK(cudaMemcpyAsync(out + r0 * n, d_out.p + r0 * n, (r1 - r0) * n * sizeof(double),
                                       cudaMemcpyDeviceToHost, cs));
                }
                CK(cudaGetLastError());
                CK(cudaStreamSynchronize(cs));
                sync(s);
                return;
            }
            plan = smb::plan_pairwise(set->max_len, mk, (int)n);
        }
        if (plan.tables_per_cta > 0) {
            // Large matrix: compute groups of row tiles in order and download every finished block
            // of rows on the copy stream while the next group is being computed (rows of group g
            // only need counts from groups <= g: c[min(i,j)][max(i,j)]).
            DevBuf<uint32_t> d_c(n * n, s);
            const int ta = plan.tables_per_cta;
            const int tiles = (int)((n + ta - 1) / ta);
            const int groups = 8;
            const int per = (tiles + groups - 1) / groups;
            cudaStream_t cs = copy_stream();
            if (t_profiling) t_timer_pairwise.begin(s);
            for (int t0 = 0; t0 < tiles; t0 += per) {
                const int cnt = std::min(per, tiles - t0);
                smb::launch_pairwise_tile(plan, set->d_hashes, set->d_off, (int)n, set->d_hashes, set->d_off, (int)n,
                                          d_c.p, n, true, smb::TileShard{t0, 1, cnt}, s);
                const size_t r0 = (size_t)t0 * ta, r1 = std::min(n, (size_t)(t0 + cnt) * ta);
                smb::launch_finalize_rows(d_c.p, n, set->d_off, (int)n, (int)r0, (int)r1, d_out.p + r0 * n, s);
                cudaEvent_t ev = pool_event();
                CK(cudaEventRecord(ev, s));
                CK(cudaStreamWaitEvent(cs, ev, 0));
                CK(cudaMemcpyAsync(out + r0 * n, d_out.p + r0 * n, (r1 - r0) * n * sizeof(double),
                                   cudaMemcpyDeviceToHost, cs));
            }
            if (t_profiling) t_timer_pairwise.end(s);
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(cs));
            sync(s);
            return;
        }
        compare_jaccard_impl(set, num, d_out.p, s);
        d_out.download(out, n * n);
        sync(s);
    });
}

void smb_compare_angular(const SmbSketchSet* set, double* out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = set->n_rows;
        if (n == 0) return;
        if (set->total() == 0) {                 // every sketch empty (no abundance buffer exists for zero hashes): all norms are 0,
            std::fill(out, out + n * n, 0.0);    // every pair is 0.0 (minhash.rs:674-676)
            return;
        }
        if (!set->d_abunds)
            fail(SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING, "sketch needs abundance for this operation");
        DevBuf<double> d_out(n * n, s);
        DevBuf<unsigned long long> d_sq(n, s);
        smb::launch_pairwise_angular(set->d_hashes, set->d_abunds, set->d_off, (int)n, d_sq.p, d_out.p, s);
        CK(cudaGetLastError());
        d_out.download(out, n * n);
        sync(s);
    });
}

// Launch-only variant for a query that (a) fits the tile kernel and (b) whose true length lives on
// the device: d_qoff = {0, n} is written by the producing kernel, `nq_cap` bounds n, `key_bound`
// bounds every key of the query.  No host synchronisation.
static void one_vs_many_small_async(const uint64_t* d_q, const uint64_t* d_qoff, size_t nq_cap,
                                    uint64_t key_bound, const SmbSketchSet& db, uint32_t* d_counts,
                                    cudaStream_t s) {
    const int nB = (int)db.n_rows;
    if (nB == 0) return;
    const uint64_t max_key = std::max(key_bound, set_max_key(db, s));
    smb::PairwisePlan one = smb::plan_pairwise(nq_cap, max_key, nB);
    one.tables_per_cta = 1;
    const size_t key_bytes = (size_t)(one.cap + 2) * 8;
    const uint64_t max_entries = std::min<uint64_t>((227 * 1024 - key_bytes) / 2 - 2, 60000);
    int sh = 0;
    while (sh < 63 && (max_key >> sh) >= max_entries) ++sh;
    one.shift = sh; one.nb = (int)((max_key >> sh) + 1);
    one.smem_bytes = key_bytes + ((size_t)one.nb + 2) * 2;
    // a few hundred candidate rows (the gather rounds): many small CTAs, each building the (small) table again, beat four
    // CTAs of 64 rows -- the launch is latency bound, not work bound
    one.cols_per_cta = std::max(nB < 4096 ? 8 : 64, std::min(512, (nB + SMB_SMS * 2 - 1) / (SMB_SMS * 2)));
    smb::launch_pairwise_tile(one, d_q, d_qoff, 1, db.d_hashes, db.d_off, nB, d_counts, (size_t)nB, false,
                              smb::TileShard{0, 1}, s);
}

static void one_vs_many_dev(const uint64_t* d_q, size_t nq, const SmbSketchSet& db, uint32_t* d_counts,
                            cudaStream_t s) {
    // query small enough for shared memory: it becomes the (single) table of the tile kernel;
    // otherwise a global-memory directory over the query.
    const int nB = (int)db.n_rows;
    if (nB == 0 || nq == 0) return;                  // callers zero the counters: nothing is shared
    if (db.index) {                                  // resident set with an inverted index: probe it
        smb::launch_index_count(db.index, d_q, nq, d_counts, s);
        CK(cudaGetLastError());
        return;
    }
    SmbSketchSet q;
    q.n_rows = 1; q.h_off = {0, (uint64_t)nq};
    q.own_off.alloc(2, s); q.own_off.upload(q.h_off.data(), 2);
    q.d_off = q.own_off.p; q.d_hashes = d_q; q.finish_offsets();
    const uint64_t q_max = set_max_key(q, s);
    const uint64_t max_key = std::max(q_max, set_max_key(db, s));
    smb::PairwisePlan plan = smb::plan_pairwise(nq, max_key, nB);
    if (plan.tables_per_cta > 0) {
        // query small enough for shared memory: it is the single table of the tile kernel
        smb::PairwisePlan one = smb::plan_pairwise(nq, max_key, nB);
        one.tables_per_cta = 1;
        {   // with one table the whole 227 KB is available: take the finest directory that fits
            const size_t key_bytes = (size_t)(one.cap + 2) * 8;
            const uint64_t max_entries = std::min<uint64_t>((227 * 1024 - key_bytes) / 2 - 2, 60000);
            int sh = 0;
            while (sh < 63 && (max_key >> sh) >= max_entries) ++sh;
            one.shift = sh; one.nb = (int)((max_key >> sh) + 1);
            one.smem_bytes = key_bytes + ((size_t)one.nb + 2) * 2;
        }
        one.cols_per_cta = std::max(64, std::min(512, (nB + SMB_SMS * 2 - 1) / (SMB_SMS * 2)));
        smb::launch_pairwise_tile(one, q.d_hashes, q.d_off, 1, db.d_hashes, db.d_off, nB, d_counts,
                                  (size_t)nB, false, smb::TileShard{0, 1}, s);
    } else {
        if (smb::range_search_enabled()) {
            // large query: stream the range-major copy of the resident set (built once, kept with the set)
            if (!db.range_major && !db.range_major_tried) {
                db.range_major_tried = true;
                CK(smb::range_major_build(db.d_hashes, db.d_off, nB, db.total(), set_max_key(db, s), &db.range_major, s));
            }
            if (db.range_major) {
                smb::launch_one_vs_many_range_major(db.range_major, d_q, nq, d_counts, s);
                CK(cudaGetLastError());
                sync(s);      // q's offsets upload reads a host temporary
                return;
            }
        }
        // directory over the query's own key range (subject keys beyond it are skipped)
        int nb_log2 = 12;
        while (nb_log2 < 26 && (1ull << nb_log2) < 2 * (uint64_t)nq) ++nb_log2;
        int shift = 0;
        while (shift < 63 && (q_max >> shift) >= (1ull << nb_log2)) ++shift;
        const uint64_t nb = (q_max >> shift) + 1;
        DevBuf<uint32_t> d_dir(nb + 2, s);
        smb::launch_build_global_dir(d_q, nq, shift, nb, d_dir.p, s);
        // L2-resident occupancy bitmap, 8x finer than the directory (1 byte per bucket)
        const int fine_log2 = 3;
        DevBuf<uint32_t> d_bm(((size_t)nb << fine_log2) / 32 + 2, s);
        d_bm.zero();
        smb::launch_build_query_bitmap(d_q, nq, shift, fine_log2, d_bm.p, s);
        smb::launch_one_vs_many_global(d_q, nq, d_dir.p, shift, nb, d_bm.p, fine_log2, db.d_hashes,
                                       db.d_off, nB, d_counts, s);
    }
    CK(cudaGetLastError());
    sync(s);      // q's offsets upload reads a host temporary
}

// Index.search_abund (index/__init__.py:172-200) over a resident set: every row's angular similarity with one abundance
// query, elements above max_hash left out on both sides (similarity(..., downsample=True) without a downsampled copy).
// One device pass (angular_search.cuh) computes the per-row terms; the scores are finalized here with libm.
void smb_search_angular(const SmbSketchSet* db, const uint64_t* q, const uint64_t* q_abunds, uintptr_t nq,
                        uint64_t max_hash, double* scores_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t n = db->n_rows;
        for (uintptr_t i = 1; i < nq; ++i)
            if (q[i] <= q[i - 1]) fail(SOURMASH_ERROR_CODE_MSG, "query hashes are not sorted and unique");
        if (n == 0) return;
        // the query cut at max_hash (a prefix) and its own sum of squares
        const uintptr_t nq_cut = (uintptr_t)(std::upper_bound(q, q + nq, max_hash) - q);
        uint64_t a_sq = 0;
        for (uintptr_t i = 0; i < nq_cut; ++i) a_sq += q_abunds[i] * q_abunds[i];
        if (db->total() == 0 || nq_cut == 0) {            // nothing on one side: every norm or every product is 0
            if (db->total() && !db->d_abunds)
                fail(SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING, "sketch needs abundance for this operation");
            std::fill(scores_out, scores_out + n, 0.0);
            return;
        }
        if (!db->d_abunds)
            fail(SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING, "sketch needs abundance for this operation");
        smb::AngularSearchArgs a{};
        a.q_has_max = q[nq_cut - 1] == UINT64_MAX;
        a.nq = nq_cut - (a.q_has_max ? 1 : 0);
        a.q_top = a.nq ? q[a.nq - 1] : 0;
        a.q_max_abund = a.q_has_max ? q_abunds[nq_cut - 1] : 0;
        std::vector<uint64_t> chunk(n + 1, 0);
        for (size_t i = 0; i < n; ++i)
            chunk[i + 1] = chunk[i] + (db->h_off[i + 1] - db->h_off[i] + smb::ANGULAR_CHUNK - 1) / smb::ANGULAR_CHUNK;
        DevBuf<uint64_t> d_q(a.nq, s), d_qa(a.nq, s), d_chunk(n + 1, s);
        d_q.upload(q, a.nq);
        d_qa.upload(q_abunds, a.nq);
        d_chunk.upload(chunk.data(), n + 1);
        DevBuf<unsigned long long> d_prod(n, s), d_bsq(n, s);
        a.q = d_q.p; a.qa = d_qa.p;
        a.h = db->d_hashes; a.ab = db->d_abunds; a.off = db->d_off;
        a.chunk_start = d_chunk.p; a.n_chunks = chunk[n]; a.n_rows = (int)n;
        a.max_hash = max_hash;
        a.prod = d_prod.p; a.bsq = d_bsq.p;
        if (t_profiling) t_timer_hash.begin(s);
        CK(smb::angular_search(a, s));
        if (t_profiling) t_timer_hash.end(s);
        std::vector<unsigned long long> prod(n), bsq(n);
        d_prod.download(prod.data(), n);
        d_bsq.download(bsq.data(), n);
        sync(s);
        for (size_t i = 0; i < n; ++i) scores_out[i] = angular_from_terms(prod[i], a_sq, bsq[i]);
    });
}

uint64_t smb_sketchset_build_index(SmbSketchSet* set) {
    return guarded<uint64_t>([&]() -> uint64_t {
        cudaStream_t s = need_gpu();
        if (set->index) return smb::db_index_n_keys(set->index);
        if (set->n_rows == 0 || set->total() == 0) return 0;
        const uint64_t mk = set_max_key(*set, s);
        smb::DbIndex* ix = nullptr;
        CK(smb::db_index_build(set->d_hashes, set->d_off, (int)set->n_rows, set->total(), mk, &ix, s));
        if (!ix) fail(SOURMASH_ERROR_CODE_MSG, "set too large for an inverted index (more than 2^31 - 1 hashes)");
        sync(s);
        set->index = ix;
        return smb::db_index_n_keys(ix);
    });
}
void smb_sketchset_drop_index(SmbSketchSet* set) {
    guarded_void([&] {
        if (set->index) { smb::db_index_destroy(set->index); set->index = nullptr; }
    });
}
bool smb_sketchset_has_index(const SmbSketchSet* set) { return set->index != nullptr; }

void smb_one_vs_many(const uint64_t* query, uintptr_t n_query, const SmbSketchSet* db,
                     uint32_t* common_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t nB = db->n_rows;
        if (nB == 0) return;
        DevBuf<uint64_t> d_q(n_query, s);
        d_q.upload(query, n_query);
        DevBuf<uint32_t> d_counts(nB, s);
        d_counts.zero();
        one_vs_many_dev(d_q.p, n_query, *db, d_counts.p, s);
        d_counts.download(common_out, nB);
        sync(s);
    });
}

// prefetch's matched / unmatched query hashes (commands.py: prefetch, ident_mh / noident_mh) as one device pass over the
// passing rows instead of a merge of the whole query per match
void smb_query_covered(const uint64_t* query, uintptr_t n_query, const SmbSketchSet* db, const uint32_t* rows,
                       uintptr_t n_rows, uint8_t* covered_out) {
    guarded_void([&] {
        for (uintptr_t i = 0; i < n_rows; ++i)
            if (rows[i] >= db->n_rows)
                fail(SOURMASH_ERROR_CODE_MSG, "row index " + std::to_string(rows[i]) + " out of range for a set of " +
                                                  std::to_string(db->n_rows) + " rows");
        for (uintptr_t i = 1; i < n_query; ++i)
            if (query[i] <= query[i - 1]) fail(SOURMASH_ERROR_CODE_MSG, "query hashes are not sorted and unique");
        std::fill(covered_out, covered_out + n_query, (uint8_t)0);
        if (n_query == 0 || n_rows == 0) return;
        cudaStream_t s = need_gpu();
        DevBuf<uint64_t> d_q(n_query, s);
        DevBuf<uint32_t> d_rows(n_rows, s);
        DevBuf<uint8_t> d_cov(n_query, s);
        d_q.upload(query, n_query);
        d_rows.upload(rows, n_rows);
        if (t_profiling) t_timer_hash.begin(s);
        CK(smb::launch_query_cover(d_q.p, n_query, query[n_query - 1], db->d_hashes, db->d_off, d_rows.p, n_rows,
                                   d_cov.p, s));
        if (t_profiling) t_timer_hash.end(s);
        d_cov.download(covered_out, n_query);
        sync(s);
    });
}

void smb_one_vs_many_dev(const uint64_t* d_query, uintptr_t n_query, const SmbSketchSet* db, uint32_t* d_common_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t nB = db->n_rows;
        if (nB == 0) return;
        CK(cudaMemsetAsync(d_common_out, 0, nB * sizeof(uint32_t), s));
        one_vs_many_dev(d_query, n_query, *db, d_common_out, s);
    });
}

// ---- gather as a session: the single-GPU loop and the sharded multi-GPU loop
// (sourmash_b200/distributed.py) are both built from these four steps.
SmbGatherState* smb_gather_begin_min(const uint64_t* query, uintptr_t n_query, const SmbSketchSet* db,
                                     uint32_t min_count) {
    return guarded<SmbGatherState*>([&]() -> SmbGatherState* {
        cudaStream_t s = need_gpu();
        auto st = std::make_unique<SmbGatherState>();
        st->db = db;
        st->nq = n_query;
        if (min_count < 1) min_count = 1;
        const size_t nB = db->n_rows;
        st->remaining = n_query;
        st->q.alloc(n_query, s); st->isect.alloc(std::max<size_t>(db->max_len, 1), s);
        st->q.upload(query, n_query);
        st->alive.alloc(n_query, s);
        CK(cudaMemsetAsync(st->alive.p, 1, std::max<size_t>(n_query, 1), s));
        st->counts.alloc(nB, s); st->d_n.alloc(2, s); st->d_best.alloc(2, s);
        st->counts.zero();
        // CounterGather.add (index/__init__.py:777-794): counters[j] = |query ∩ S_j|
        if (n_query && nB) one_vs_many_dev(st->q.p, n_query, *db, st->counts.p, s);
        // Rows whose overlap is below min_count can never be picked and their counters only
        // shrink: drop them once, so that every later round streams the surviving rows only
        // (the reference's counter holds prefetch matches only, index/__init__.py:302-320).
        std::vector<uint32_t> cnt(nB);
        st->counts.download(cnt.data(), nB);
        sync(s);
        std::vector<uint32_t> keep;
        for (size_t j = 0; j < nB; ++j) if (cnt[j] >= min_count) keep.push_back((uint32_t)j);
        if (!db->index && keep.size() * 4 < nB * 3) {      // (an indexed set is never streamed: keep it whole)
            const size_t m = keep.size();
            auto sub = std::make_unique<SmbSketchSet>();
            sub->n_rows = m;
            sub->h_off.assign(m + 1, 0);
            std::vector<uint64_t> src_off(m + 1, 0);
            std::vector<uint32_t> len(m + 1, 0), kept(m + 1, 0);
            for (size_t i = 0; i < m; ++i) {
                const size_t j = keep[i];
                src_off[i] = db->h_off[j];
                len[i] = (uint32_t)(db->h_off[j + 1] - db->h_off[j]);
                sub->h_off[i + 1] = sub->h_off[i] + len[i];
                kept[i] = cnt[j];
            }
            DevBuf<uint64_t> d_src(m + 1, s);
            DevBuf<uint32_t> d_len(m + 1, s);
            d_src.upload(src_off.data(), m + 1);
            d_len.upload(len.data(), m + 1);
            sub->own_off.alloc(m + 1, s);
            sub->own_off.upload(sub->h_off.data(), m + 1);
            sub->own_hashes.alloc(sub->total(), s);
            smb::launch_compact_rows(db->d_hashes, d_src.p, d_len.p, sub->own_off.p, sub->own_hashes.p, (int)m, s);
            st->counts.alloc(m, s);
            st->counts.upload(kept.data(), m);
            CK(cudaGetLastError());
            sync(s);
            sub->d_off = sub->own_off.p; sub->d_hashes = sub->own_hashes.p;
            sub->finish_offsets();
            st->rowmap = std::move(keep);
            st->sub = std::move(sub);
            st->db = st->sub.get();
        }
        st->delta.alloc(st->db->n_rows, s);
        return st.release();
    });
}

SmbGatherState* smb_gather_begin(const uint64_t* query, uintptr_t n_query, const SmbSketchSet* db) {
    return smb_gather_begin_min(query, n_query, db, 1);
}

void smb_gather_end(SmbGatherState* st) { delete st; }

// best remaining (count, row); lowest row index wins ties (Counter.most_common()[0], :841)
void smb_gather_peek(SmbGatherState* st, uint32_t* best_count, uint32_t* best_row) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        *best_count = 0; *best_row = 0;
        if (st->db->n_rows == 0) return;
        smb::launch_counter_update_argmax(st->counts.p, st->delta_pending ? st->delta.p : nullptr,
                                          (int)st->db->n_rows, st->d_best.p, s);
        st->delta_pending = false;
        unsigned long long best[2];
        st->d_best.download(best, 2);
        sync(s);
        *best_count = (uint32_t)best[0];
        *best_row = st->rowmap.empty() ? (uint32_t)best[1] : st->rowmap[(size_t)best[1]];
    });
}

// intersect = remaining query ∩ row `row` of the local database -> host buffer (capacity = |row|)
uintptr_t smb_gather_intersect(SmbGatherState* st, uint32_t row, uint64_t* out_hashes) {
    return guarded<uintptr_t>([&]() -> uintptr_t {
        cudaStream_t s = need_gpu();
        const SmbSketchSet* db = st->db;
        if (!st->rowmap.empty()) {           // caller's row -> compact row
            auto it = std::lower_bound(st->rowmap.begin(), st->rowmap.end(), row);
            if (it == st->rowmap.end() || *it != row) fail(SOURMASH_ERROR_CODE_MSG, "row is not an active gather candidate");
            row = (uint32_t)(it - st->rowmap.begin());
        }
        const uint64_t* r = db->d_hashes + db->h_off[row];
        const size_t rn = db->h_off[row + 1] - db->h_off[row];
        smb::launch_intersect_alive(st->q.p, st->nq, st->alive.p, r, rn, st->isect.p, st->d_n.p, s);
        uint32_t n = 0;
        st->d_n.download(&n, 1);
        sync(s);
        if (n && out_hashes) { CK(cudaMemcpyAsync(out_hashes, st->isect.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s)); sync(s); }
        return n;
    });
}

// consume (index/__init__.py:882-909): every counter -= |intersect ∩ S_j|; query -= intersect.
// `intersect` is a host array (it may come from another rank).  Returns the remaining query size.
uintptr_t smb_gather_apply(SmbGatherState* st, const uint64_t* intersect, uintptr_t n) {
    return guarded<uintptr_t>([&]() -> uintptr_t {
        cudaStream_t s = need_gpu();
        if (n == 0) return st->remaining;
        DevBuf<uint64_t> d_i(n, s);
        d_i.upload(intersect, n);
        st->delta.zero();
        if (st->db->n_rows) one_vs_many_dev(d_i.p, n, *st->db, st->delta.p, s);
        st->delta_pending = true;
        smb::launch_mark_dead(st->q.p, st->nq, st->alive.p, d_i.p, n, s);
        CK(cudaGetLastError());
        sync(s);                                   // d_i is released on return
        st->remaining = st->remaining > n ? st->remaining - n : 0;
        return st->remaining;
    });
}

uintptr_t smb_gather(const uint64_t* query, uintptr_t n_query, const SmbSketchSet* db,
                     uint32_t threshold, uint32_t* match_ids, uint32_t* isect_sizes,
                     uintptr_t max_rounds) {
    // CounterGather + GatherDatabases loop (index/__init__.py:777-909, search.py:877-949), all
    // state in HBM.  Per round: argmax (one 24-byte readback = the only synchronisation),
    // intersect kernel, one-vs-many of the intersection, flag the consumed hashes.
    if (db->n_rows == 0 || n_query == 0 || max_rounds == 0) return 0;
    if (threshold < 1) threshold = 1;
    SmbGatherState* st = smb_gather_begin_min(query, n_query, db, threshold);
    if (!st) return 0;
    return guarded<uintptr_t>([&]() -> uintptr_t {
        std::unique_ptr<SmbGatherState> owner(st);
        cudaStream_t s = need_gpu();
        const SmbSketchSet* cdb = st->db;
        if (cdb->n_rows == 0) return 0;
        const uint64_t q_max = query[n_query - 1];             // query is sorted: bounds every intersection
        const bool small_rows = smb::plan_pairwise(cdb->max_len, std::max(q_max, set_max_key(*cdb, s)),
                                                   (int)cdb->n_rows).tables_per_cta > 0;
        DevBuf<uint64_t> d_qoff(2, s);
        if (small_rows && !cdb->index && max_rounds <= 0xffffffffull) {
            // Rounds picked on the device (search_kernels.cuh): argmax + pick, intersect the picked row with the live
            // query (consuming its hashes on the spot), one-vs-many of the intersection over the candidates -- four launches
            // and a memset per round and NO readback; the host enqueues rounds in batches and looks at the pick counter once per batch.
            const uint32_t cap = (uint32_t)std::min<uint64_t>(max_rounds, cdb->n_rows);   // a row is picked at most once
            DevBuf<uint32_t> d_rows(cap + 1, s), d_sizes(cap + 1, s), d_state(2, s);
            d_state.zero();
            st->delta.zero();
            smb::GatherPicks g{d_rows.p, d_sizes.p, d_state.p, threshold, cap};
            uint32_t state[2] = {0, 0};
            const uint32_t batch = 16;
            for (uint32_t issued = 0; !state[1] && issued < cap + 1; issued += batch) {
                for (uint32_t k = 0; k < batch; ++k) {
                    smb::launch_counter_update_argmax_pick(st->counts.p, st->delta.p, (int)cdb->n_rows, g, s);
                    smb::launch_intersect_alive_pick(st->q.p, st->nq, st->alive.p, cdb->d_hashes, cdb->d_off, g, st->isect.p, st->d_n.p, s);
                    smb::launch_make_row_offsets(st->d_n.p, d_qoff.p, s);
                    st->delta.zero();
                    one_vs_many_small_async(st->isect.p, d_qoff.p, cdb->max_len, q_max, *cdb, st->delta.p, s);
                }
                CK(cudaGetLastError());
                d_state.download(state, 2);
                sync(s);
                if (state[0] >= cap) break;
            }
            const uint32_t rounds = state[0];
            std::vector<uint32_t> rows(rounds), sizes(rounds);
            if (rounds) { d_rows.download(rows.data(), rounds); d_sizes.download(sizes.data(), rounds); sync(s); }
            for (uint32_t r = 0; r < rounds; ++r) {
                match_ids[r] = st->rowmap.empty() ? rows[r] : st->rowmap[rows[r]];
                isect_sizes[r] = sizes[r];
            }
            return rounds;
        }
        DevBuf<unsigned long long> d_info(4, s);               // {best count, best row, previous |intersect|}
        uintptr_t rounds = 0;
        bool have_delta = false;
        while (rounds < max_rounds) {
            smb::launch_counter_update_argmax(st->counts.p, have_delta ? st->delta.p : nullptr, (int)cdb->n_rows,
                                              st->d_best.p, s);
            unsigned long long best[2];
            uint32_t prev_n = 0;
            st->d_best.download(best, 2);
            if (rounds) CK(cudaMemcpyAsync(&prev_n, st->d_n.p, 4, cudaMemcpyDeviceToHost, s));
            sync(s);
            if (rounds) {
                isect_sizes[rounds - 1] = prev_n;
                st->remaining = st->remaining > prev_n ? st->remaining - prev_n : 0;
                if (st->remaining == 0) break;
            }
            if (best[0] < threshold || best[0] == 0) break;
            const uint32_t row = (uint32_t)best[1];
            match_ids[rounds] = st->rowmap.empty() ? row : st->rowmap[row];
            isect_sizes[rounds] = (uint32_t)best[0];            // == |intersect|; confirmed next round
            ++rounds;
            const uint64_t* r = cdb->d_hashes + cdb->h_off[row];
            const size_t rn = cdb->h_off[row + 1] - cdb->h_off[row];
            smb::launch_intersect_alive(st->q.p, st->nq, st->alive.p, r, rn, st->isect.p, st->d_n.p, s);
            if (cdb->index) {                                   // probe the inverted index, length stays on the device
                st->delta.zero();
                smb::launch_index_count_n(cdb->index, st->isect.p, st->d_n.p, rn, st->delta.p, s);
                smb::launch_mark_dead_n(st->q.p, st->nq, st->alive.p, st->isect.p, st->d_n.p, s);
            } else if (small_rows) {
                smb::launch_make_row_offsets(st->d_n.p, d_qoff.p, s);
                st->delta.zero();
                one_vs_many_small_async(st->isect.p, d_qoff.p, rn, q_max, *cdb, st->delta.p, s);
                smb::launch_mark_dead_n(st->q.p, st->nq, st->alive.p, st->isect.p, st->d_n.p, s);
            } else {                                           // huge rows: synchronous path
                uint32_t n = 0;
                st->d_n.download(&n, 1);
                sync(s);
                st->delta.zero();
                if (n) one_vs_many_dev(st->isect.p, n, *cdb, st->delta.p, s);
                smb::launch_mark_dead(st->q.p, st->nq, st->alive.p, st->isect.p, n, s);
            }
            have_delta = true;
            CK(cudaGetLastError());
        }
        if (rounds && st->remaining) {                          // size of the last intersection
            uint32_t last_n = 0;
            CK(cudaMemcpyAsync(&last_n, st->d_n.p, 4, cudaMemcpyDeviceToHost, s));
            sync(s);
            if (isect_sizes[rounds - 1] != last_n) isect_sizes[rounds - 1] = last_n;
        }
        sync(s);
        return rounds;
    });
}

// ---- multigather: the gather rounds of many queries against one resident database (multigather_kernels.cuh)
struct SmbMultiGather {
    std::vector<uint64_t> pick_off;          // [Q+1] into rows / sizes
    std::vector<uint32_t> rows, sizes;       // the picks of every query, query after query
    std::vector<uint32_t> overlaps;          // |picked row ∩ query| (its first counter)
    std::vector<uint32_t> consumed;          // [total query hashes]: round that took the hash, UINT32_MAX if none
    uint64_t round_launches = 0;             // kernel launches of the batched rounds
};

}  // extern "C"
namespace {

// a call through the C ABI (which records its own error) whose error is raised again inside the caller's guard
template <typename F>
auto abi_call(F&& f) -> decltype(f()) {
    t_has_error = false;
    auto r = f();
    if (t_has_error) { t_has_error = false; throw SmbError(t_error); }
    return r;
}

// device bytes one group of queries may take (SMB_MULTIGATHER_GROUP_BYTES overrides; the results do not depend on the
// grouping): the queries' hashes and consumed rounds, and the candidates, picks and intersections of the batched rounds
size_t multigather_group_bytes() {
    const char* e = getenv("SMB_MULTIGATHER_GROUP_BYTES");
    const long long v = e ? atoll(e) : 0;
    return v > 0 ? (size_t)v : ((size_t)1 << 30);
}

// the checks of a query CSR (smb_multigather, smb_many_vs_many): hashes on the host, or null (checked on the device)
void check_query_csr(const uint64_t* h, const uint64_t* off, size_t Q) {
    if (Q && off[0] != 0) fail(SOURMASH_ERROR_CODE_MSG, "query offsets must start at 0");
    for (size_t i = 0; i < Q; ++i) {
        if (off[i + 1] < off[i]) fail(SOURMASH_ERROR_CODE_MSG, "query offsets must not decrease");
        if (h)
            for (uint64_t k = off[i] + 1; k < off[i + 1]; ++k)
                if (h[k] <= h[k - 1]) fail(SOURMASH_ERROR_CODE_MSG, "every query must be sorted and unique");
    }
}

// device bytes one group of many_vs_many may take: its G x n counters and 12 bytes per query hash (the merged key
// stream and its query ids).  SMB_MANY_VS_MANY_GROUP_BYTES overrides; the counts do not depend on the grouping
size_t many_vs_many_group_bytes() {
    const char* e = getenv("SMB_MANY_VS_MANY_GROUP_BYTES");
    const long long v = e ? atoll(e) : 0;
    return v > 0 ? (size_t)v : ((size_t)1 << 30);
}

// How the counts of many queries against one set are made, chosen from the input alone: groups of two or more
// consecutive queries share one range-major pass (the copy built on first use, as one_vs_many_dev builds it); a group
// of one query, an indexed set, SMB_SEARCH_LAYOUT=global and a set the copy declines take one_vs_many_dev per query.
struct MvmPlan {
    const smb::RangeMajor* rm = nullptr;     // null: query by query
    std::vector<size_t> cuts;                // group g = queries [cuts[g], cuts[g + 1])
};

// off: the Q + 1 offsets of the queries' CSR.  A group's counters and key stream stay within the byte budget, and its
// keys within range_major_group_keys (sparse per-range bitmaps)
MvmPlan many_vs_many_plan(const uint64_t* off, size_t Q, const SmbSketchSet& db, cudaStream_t s) {
    MvmPlan p;
    const size_t nB = db.n_rows;
    if (Q >= 2 && nB && !db.index && smb::range_search_enabled()) {
        if (!db.range_major && !db.range_major_tried) {
            db.range_major_tried = true;
            CK(smb::range_major_build(db.d_hashes, db.d_off, (int)nB, db.total(), set_max_key(db, s), &db.range_major, s));
        }
        p.rm = db.range_major;
    }
    const size_t budget = many_vs_many_group_bytes();
    const uint64_t key_cap = p.rm ? smb::range_major_group_keys(p.rm) : UINT64_MAX;
    p.cuts.push_back(0);
    for (size_t i = 0, j; i < Q; i = j) {
        uint64_t keys = off[i + 1] - off[i];
        for (j = i + 1; j < Q; ++j) {
            const uint64_t nk = off[j + 1] - off[j];
            if ((j + 1 - i) * nB * 4 + (keys + nk) * 12 > budget || keys + nk > key_cap) break;
            keys += nk;
        }
        p.cuts.push_back(j);
    }
    return p;
}

// counters of the plan's queries [a, b) into d_counts ((b - a) x n, query-major, zeroed by the caller); off: the CSR
// offsets, the hashes of query a at d_q[0]
void many_vs_many_group(const MvmPlan& p, const uint64_t* d_q, const uint64_t* off, size_t a, size_t b,
                        const SmbSketchSet& db, uint32_t* d_counts, cudaStream_t s) {
    const size_t nB = db.n_rows;
    if (p.rm && b - a >= 2) {
        std::vector<uint64_t> rel(b - a + 1);
        for (size_t k = a; k <= b; ++k) rel[k - a] = off[k] - off[a];
        DevBuf<uint64_t> d_off(rel.size(), s);
        d_off.upload(rel.data(), rel.size());
        bool unsorted = false;
        CK(smb::many_vs_many_range_major(p.rm, d_q, d_off.p, (int)(b - a), rel.back(), d_counts, &unsorted, s));
        sync(s);      // rel is a host temporary
        if (unsorted) fail(SOURMASH_ERROR_CODE_MSG, "every query must be sorted and unique");
        return;
    }
    for (size_t k = a; k < b; ++k)
        one_vs_many_dev(d_q + (off[k] - off[a]), off[k + 1] - off[k], db, d_counts + (k - a) * nB, s);
}

struct MgQuery {
    const uint64_t* q = nullptr;
    size_t nq = 0;
    uint64_t q_begin = 0;                    // offset of the query in the caller's CSR
    uint32_t threshold = 1, min_count = 1;
    std::vector<uint32_t> cand, cand_counts; // candidate rows (ascending) and their first counters
    uint64_t isect_cap = 0, pick_cap = 0;
    std::vector<uint32_t> rows, sizes;
};

// one query through the session loop: an indexed set, or candidate rows too large for the shared-memory table
void multigather_session(MgQuery& g, const SmbSketchSet* db, uint32_t* consumed) {
    if (g.cand.empty() || g.pick_cap == 0) return;
    std::unique_ptr<SmbSketchSet> sub;
    const SmbSketchSet* gdb = db;
    // rows below min_count must not enter the counters; below the threshold they can never be picked anyway
    if (g.min_count > g.threshold && g.cand.size() < db->n_rows) {
        sub.reset(abi_call([&] { return smb_sketchset_take_rows(db, g.cand.data(), g.cand.size()); }));
        gdb = sub.get();
    }
    std::unique_ptr<SmbGatherState> st(abi_call([&] { return smb_gather_begin_min(g.q, g.nq, gdb, g.threshold); }));
    std::vector<uint64_t> buf(std::max<uint64_t>(gdb->max_len, 1));
    size_t remaining = g.nq;
    for (uint32_t r = 0; r < g.pick_cap && remaining > 0; ++r) {
        uint32_t best = 0, row = 0;
        abi_call([&] { smb_gather_peek(st.get(), &best, &row); return 0; });
        if (best == 0 || best < g.threshold) break;
        const size_t k = abi_call([&] { return smb_gather_intersect(st.get(), row, buf.data()); });
        for (size_t i = 0; i < k; ++i) consumed[std::lower_bound(g.q, g.q + g.nq, buf[i]) - g.q] = r;
        g.rows.push_back(sub ? g.cand[row] : row);
        g.sizes.push_back((uint32_t)k);
        remaining = abi_call([&] { return smb_gather_apply(st.get(), buf.data(), k); });
    }
}

// the batched rounds of queries whose candidate rows fit the shared-memory table; their hashes and consumed rounds
// already sit on the device at (q_begin - base) of d_q / d_consumed
uint64_t multigather_batched(std::vector<MgQuery*>& grp, const SmbSketchSet* db, const uint64_t* d_q, uint32_t* d_consumed,
                             uint64_t base, cudaStream_t s) {
    const size_t K = grp.size();
    std::vector<uint64_t> q_begin(K), q_end(K), cand_off(K + 1, 0), pick_off(K + 1, 0), isect_off(K + 1, 0);
    std::vector<uint32_t> thr(K), cta_start(K + 1, 0);
    constexpr int COLS = 16;                                  // candidate rows per decrement CTA (one per warp)
    uint64_t max_cap = 0, max_isect = 0, max_key = set_max_key(*db, s);
    for (size_t k = 0; k < K; ++k) {
        const MgQuery& g = *grp[k];
        q_begin[k] = g.q_begin - base;
        q_end[k] = q_begin[k] + g.nq;
        cand_off[k + 1] = cand_off[k] + g.cand.size();
        pick_off[k + 1] = pick_off[k] + g.pick_cap;
        isect_off[k + 1] = isect_off[k] + g.isect_cap;
        cta_start[k + 1] = cta_start[k] + (uint32_t)((g.cand.size() + COLS - 1) / COLS);
        thr[k] = g.threshold;
        max_cap = std::max(max_cap, g.pick_cap);
        max_isect = std::max(max_isect, g.isect_cap);
        max_key = std::max(max_key, g.q[g.nq - 1]);
    }
    std::vector<uint32_t> cand(cand_off[K]), counts(cand_off[K]);
    for (size_t k = 0; k < K; ++k) {
        std::copy(grp[k]->cand.begin(), grp[k]->cand.end(), cand.begin() + cand_off[k]);
        std::copy(grp[k]->cand_counts.begin(), grp[k]->cand_counts.end(), counts.begin() + cand_off[k]);
    }
    // one split table per decrement CTA: the longest intersection, a directory of about four buckets per key
    smb::PairwisePlan one = smb::plan_pairwise(max_isect, max_key, 1);
    const size_t key_bytes = (size_t)(one.cap + 2) * 8;
    const uint64_t max_entries = std::min<uint64_t>((227 * 1024 - key_bytes) / 2 - 2, 60000);
    const uint64_t want_entries = std::min<uint64_t>(max_entries, std::max<uint64_t>(4096, 4 * max_isect));
    int sh = 0;
    while (sh < 63 && (max_key >> sh) >= want_entries) ++sh;
    const int nb = (int)((max_key >> sh) + 1);
    const size_t smem = key_bytes + ((size_t)nb + 2) * 2;

    DevBuf<uint64_t> d_qb(K, s), d_qe(K, s), d_cand_off(K + 1, s), d_pick_off(K + 1, s),
        d_isect(std::max<uint64_t>(isect_off[K], 1), s), d_isect_off(K + 1, s);
    DevBuf<uint32_t> d_cand(cand.size(), s), d_counts(counts.size(), s), d_delta(counts.size(), s),
        d_pick_rows(std::max<uint64_t>(pick_off[K], 1), s), d_pick_sizes(std::max<uint64_t>(pick_off[K], 1), s),
        d_state(2 * K, s), d_live(1, s), d_thr(K, s), d_isect_n(K, s), d_cta(K + 1, s);
    d_qb.upload(q_begin.data(), K); d_qe.upload(q_end.data(), K);
    d_cand.upload(cand.data(), cand.size()); d_cand_off.upload(cand_off.data(), K + 1);
    d_counts.upload(counts.data(), counts.size()); d_delta.zero();
    d_pick_off.upload(pick_off.data(), K + 1); d_isect_off.upload(isect_off.data(), K + 1);
    d_state.zero(); d_thr.upload(thr.data(), K); d_cta.upload(cta_start.data(), K + 1);
    uint32_t live = (uint32_t)K;
    d_live.upload(&live, 1);
    smb::MultiGatherArgs a{d_q, d_qb.p, d_qe.p, d_cand.p, d_cand_off.p, d_counts.p, d_delta.p, d_pick_off.p, d_pick_rows.p,
                           d_pick_sizes.p, d_state.p, d_live.p, d_thr.p, d_consumed, d_isect.p, d_isect_off.p, d_isect_n.p,
                           db->d_hashes, db->d_off, d_cta.p, (int)K, COLS, sh, nb, one.cap + 2};
    // rounds enqueued in batches, the live counter read once per batch; a query stops by itself at its cap
    const uint64_t launches0 = smb::g_launches.load();
    const uint32_t batch = 16;
    for (uint64_t issued = 0; live && issued < max_cap + 1; issued += batch) {
        for (uint32_t k = 0; k < batch; ++k) smb::launch_multi_gather_round(a, cta_start[K], smem, s);
        CK(cudaGetLastError());
        d_live.download(&live, 1);
        sync(s);
    }
    const uint64_t launches = smb::g_launches.load() - launches0;
    std::vector<uint32_t> state(2 * K), prow(pick_off[K]), psize(pick_off[K]);
    d_state.download(state.data(), 2 * K);
    d_pick_rows.download(prow.data(), pick_off[K]);
    d_pick_sizes.download(psize.data(), pick_off[K]);
    sync(s);
    for (size_t k = 0; k < K; ++k) {
        MgQuery& g = *grp[k];
        const uint32_t n = state[2 * k];
        g.rows.assign(prow.begin() + pick_off[k], prow.begin() + pick_off[k] + n);
        g.sizes.assign(psize.begin() + pick_off[k], psize.begin() + pick_off[k] + n);
    }
    return launches;
}

// queries [i, j): hashes uploaded once, first counters (the many-query pass of many_vs_many_group; one readback per
// group of its plan), then the batched rounds, the consumed rounds read back once, and the queries that need the
// session loop
void multigather_group(std::vector<MgQuery>& qs, size_t i, size_t j, const SmbSketchSet* db, uint64_t max_rounds,
                       SmbMultiGather* m, cudaStream_t s) {
    const uint64_t base = qs[i].q_begin, n = qs[j - 1].q_begin + qs[j - 1].nq - base;
    const size_t nB = db->n_rows;
    DevBuf<uint64_t> d_q(std::max<uint64_t>(n, 1), s);
    DevBuf<uint32_t> d_consumed(std::max<uint64_t>(n, 1), s);
    d_q.upload(qs[i].q, n);
    CK(cudaMemsetAsync(d_consumed.p, 0xff, std::max<uint64_t>(n, 1) * 4, s));
    std::vector<uint64_t> off(j - i + 1);
    for (size_t k = i; k < j; ++k) off[k - i] = qs[k].q_begin - base;
    off[j - i] = n;
    const MvmPlan plan = many_vs_many_plan(off.data(), j - i, *db, s);
    std::vector<uint32_t> cnt;
    for (size_t c = 0; c + 1 < plan.cuts.size(); ++c) {
        const size_t a = plan.cuts[c], b = plan.cuts[c + 1];
        DevBuf<uint32_t> d_cnt((b - a) * nB, s);
        d_cnt.zero();
        many_vs_many_group(plan, d_q.p + off[a], off.data(), a, b, *db, d_cnt.p, s);
        cnt.resize((b - a) * nB);
        d_cnt.download(cnt.data(), cnt.size());
        sync(s);
        for (size_t k = a; k < b; ++k) {
            MgQuery& g = qs[i + k];
            if (g.nq == 0) continue;
            const uint32_t* row_cnt = cnt.data() + (k - a) * nB;
            uint64_t longest = 0;
            for (size_t r = 0; r < nB; ++r)
                if (row_cnt[r] >= g.min_count) {
                    g.cand.push_back((uint32_t)r);
                    g.cand_counts.push_back(row_cnt[r]);
                    longest = std::max<uint64_t>(longest, db->h_off[r + 1] - db->h_off[r]);
                }
            g.isect_cap = std::min<uint64_t>(g.nq, longest);
            g.pick_cap = std::min<uint64_t>(max_rounds, g.cand.size());
        }
    }
    const uint64_t mk = set_max_key(*db, s);
    std::vector<MgQuery*> batched, session;
    for (size_t k = i; k < j; ++k) {
        MgQuery& g = qs[k];
        if (g.cand.empty() || g.pick_cap == 0) continue;
        const smb::PairwisePlan p = smb::plan_pairwise(g.isect_cap, std::max(mk, g.q[g.nq - 1]), 1);
        (db->index || p.tables_per_cta == 0 || p.cap >= 32760 ? session : batched).push_back(&g);
    }
    // the candidates, picks and intersections of one launch of the rounds stay within the budget
    const size_t budget = multigather_group_bytes();
    std::vector<MgQuery*> part;
    size_t part_bytes = 0;
    auto flush = [&] {
        if (!part.empty()) m->round_launches += multigather_batched(part, db, d_q.p, d_consumed.p, base, s);
        part.clear();
        part_bytes = 0;
    };
    for (MgQuery* g : batched) {
        const size_t bytes = g->isect_cap * 8 + g->cand.size() * 16 + g->pick_cap * 8 + 64;
        if (!part.empty() && part_bytes + bytes > budget) flush();
        part.push_back(g);
        part_bytes += bytes;
    }
    flush();
    d_consumed.download(m->consumed.data() + base, n);
    sync(s);
    for (MgQuery* g : session) multigather_session(*g, db, m->consumed.data() + g->q_begin);
}

}  // namespace
extern "C" {

SmbMultiGather* smb_multigather(const uint64_t* q_hashes, const uint64_t* q_offsets, uintptr_t n_queries,
                                const SmbSketchSet* db, const uint32_t* thresholds, const uint32_t* min_counts,
                                uintptr_t max_rounds) {
    return guarded<SmbMultiGather*>([&]() -> SmbMultiGather* {
        cudaStream_t s = need_gpu();
        const size_t Q = n_queries;
        check_query_csr(q_hashes, q_offsets, Q);
        std::vector<MgQuery> qs(Q);
        for (size_t i = 0; i < Q; ++i) {
            MgQuery& g = qs[i];
            g.q_begin = q_offsets[i];
            g.q = q_hashes + g.q_begin;
            g.nq = q_offsets[i + 1] - g.q_begin;
            g.threshold = std::max<uint32_t>(thresholds ? thresholds[i] : 1, 1);
            g.min_count = std::max<uint32_t>(min_counts ? min_counts[i] : 1, 1);
        }
        auto m = std::make_unique<SmbMultiGather>();
        m->consumed.assign(Q ? q_offsets[Q] : 0, UINT32_MAX);
        if (db->n_rows && max_rounds) {
            // groups of consecutive queries: 12 bytes per query hash on the device, the rest of the budget for the rounds
            const size_t budget = multigather_group_bytes();
            for (size_t i = 0, j; i < Q; i = j) {
                size_t bytes = qs[i].nq * 12;
                for (j = i + 1; j < Q && bytes + qs[j].nq * 12 <= budget / 2; ++j) bytes += qs[j].nq * 12;
                multigather_group(qs, i, j, db, max_rounds, m.get(), s);
            }
        }
        m->pick_off.assign(Q + 1, 0);
        for (size_t i = 0; i < Q; ++i) {
            m->pick_off[i + 1] = m->pick_off[i] + qs[i].rows.size();
            m->rows.insert(m->rows.end(), qs[i].rows.begin(), qs[i].rows.end());
            m->sizes.insert(m->sizes.end(), qs[i].sizes.begin(), qs[i].sizes.end());
            for (uint32_t r : qs[i].rows)
                m->overlaps.push_back(qs[i].cand_counts[std::lower_bound(qs[i].cand.begin(), qs[i].cand.end(), r) - qs[i].cand.begin()]);
        }
        return m.release();
    });
}

// many_vs_many: the one-vs-many counts of many queries, groups of them sharing one pass over the database
void smb_many_vs_many(const uint64_t* q_hashes, const uint64_t* q_offsets, uintptr_t n_queries, const SmbSketchSet* db,
                      uint32_t* counts_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t Q = n_queries, nB = db->n_rows;
        check_query_csr(q_hashes, q_offsets, Q);
        if (Q == 0 || nB == 0) return;
        const MvmPlan plan = many_vs_many_plan(q_offsets, Q, *db, s);
        for (size_t c = 0; c + 1 < plan.cuts.size(); ++c) {
            const size_t a = plan.cuts[c], b = plan.cuts[c + 1];
            const uint64_t nk = q_offsets[b] - q_offsets[a];
            DevBuf<uint64_t> d_q(nk, s);
            d_q.upload(q_hashes + q_offsets[a], nk);
            DevBuf<uint32_t> d_cnt((b - a) * nB, s);
            d_cnt.zero();
            many_vs_many_group(plan, d_q.p, q_offsets, a, b, *db, d_cnt.p, s);
            d_cnt.download(counts_out + a * nB, (b - a) * nB);
            sync(s);
        }
    });
}

void smb_many_vs_many_dev(const uint64_t* d_q_hashes, const uint64_t* q_offsets, uintptr_t n_queries,
                          const SmbSketchSet* db, uint32_t* d_counts_out) {
    guarded_void([&] {
        cudaStream_t s = need_gpu();
        const size_t Q = n_queries, nB = db->n_rows;
        check_query_csr(nullptr, q_offsets, Q);
        if (Q == 0 || q_offsets[Q] == 0) {
            if (Q && nB) CK(cudaMemsetAsync(d_counts_out, 0, Q * nB * sizeof(uint32_t), s));
            return;
        }
        {   // every query sorted and unique: one pass over the keys on the device
            DevBuf<uint64_t> d_off(Q + 1, s);
            DevBuf<unsigned long long> d_stat(2, s);
            d_off.upload(q_offsets, Q + 1);
            d_stat.zero();
            smb::launch_query_stats(d_q_hashes, d_off.p, (int)Q, nullptr, d_stat.p, s);
            CK(cudaGetLastError());
            unsigned long long stat[2] = {0, 0};
            d_stat.download(stat, 2);
            sync(s);
            if (stat[1]) fail(SOURMASH_ERROR_CODE_MSG, "every query must be sorted and unique");
        }
        if (nB == 0) return;
        CK(cudaMemsetAsync(d_counts_out, 0, Q * nB * sizeof(uint32_t), s));
        const MvmPlan plan = many_vs_many_plan(q_offsets, Q, *db, s);
        for (size_t c = 0; c + 1 < plan.cuts.size(); ++c) {
            const size_t a = plan.cuts[c], b = plan.cuts[c + 1];
            many_vs_many_group(plan, d_q_hashes + q_offsets[a], q_offsets, a, b, *db, d_counts_out + a * nB, s);
        }
    });
}

uintptr_t smb_multigather_rounds(const SmbMultiGather* m, uintptr_t query) {
    return guarded<uintptr_t>([&]() -> uintptr_t {
        if (query + 1 >= m->pick_off.size()) fail(SOURMASH_ERROR_CODE_MSG, "query index out of range");
        return m->pick_off[query + 1] - m->pick_off[query];
    });
}

void smb_multigather_picks(const SmbMultiGather* m, uintptr_t query, uint32_t* rows, uint32_t* sizes, uint32_t* overlaps) {
    guarded_void([&] {
        if (query + 1 >= m->pick_off.size()) fail(SOURMASH_ERROR_CODE_MSG, "query index out of range");
        const uint64_t b = m->pick_off[query], e = m->pick_off[query + 1];
        if (rows) std::copy(m->rows.begin() + b, m->rows.begin() + e, rows);
        if (sizes) std::copy(m->sizes.begin() + b, m->sizes.begin() + e, sizes);
        if (overlaps) std::copy(m->overlaps.begin() + b, m->overlaps.begin() + e, overlaps);
    });
}

void smb_multigather_consumed(const SmbMultiGather* m, uint32_t* consumed_round) {
    std::copy(m->consumed.begin(), m->consumed.end(), consumed_round);
}

uint64_t smb_multigather_round_launches(const SmbMultiGather* m) { return m->round_launches; }

void smb_multigather_free(SmbMultiGather* m) { delete m; }

// ==========================================================================================
// Part 3: native ingest (csrc/ingest.cu) -- sequence files and .sig JSON without per-record Python
// ==========================================================================================
SmbRecords* smb_records_read(const char* const* paths, uintptr_t n_paths, int32_t n_threads) {
    return guarded<SmbRecords*>([&]() -> SmbRecords* {
        auto r = std::make_unique<SmbRecords>();
        probe_devices();
        std::string err = smb::read_sequence_files(paths, n_paths, n_threads > 0 ? n_threads : default_threads(),
                                                   g_device_count > 0, r->b);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_IO, err);
        return r.release();
    });
}
void smb_records_free(SmbRecords* r) { delete r; }
uintptr_t smb_records_len(const SmbRecords* r) { return r->b.file.size(); }
uint64_t smb_records_total_bytes(const SmbRecords* r) { return r->b.total; }
const uint8_t* smb_records_data(const SmbRecords* r) { return r->b.seqs; }
const uint64_t* smb_records_starts(const SmbRecords* r) { return r->b.start.data(); }
const uint64_t* smb_records_lengths(const SmbRecords* r) { return r->b.len.data(); }
const uint32_t* smb_records_files(const SmbRecords* r) { return r->b.file.data(); }
const char* smb_records_names(const SmbRecords* r, const uint64_t** name_offsets) {
    *name_offsets = r->b.name_off.data();
    return r->b.names.data();
}
SmbSketchSet* smb_sketch_records(const SmbRecords* r, const uint32_t* rec_to_sketch, uintptr_t n_sketches,
                                 const uint32_t* ksizes, uintptr_t n_ksizes, HashFunctions hash_function,
                                 bool input_is_protein, uint64_t scaled, uint32_t num, uint64_t seed,
                                 bool track_abundance, uint64_t* n_kmers_out) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        const smb::RecordBatch& b = r->b;
        const size_t n = b.file.size();
        cudaStream_t s = need_gpu();
        DevBuf<uint8_t> d_bases(b.extent + 32, s);
        StreamList in;
        in.d_bases = d_bases.p;
        in.h_bases = b.seqs;                             // uploaded in groups, overlapped with hashing
        in.total_bytes = b.extent;
        in.off = b.start;
        in.len = b.len;
        if (rec_to_sketch) in.row.assign(rec_to_sketch, rec_to_sketch + n);
        in.n_sketches = rec_to_sketch ? n_sketches : n;
        SketchParams P = make_params(ksizes, n_ksizes, scaled, num, seed, track_abundance);
        P.hash_function = hash_function;
        P.input_is_protein = hash_function != HASH_FUNCTIONS_MURMUR64_DNA && input_is_protein;
        return sketch_streams(in, P, s, n_kmers_out).release();
    });
}

// `sig kmers` over a batch of records (sig/__main__.py:1206-1256): every window of every record hashed and probed against
// the merged query on the device (kmer_match_kernels.cuh), the matches sorted into file order, the per-record flags and
// the found hashes of the query.  query: sorted-unique hashes of the merged sketch (for num sketches its bottom num).
struct SmbKmerMatches {
    std::vector<uint64_t> keys, hashes, found;
    std::vector<uint8_t> matched, has_invalid;
};

SmbKmerMatches* smb_kmer_match_records(const SmbRecords* r, const uint64_t* query, uintptr_t n_query, uint32_t ksize,
                                       HashFunctions hash_function, uint64_t seed, uint64_t max_hash, uint32_t num,
                                       bool input_is_protein, bool skip_invalid) {
    return guarded<SmbKmerMatches*>([&]() -> SmbKmerMatches* {
        const smb::RecordBatch& b = r->b;
        const size_t n = b.file.size();
        cudaStream_t s = need_gpu();
        for (uintptr_t i = 1; i < n_query; ++i)
            if (query[i] <= query[i - 1]) fail(SOURMASH_ERROR_CODE_MSG, "query hashes must be sorted and unique");
        if (n >= (1ull << 32)) fail(SOURMASH_ERROR_CODE_MSG, "more than 2^32 - 1 records in one batch");
        const bool dna = hash_function == HASH_FUNCTIONS_MURMUR64_DNA;
        if (dna && input_is_protein)
            fail(SOURMASH_ERROR_CODE_INVALID_HASH_FUNCTION, "Invalid hash function: \"DNA\"");   // signature.rs:376-380
        const uint32_t kaa = ksize / 3;
        const bool translate = !dna && !input_is_protein;
        if (!dna && kaa > smb::aa_max_k(translate))
            fail(SOURMASH_ERROR_CODE_INTERNAL, "protein-family ksize too large for the shared-memory tile");
        auto res = std::make_unique<SmbKmerMatches>();
        res->matched.assign(n, 0);
        res->has_invalid.assign(n, 0);
        const bool stores = num > 0 || max_hash > 0;                 // minhash.rs:324-327
        if (n == 0 || n_query == 0 || !stores) return res.release();

        // chunks of W windows (window starts) per record; the ordinal of a window must fit 32 bits
        smb::KmerMatchArgs a{};
        a.mode = dna ? (smb::k_has_rolled_kernel(ksize) ? 0 : 1) : (translate ? 3 : 2);
        a.K = dna ? ksize : kaa;
        a.W = a.mode == 0 ? 32 : 8;
        std::vector<uint64_t> chunk(n + 1, 0);
        uint64_t n_windows = 0;
        for (size_t i = 0; i < n; ++i) {
            const uint64_t L = b.len[i];
            uint64_t starts = 0, wins = 0, span_bytes = 0;
            if (dna) { starts = ksize && L >= ksize ? L - ksize + 1 : 0; wins = starts; }
            else { const uint64_t span = translate ? 3ull * kaa : kaa; starts = kaa && L >= span ? L - span + 1 : 0;
                   wins = translate ? 2 * starts : starts; }
            if (wins >= (1ull << 32)) fail(SOURMASH_ERROR_CODE_MSG, "record " + std::to_string(i) + " has 2^32 or more k-mers");
            // rolled kernel: chunks tile the record's aligned coordinates (hash_thread_windows)
            span_bytes = a.mode == 0 ? (starts ? (b.start[i] & 15) + L : 0) : starts;
            chunk[i + 1] = chunk[i] + (span_bytes + a.W - 1) / a.W;
            n_windows += wins;
        }
        DevBuf<uint8_t> d_bases(b.extent + 32, s);
        d_bases.upload(b.seqs, b.extent);
        DevBuf<uint64_t> d_off(n, s), d_len(n, s), d_chunk(n + 1, s), d_q(n_query, s);
        d_off.upload(b.start.data(), n);
        d_len.upload(b.len.data(), n);
        d_chunk.upload(chunk.data(), n + 1);
        d_q.upload(query, n_query);
        DevBuf<uint8_t> d_hit(n, s), d_invalid(n, s), d_tabs;
        d_hit.zero(); d_invalid.zero();
        if (!dna) {
            const smb::AaTables T = smb::build_aa_tables((int)hash_function);
            d_tabs.alloc(sizeof T, s);
            d_tabs.upload((const uint8_t*)&T, sizeof T);
            sync(s);                                                 // T is a stack temporary
        }
        a.bases = d_bases.p; a.rec_off = d_off.p; a.rec_len = d_len.p; a.chunk_start = d_chunk.p;
        a.n_chunks = chunk[n]; a.n_rec = (int)n;
        a.seed = seed; a.max_hash = num > 0 ? UINT64_MAX : max_hash;
        a.tabs = (const smb::AaTables*)d_tabs.p;
        a.rec_hit = d_hit.p; a.rec_invalid = dna ? d_invalid.p : nullptr;
        // Q: UINT64_MAX answered by a flag, the rest by the split table (small Q) or the global directory
        a.q_has_max = query[n_query - 1] == UINT64_MAX;
        a.q = d_q.p; a.nq = n_query - (a.q_has_max ? 1 : 0);
        a.q_top = a.nq ? query[a.nq - 1] : 0;
        DevBuf<uint32_t> d_dir, d_bm;
        a.split = smb::kmer_match_split_fits(a.nq);
        if (a.split) {
            const uint64_t entries = std::max<uint64_t>(a.nq, 256);          // about one key per bucket
            uint32_t sh = 0;
            while (sh < 63 && (a.q_top >> sh) >= entries) ++sh;
            a.shift = sh; a.nb = (a.q_top >> sh) + 1;
        } else {
            int nb_log2 = 12;                                              // as one_vs_many_dev
            while (nb_log2 < 26 && (1ull << nb_log2) < 2 * a.nq) ++nb_log2;
            uint32_t sh = 0;
            while (sh < 63 && (a.q_top >> sh) >= (1ull << nb_log2)) ++sh;
            a.shift = sh; a.nb = (a.q_top >> sh) + 1;
            d_dir.alloc(a.nb + 2, s);
            smb::launch_build_global_dir(d_q.p, a.nq, (int)sh, a.nb, d_dir.p, s);
            a.fine_log2 = 3;
            d_bm.alloc(((size_t)a.nb << a.fine_log2) / 32 + 2, s);
            d_bm.zero();
            smb::launch_build_query_bitmap(d_q.p, a.nq, (int)sh, a.fine_log2, d_bm.p, s);
            a.gdir = d_dir.p; a.bitmap = d_bm.p;
        }
        // match buffer: room for about four times the expected probes' worth of hits; an overflow reruns at the exact size
        const long double probes = num > 0 ? (long double)n_windows
                                           : (long double)n_windows * (((long double)max_hash + 1.0L) / 18446744073709551616.0L);
        uint64_t cap = (uint64_t)std::min<long double>((long double)n_windows, probes + 4.0L * n_query + 4096.0L);
        DevBuf<unsigned long long> d_count(1, s);
        DevBuf<uint64_t> d_keys, d_hashes;
        unsigned long long count = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            d_keys.alloc(cap, s); d_hashes.alloc(cap, s);
            d_count.zero();
            a.keys = d_keys.p; a.hashes = d_hashes.p; a.cap = cap; a.count = d_count.p;
            if (t_profiling) t_timer_hash.begin(s);
            smb::launch_kmer_match(a, s);
            if (t_profiling) t_timer_hash.end(s);
            CK(cudaGetLastError());
            d_count.download(&count, 1);
            sync(s);
            if (count <= cap) break;
            cap = count;                                              // rerun with the exact count
        }
        if (count > cap) fail(SOURMASH_ERROR_CODE_INTERNAL, "k-mer match buffer overflowed twice");
        // file order: one radix sort of (record << 32 | ordinal, hash)
        const uint64_t m = count;
        DevBuf<uint64_t> d_keys2(m, s), d_hashes2(m, s);
        if (m) {
            int end_bit = 33;
            while (end_bit < 64 && (n >> (end_bit - 32)) != 0) ++end_bit;
            CK(smb::sort_kmer_matches(d_keys.p, d_hashes.p, d_keys2.p, d_hashes2.p, m, end_bit, s));
        }
        // found hashes: for a scaled query every match; for a num query the common hashes of the passing records.
        // skip_invalid: records with an invalid DNA window add nothing (`sig kmers --check-sequence --force` skips them)
        const uint8_t* skip = skip_invalid && dna ? d_invalid.p : nullptr;
        DevBuf<uint8_t> d_flag(n_query, s);
        d_flag.zero();
        if (num == 0) {
            smb::launch_match_mark_found(d_keys2.p, d_hashes2.p, m, skip, d_q.p, n_query, d_flag.p, s);
        } else {
            d_hit.download(res->matched.data(), n);
            sync(s);
            std::vector<uint32_t> recs;
            for (size_t i = 0; i < n; ++i) if (res->matched[i]) recs.push_back((uint32_t)i);
            if (!recs.empty()) {
                StreamList in;
                in.d_bases = d_bases.p;
                in.n_sketches = recs.size();
                for (uint32_t i : recs) { in.off.push_back(b.start[i]); in.len.push_back(b.len[i]); }
                SketchParams P;
                P.ksizes = {ksize}; P.num = num; P.seed = seed;
                P.hash_function = hash_function; P.input_is_protein = input_is_protein;
                const bool prof = t_profiling;
                t_profiling = false;                                 // the timer keeps the match pass
                auto bottom = sketch_streams(in, P, s, nullptr);
                t_profiling = prof;
                DevBuf<uint32_t> d_recs(recs.size(), s);
                d_recs.upload(recs.data(), recs.size());
                smb::launch_match_num_common(bottom->d_hashes, bottom->d_off, d_recs.p, (int)recs.size(), d_q.p, n_query,
                                             num, skip, d_hit.p, d_flag.p, s);
                CK(cudaGetLastError());
                sync(s);                                             // recs is a host temporary
            }
        }
        CK(cudaGetLastError());
        res->keys.resize(m); res->hashes.resize(m);
        std::vector<uint8_t> flag(n_query);
        d_keys2.download(res->keys.data(), m);
        d_hashes2.download(res->hashes.data(), m);
        d_hit.download(res->matched.data(), n);
        if (dna) d_invalid.download(res->has_invalid.data(), n);
        d_flag.download(flag.data(), n_query);
        sync(s);
        for (uintptr_t i = 0; i < n_query; ++i) if (flag[i]) res->found.push_back(query[i]);
        return res.release();
    });
}
uintptr_t smb_kmer_matches_len(const SmbKmerMatches* m) { return m->keys.size(); }
const uint64_t* smb_kmer_matches_keys(const SmbKmerMatches* m) { return m->keys.data(); }
const uint64_t* smb_kmer_matches_hashes(const SmbKmerMatches* m) { return m->hashes.data(); }
const uint8_t* smb_kmer_matches_matched(const SmbKmerMatches* m) { return m->matched.data(); }
const uint8_t* smb_kmer_matches_has_invalid(const SmbKmerMatches* m) { return m->has_invalid.data(); }
uintptr_t smb_kmer_matches_n_found(const SmbKmerMatches* m) { return m->found.size(); }
const uint64_t* smb_kmer_matches_found(const SmbKmerMatches* m) { return m->found.data(); }
void smb_kmer_matches_free(SmbKmerMatches* m) { delete m; }

// `sig merge` / `sig intersect` / `sig subtract` over a resident set (sig/__main__.py:459-712): one device sort of the
// whole set and one pass over its runs (sketch_combine.cuh); the only readback before the copy-out is the length
struct SmbCombined {
    std::vector<uint64_t> hashes, abunds;
    bool has_abunds = false;
};

SmbCombined* smb_sketchset_combine(const SmbSketchSet* set, uint32_t op, uint32_t num) {
    return guarded<SmbCombined*>([&]() -> SmbCombined* {
        cudaStream_t s = need_gpu();
        if (op > SMB_COMBINE_FIRST_ONLY) fail(SOURMASH_ERROR_CODE_MSG, "unknown combine op " + std::to_string(op));
        auto res = std::make_unique<SmbCombined>();
        res->has_abunds = op == SMB_COMBINE_UNION && set->d_abunds != nullptr;
        const uint64_t T = set->total();
        if (T > 0x7fffffffull)
            fail(SOURMASH_ERROR_CODE_MSG, "set too large to combine (more than 2^31 - 1 hashes)");
        if (set->n_rows == 0 || T == 0) return res.release();
        uint64_t *d_h = nullptr, *d_v = nullptr, n = 0;
        const uint64_t max_key = set_max_key(*set, s);
        if (t_profiling) t_timer_hash.begin(s);                      // the sort, the run pass, the scan, the scatter
        CK(smb::sketchset_combine(set->d_hashes, set->d_abunds, set->n_rows, T, set->h_off[1], max_key, op, &d_h, &d_v,
                                  &n, s));
        if (t_profiling) t_timer_hash.end(s);
        DevBuf<uint64_t> out_h, out_v;                                // owned from here on, freed on every path
        out_h.p = d_h; out_h.n = T; out_h.s = s;
        out_v.p = d_v; out_v.n = d_v ? T : 0; out_v.s = s;
        if (op == SMB_COMBINE_UNION && num > 0 && n > num) n = num;   // the bottom num of the union
        res->hashes.resize(n);
        out_h.download(res->hashes.data(), n);
        if (res->has_abunds) { res->abunds.resize(n); out_v.download(res->abunds.data(), n); }
        sync(s);
        return res.release();
    });
}
uintptr_t smb_combined_len(const SmbCombined* c) { return c->hashes.size(); }
const uint64_t* smb_combined_hashes(const SmbCombined* c) { return c->hashes.data(); }
const uint64_t* smb_combined_abunds(const SmbCombined* c) { return c->has_abunds ? c->abunds.data() : nullptr; }
void smb_combined_free(SmbCombined* c) { delete c; }

// `lca classify` / `lca summarize` (lca/lca_utils.py:186-225): the LCA node of every database hash, found once per
// command (lca_table_build), then per batch of queries the distinct (query, node) of their hashes with summed weights
// and first positions (lca_counts).  Only those rows come back to the host.
struct SmbLcaHashvals {
    std::vector<uint64_t> hashes;
    std::vector<uint32_t> idx;
    int64_t begin = -1, end = -1;
};

SmbLcaHashvals* smb_lca_parse_hashvals(const char* text, uintptr_t len) {
    return guarded<SmbLcaHashvals*>([&]() -> SmbLcaHashvals* {
        auto r = std::make_unique<SmbLcaHashvals>();
        std::string err = smb::parse_lca_hashvals(text, len, r->hashes, r->idx, &r->begin, &r->end);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return r.release();
    });
}
uintptr_t smb_lca_hashvals_len(const SmbLcaHashvals* h) { return h->hashes.size(); }
const uint64_t* smb_lca_hashvals_hashes(const SmbLcaHashvals* h) { return h->hashes.data(); }
const uint32_t* smb_lca_hashvals_idx(const SmbLcaHashvals* h) { return h->idx.data(); }
void smb_lca_hashvals_span(const SmbLcaHashvals* h, int64_t* begin, int64_t* end) { *begin = h->begin; *end = h->end; }
void smb_lca_hashvals_free(SmbLcaHashvals* h) { delete h; }

struct SmbLcaTable {
    DevBuf<uint64_t> hashes;
    DevBuf<uint32_t> lca, parent;
    DevBuf<uint8_t> depth;
    uint64_t n = 0;
    uint32_t n_nodes = 0;
};

SmbLcaTable* smb_lca_table_build(const uint64_t* hashes, const uint32_t* nodes, uintptr_t n, const uint32_t* parent,
                                 const uint8_t* depth, uint32_t n_nodes, uint64_t max_hash) {
    return guarded<SmbLcaTable*>([&]() -> SmbLcaTable* {
        if (n_nodes == 0) fail(SOURMASH_ERROR_CODE_MSG, "the taxonomy trie has no nodes (node 0 is the root)");
        if (n_nodes == smb::LCA_NO_NODE) fail(SOURMASH_ERROR_CODE_MSG, "the taxonomy trie has too many nodes");
        if (depth[0] != 0) fail(SOURMASH_ERROR_CODE_MSG, "node 0 must be the root, at depth 0");
        for (uint32_t i = 1; i < n_nodes; ++i)
            if (parent[i] >= i || depth[i] != depth[parent[i]] + 1)
                fail(SOURMASH_ERROR_CODE_MSG, "trie node " + std::to_string(i) + " needs a parent below it, one rank up");
        for (uintptr_t i = 0; i < n; ++i)
            if (nodes[i] >= n_nodes && nodes[i] != smb::LCA_NO_NODE)
                fail(SOURMASH_ERROR_CODE_MSG, "node " + std::to_string(nodes[i]) + " out of range for a trie of " +
                                                  std::to_string(n_nodes) + " nodes");
        if (n > 0x7fffffffull) fail(SOURMASH_ERROR_CODE_MSG, "LCA table too large (more than 2^31 - 1 pairs)");
        auto t = std::make_unique<SmbLcaTable>();
        t->n_nodes = n_nodes;
        if (n == 0) return t.release();
        cudaStream_t s = need_gpu();
        uint64_t max_key = 0;
        for (uintptr_t i = 0; i < n; ++i) max_key = std::max(max_key, hashes[i]);
        t->parent.alloc(n_nodes, s); t->parent.upload(parent, n_nodes);
        t->depth.alloc(n_nodes, s); t->depth.upload(depth, n_nodes);
        DevBuf<uint64_t> d_h(n, s);
        DevBuf<uint32_t> d_nodes(n, s);
        d_h.upload(hashes, n);
        d_nodes.upload(nodes, n);
        uint64_t* out_h = nullptr;
        uint32_t* out_lca = nullptr;
        if (t_profiling) t_timer_hash.begin(s);
        CK(smb::lca_table_build(d_h.p, d_nodes.p, n, max_hash, max_key, t->parent.p, t->depth.p, &out_h, &out_lca,
                                &t->n, s));
        if (t_profiling) t_timer_hash.end(s);
        t->hashes.p = out_h; t->hashes.n = n; t->hashes.s = s;
        t->lca.p = out_lca; t->lca.n = n; t->lca.s = s;
        return t.release();
    });
}
uintptr_t smb_lca_table_len(const SmbLcaTable* t) { return t->n; }
void smb_lca_table_copy(const SmbLcaTable* t, uint64_t* hashes, uint32_t* lca) {
    guarded_void([&] {
        if (t->n == 0) return;
        t->hashes.download(hashes, t->n);
        t->lca.download(lca, t->n);
        sync(t->hashes.s);
    });
}
void smb_lca_table_free(SmbLcaTable* t) { delete t; }

struct SmbLcaCounts {
    std::vector<uint32_t> query, node;
    std::vector<uint64_t> count, first;
};

SmbLcaCounts* smb_lca_counts(const SmbLcaTable* t, const SmbSketchSet* queries, bool use_abunds) {
    return guarded<SmbLcaCounts*>([&]() -> SmbLcaCounts* {
        const std::vector<uint64_t>& off = queries->h_off;
        if (queries->n_rows >= smb::LCA_NO_NODE) fail(SOURMASH_ERROR_CODE_MSG, "too many queries in one batch");
        if (!off.empty() && off[0] != 0) fail(SOURMASH_ERROR_CODE_MSG, "query offsets must start at 0");
        for (size_t i = 1; i < off.size(); ++i)
            if (off[i] < off[i - 1]) fail(SOURMASH_ERROR_CODE_MSG, "query offsets decrease at " + std::to_string(i));
        if (use_abunds && !queries->d_abunds) fail(SOURMASH_ERROR_CODE_MSG, "the queries carry no abundances");
        const uint64_t Tq = queries->total();
        if (Tq > 0x7fffffffull) fail(SOURMASH_ERROR_CODE_MSG, "query batch too large (more than 2^31 - 1 hashes)");
        auto r = std::make_unique<SmbLcaCounts>();
        if (Tq == 0 || t->n == 0) return r.release();
        cudaStream_t s = need_gpu();
        uint32_t *d_q = nullptr, *d_node = nullptr;
        uint64_t *d_w = nullptr, *d_first = nullptr, n = 0;
        if (t_profiling) t_timer_hash.begin(s);
        CK(smb::lca_counts(t->hashes.p, t->lca.p, t->n, queries->d_hashes, queries->d_off, (uint32_t)queries->n_rows,
                           Tq, use_abunds ? queries->d_abunds : nullptr, &d_q, &d_node, &d_w, &d_first, &n, s));
        if (t_profiling) t_timer_hash.end(s);
        DevBuf<uint32_t> b_q, b_node;                                  // owned from here on, freed on every path
        DevBuf<uint64_t> b_w, b_first;
        b_q.p = d_q; b_q.n = Tq; b_q.s = s;
        b_node.p = d_node; b_node.n = Tq; b_node.s = s;
        b_w.p = d_w; b_w.n = Tq; b_w.s = s;
        b_first.p = d_first; b_first.n = Tq; b_first.s = s;
        r->query.resize(n); r->node.resize(n); r->count.resize(n); r->first.resize(n);
        b_q.download(r->query.data(), n);
        b_node.download(r->node.data(), n);
        b_w.download(r->count.data(), n);
        b_first.download(r->first.data(), n);
        sync(s);
        return r.release();
    });
}
uintptr_t smb_lca_counts_len(const SmbLcaCounts* c) { return c->query.size(); }
const uint32_t* smb_lca_counts_query(const SmbLcaCounts* c) { return c->query.data(); }
const uint32_t* smb_lca_counts_node(const SmbLcaCounts* c) { return c->node.data(); }
const uint64_t* smb_lca_counts_count(const SmbLcaCounts* c) { return c->count.data(); }
const uint64_t* smb_lca_counts_first(const SmbLcaCounts* c) { return c->first.data(); }
void smb_lca_counts_free(SmbLcaCounts* c) { delete c; }

// `lca index` (lca/lca_db.py:145-205, 420-465): every hash's idx grouped on the device, and the JSON text of
// "hashval_to_idx" written there in key ranges, each copied back once
struct SmbLcaIndex {
    smb::LcaIndexDev d;
    cudaStream_t s = 0;
    ~SmbLcaIndex() {
        void* p[5] = {d.hash, d.koff, d.idx, d.key_of, d.at};
        for (void* q : p) if (q) cudaFreeAsync(q, s);
    }
};

SmbLcaIndex* smb_lca_index_build(const SmbSketchSet* sigs) {
    return guarded<SmbLcaIndex*>([&]() -> SmbLcaIndex* {
        const std::vector<uint64_t>& off = sigs->h_off;
        if (sigs->n_rows > 0xffffffffull) fail(SOURMASH_ERROR_CODE_MSG, "too many signatures (idx is 32-bit)");
        if (!off.empty() && off[0] != 0) fail(SOURMASH_ERROR_CODE_MSG, "row offsets must start at 0");
        for (size_t i = 1; i < off.size(); ++i)
            if (off[i] < off[i - 1]) fail(SOURMASH_ERROR_CODE_MSG, "row offsets decrease at " + std::to_string(i));
        const uint64_t T = sigs->total();
        if (T > 0x7ffffffeull) fail(SOURMASH_ERROR_CODE_MSG, "LCA index too large (more than 2^31 - 2 pairs)");
        auto x = std::make_unique<SmbLcaIndex>();
        if (T == 0) return x.release();
        cudaStream_t s = need_gpu();
        x->s = s;
        const uint64_t max_key = set_max_key(*sigs, s);
        if (t_profiling) t_timer_hash.begin(s);
        CK(smb::lca_index_build(sigs->d_hashes, sigs->d_off, (uint32_t)sigs->n_rows, T, max_key, &x->d, s));
        if (t_profiling) t_timer_hash.end(s);
        return x.release();
    });
}
uintptr_t smb_lca_index_len(const SmbLcaIndex* x) { return x->d.K; }
uintptr_t smb_lca_index_pairs(const SmbLcaIndex* x) { return x->d.T; }
void smb_lca_index_copy(const SmbLcaIndex* x, uint64_t* hashes, uint64_t* offsets, uint32_t* idx) {
    guarded_void([&] {
        const uint64_t K = x->d.K, T = x->d.T;
        offsets[0] = 0;
        if (K == 0) return;
        std::vector<uint32_t> koff(K + 1);
        CK(cudaMemcpyAsync(hashes, x->d.hash, K * sizeof(uint64_t), cudaMemcpyDeviceToHost, x->s));
        CK(cudaMemcpyAsync(koff.data(), x->d.koff, (K + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, x->s));
        CK(cudaMemcpyAsync(idx, x->d.idx, T * sizeof(uint32_t), cudaMemcpyDeviceToHost, x->s));
        sync(x->s);
        for (uint64_t k = 0; k <= K; ++k) offsets[k] = koff[k];
    });
}
uintptr_t smb_lca_index_text(const SmbLcaIndex* x, uintptr_t first_key, uintptr_t max_bytes, char* out,
                             uintptr_t* n_bytes) {
    return guarded<uintptr_t>([&]() -> uintptr_t {
        const uint64_t K = x->d.K;
        if (K == 0) {
            if (first_key != 0) fail(SOURMASH_ERROR_CODE_MSG, "first key out of range (the index has no keys)");
            if (out && *n_bytes >= 2) { out[0] = '{'; out[1] = '}'; }
            *n_bytes = 2;
            return 0;
        }
        if (first_key >= K) fail(SOURMASH_ERROR_CODE_MSG, "first key " + std::to_string(first_key) + " out of range");
        uint64_t plan[4];
        CK(smb::lca_index_plan(x->d, first_key, max_bytes, plan, x->s));
        const uint64_t next = plan[0], lead = first_key == 0, trail = next == K;
        const uint64_t size = plan[1] + lead + trail;
        if (out && *n_bytes >= size) {                                 // the range fits the caller's buffer
            DevBuf<char> d_out(plan[1], x->s);
            if (t_profiling) t_timer_hash.begin(x->s);
            CK(smb::lca_index_text(x->d, plan[2], plan[3], d_out.p, x->s));
            if (t_profiling) t_timer_hash.end(x->s);
            d_out.download(out + lead, plan[1]);
            sync(x->s);
            if (lead) out[0] = '{';
            if (trail) out[size - 1] = '}';
        }
        *n_bytes = size;
        return next;
    });
}
void smb_lca_index_free(SmbLcaIndex* x) { delete x; }

// signatures straight from a sketch set (the tail of _compute_individual, command_sketch.py:770-789):
// signature s gets rows [s * n_ksizes, (s + 1) * n_ksizes) of `set` as its sketches
SourmashSignature** smb_signatures_from_sketchset(const SmbSketchSet* set, const uint32_t* ksizes,
                                                  uintptr_t n_ksizes, HashFunctions hash_function,
                                                  uint64_t scaled, uint32_t num, uint64_t seed,
                                                  uintptr_t* size) {
    return guarded<SourmashSignature**>([&]() -> SourmashSignature** {
        cudaStream_t s = need_gpu();
        const size_t n_rows = set->n_rows, nk = n_ksizes;
        if (nk == 0 || n_rows % nk != 0) fail(SOURMASH_ERROR_CODE_INTERNAL, "sketch set does not hold n_ksizes rows per signature");
        const size_t tot = set->total();
        std::vector<uint64_t> h(tot), ab(set->d_abunds ? tot : 0);
        if (tot) {
            CK(cudaMemcpyAsync(h.data(), set->d_hashes, tot * 8, cudaMemcpyDeviceToHost, s));
            if (set->d_abunds) CK(cudaMemcpyAsync(ab.data(), set->d_abunds, tot * 8, cudaMemcpyDeviceToHost, s));
            sync(s);
        }
        const size_t n_sig = n_rows / nk;
        auto** arr = (SourmashSignature**)malloc(std::max<size_t>(n_sig, 1) * sizeof(void*));
        for (size_t g = 0; g < n_sig; ++g) {
            auto* sig = new SourmashSignature();
            for (size_t j = 0; j < nk; ++j) {
                const size_t r0 = set->h_off[g * nk + j], r1 = set->h_off[g * nk + j + 1];
                MH m;
                m.num = num; m.ksize = ksizes[j]; m.seed = seed; m.hash_function = hash_function;
                m.max_hash = max_hash_for_scaled(scaled); m.track = set->d_abunds != nullptr;
                m.mins.assign(h.begin() + r0, h.begin() + r1);
                if (m.track) m.abunds.assign(ab.begin() + r0, ab.begin() + r1);
                sig->sketches.push_back(std::move(m));
            }
            arr[g] = sig;
        }
        *size = n_sig;
        return arr;
    });
}

SmbSigs* smb_sigs_read_opts(const char* const* paths, uintptr_t n_paths, int32_t n_threads, uint32_t flags) {
    return guarded<SmbSigs*>([&]() -> SmbSigs* {
        auto r = std::make_unique<SmbSigs>();
        std::string err = smb::read_signature_files(paths, n_paths, n_threads > 0 ? n_threads : default_threads(),
                                                    flags, r->b);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return r.release();
    });
}
SmbSigs* smb_sigs_read_loose(const char* const* paths, uintptr_t n_paths, int32_t n_threads, uint32_t flags,
                             const uint8_t* loose) {
    return guarded<SmbSigs*>([&]() -> SmbSigs* {
        auto r = std::make_unique<SmbSigs>();
        std::string err = smb::read_signature_files(paths, n_paths, n_threads > 0 ? n_threads : default_threads(),
                                                    flags, r->b, loose);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return r.release();
    });
}
SmbSigs* smb_sigs_read(const char* const* paths, uintptr_t n_paths, int32_t n_threads) {
    return smb_sigs_read_opts(paths, n_paths, n_threads, 0);
}
SmbSigs* smb_sigs_parse(const char* data, uintptr_t len) {
    return guarded<SmbSigs*>([&]() -> SmbSigs* {
        auto r = std::make_unique<SmbSigs>();
        std::string text;
        if (len >= 2 && (uint8_t)data[0] == 0x1f && (uint8_t)data[1] == 0x8b) {
            text = gunzip_bytes((const uint8_t*)data, len);
            data = text.data(); len = text.size();
        }
        std::string err = smb::parse_signature_json(data, len, 0, r->b);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return r.release();
    });
}
// in-memory objects -> the same CSR batch as the file parser (first sketch of every signature, like
// SourmashSignature.minhash): lets compare / search pull N sketches out of N objects in one call
static void batch_push(smb::SigBatch& B, const MH& m, const std::string& name, const std::string& filename) {
    if (B.off.empty()) B.off.push_back(0);
    smb::SigRecord rec;
    rec.name = name; rec.filename = filename; rec.license = "CC0"; rec.klass = "sourmash_signature";
    rec.has_name = !name.empty(); rec.has_filename = !filename.empty();
    smb::SigSketch sk;
    sk.sig_index = (uint32_t)B.sigs.size(); sk.file = 0;
    sk.ksize = m.ksize; sk.num = m.num; sk.max_hash = m.max_hash; sk.seed = m.seed;
    sk.hash_function = (uint32_t)m.hash_function; sk.has_abund = m.track;
    B.sigs.push_back(std::move(rec));
    B.sketches.push_back(std::move(sk));
    B.mins.insert(B.mins.end(), m.mins.begin(), m.mins.end());
    if (m.track) B.abunds.insert(B.abunds.end(), m.abunds.begin(), m.abunds.end());
    else B.abunds.insert(B.abunds.end(), m.mins.size(), 1);
    B.any_abund = B.any_abund || m.track;
    B.off.push_back(B.mins.size());
}
SmbSigs* smb_sigs_from_signatures(const SourmashSignature* const* sigs, uintptr_t n) {
    return guarded<SmbSigs*>([&]() -> SmbSigs* {
        auto r = std::make_unique<SmbSigs>();
        r->b.off.push_back(0);
        for (uintptr_t i = 0; i < n; ++i) {
            if (sigs[i]->sketches.empty())
                fail(SOURMASH_ERROR_CODE_INTERNAL, "internal error: \"found unsupported sketch type\"");
            batch_push(r->b, sigs[i]->sketches[0], sigs[i]->name, sigs[i]->filename);
        }
        return r.release();
    });
}
SmbSigs* smb_sigs_from_minhashes(const SourmashKmerMinHash* const* mhs, uintptr_t n) {
    return guarded<SmbSigs*>([&]() -> SmbSigs* {
        auto r = std::make_unique<SmbSigs>();
        r->b.off.push_back(0);
        for (uintptr_t i = 0; i < n; ++i) batch_push(r->b, *mhs[i], "", "");
        return r.release();
    });
}
void smb_sigs_free(SmbSigs* s) { delete s; }
uintptr_t smb_sigs_n_signatures(const SmbSigs* s) { return s->b.sigs.size(); }
uintptr_t smb_sigs_n_sketches(const SmbSigs* s) { return s->b.sketches.size(); }
bool smb_sigs_any_abund(const SmbSigs* s) { return s->b.any_abund; }
void smb_sigs_sketch_info(const SmbSigs* s, uintptr_t i, SmbSketchInfo* out) {
    const smb::SigSketch& k = s->b.sketches[i];
    out->sig_index = k.sig_index; out->file = k.file; out->ksize = k.ksize; out->num = k.num;
    out->max_hash = k.max_hash; out->seed = k.seed; out->hash_function = k.hash_function;
    out->has_abund = k.has_abund; out->n_mins = s->b.off[i + 1] - s->b.off[i];
}
void smb_sigs_sketch_info_all(const SmbSigs* s, SmbSketchInfo* out) {
    for (uintptr_t i = 0; i < s->b.sketches.size(); ++i) smb_sigs_sketch_info(s, i, out + i);
}
SourmashStr smb_sigs_sketch_md5(const SmbSigs* s, uintptr_t i) { return make_str(s->b.sketches[i].md5sum); }
void smb_sigs_md5_all(const SmbSigs* s, char* out) {
    // identities computed from the hashes (what ss.md5sum() returns), not the md5sum field of the file
    guarded_void([&] {
        const smb::SigBatch& B = s->b;
        const size_t n = B.sketches.size();
        std::atomic<size_t> next{0};
        auto worker = [&] {
            for (;;) {
                const size_t i = next.fetch_add(1);
                if (i >= n) return;
                const std::string d = smb::sketch_md5(B.sketches[i].ksize, B.mins.data() + B.off[i], (size_t)(B.off[i + 1] - B.off[i]));
                memcpy(out + 32 * i, d.data(), 32);
            }
        };
        const size_t nt = std::min<size_t>((size_t)default_threads(), std::max<size_t>(n / 64, 1));
        std::vector<std::thread> pool;
        for (size_t t = 1; t < nt; ++t) pool.emplace_back(worker);
        worker();
        for (auto& t : pool) t.join();
    });
}
SourmashStr smb_sigs_sig_name(const SmbSigs* s, uintptr_t j) { return make_str(s->b.sigs[j].name); }
SourmashStr smb_sigs_sig_filename(const SmbSigs* s, uintptr_t j) { return make_str(s->b.sigs[j].filename); }
SourmashStr smb_sigs_sig_license(const SmbSigs* s, uintptr_t j) { return make_str(s->b.sigs[j].license); }
SourmashStr smb_sigs_sig_location(const SmbSigs* s, uintptr_t j) { return make_str(s->b.sigs[j].location); }
const uint64_t* smb_sigs_offsets(const SmbSigs* s) { return s->b.off.data(); }
const uint64_t* smb_sigs_mins(const SmbSigs* s) { return s->b.mins.data(); }
const uint64_t* smb_sigs_abunds(const SmbSigs* s) { return s->b.abunds.data(); }
SourmashKmerMinHash* smb_sigs_minhash(const SmbSigs* s, uintptr_t i) {
    return guarded<SourmashKmerMinHash*>([&] { return new MH(mh_from_batch(s->b, i)); });
}
// rows (NULL: all) of the parsed sketches -> device CSR, optionally cut at max_hash (0: as stored)
SourmashSignature** smb_sigs_signatures(const SmbSigs* s, const uint32_t* rows, uintptr_t n_rows, uintptr_t* size) {
    return guarded<SourmashSignature**>([&]() -> SourmashSignature** {
        const size_t n = rows ? n_rows : s->b.sketches.size();
        auto** arr = (SourmashSignature**)malloc(std::max<size_t>(n, 1) * sizeof(void*));
        for (size_t r = 0; r < n; ++r) {
            const size_t i = rows ? rows[r] : r;
            if (i >= s->b.sketches.size()) {
                for (size_t q = 0; q < r; ++q) delete arr[q];
                free(arr);
                fail(SOURMASH_ERROR_CODE_INTERNAL, "sketch row out of range");
            }
            arr[r] = sig_from_batch(s->b, i);
        }
        *size = n;
        return arr;
    });
}
// Copies row r of n (src_h[r], src_a[r], off[r + 1] - off[r] elements) into the CSR h / a, rows spread over the host
// threads: gathering the rows of a large index is a few GB of memcpy
static void pack_rows(size_t n, const std::vector<uint64_t>& off, const std::vector<const uint64_t*>& src_h,
                      const std::vector<const uint64_t*>& src_a, uint64_t* h, uint64_t* a) {
    std::atomic<size_t> next{0};
    auto worker = [&] {
        for (;;) {
            const size_t r0 = next.fetch_add(256);
            if (r0 >= n) return;
            for (size_t r = r0; r < std::min(n, r0 + 256); ++r) {
                const size_t len = off[r + 1] - off[r];
                if (!len) continue;
                memcpy(h + off[r], src_h[r], len * 8);
                if (a) memcpy(a + off[r], src_a[r], len * 8);
            }
        }
    };
    const size_t nt = std::min<size_t>((size_t)default_threads(), std::max<size_t>(off[n] / (1u << 20), 1));
    std::vector<std::thread> pool;
    for (size_t t = 1; t < nt; ++t) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
}

SmbSketchSet* smb_sigs_to_sketchset(const SmbSigs* s, const uint32_t* rows, uintptr_t n_rows, uint64_t max_hash,
                                    bool with_abunds) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        const smb::SigBatch& B = s->b;
        const size_t n = rows ? n_rows : B.sketches.size();
        std::vector<uint64_t> off(n + 1, 0);
        std::vector<const uint64_t*> src_h(n), src_a(n);
        for (size_t r = 0; r < n; ++r) {
            const size_t i = rows ? rows[r] : r;
            if (i >= B.sketches.size()) fail(SOURMASH_ERROR_CODE_INTERNAL, "sketch row out of range");
            const uint64_t* b = B.mins.data() + B.off[i];
            const uint64_t* e = B.mins.data() + B.off[i + 1];
            if (max_hash) e = std::upper_bound(b, e, max_hash);        // downsample_scaled == prefix
            src_h[r] = b; src_a[r] = B.abunds.data() + B.off[i];
            off[r + 1] = off[r] + (uint64_t)(e - b);
        }
        std::unique_ptr<uint64_t[]> h(new uint64_t[std::max<uint64_t>(off[n], 1)]);
        std::unique_ptr<uint64_t[]> ab(with_abunds ? new uint64_t[std::max<uint64_t>(off[n], 1)] : nullptr);
        pack_rows(n, off, src_h, src_a, h.get(), ab.get());
        return smb_sketchset_from_host(h.get(), off.data(), n, ab.get());
    });
}

// The first sketch of subject i of a search: the signature sigs[i] when it is not null, else the sketch mhs[i]
static const MH& subject_sketch(const SourmashSignature* const* sigs, const SourmashKmerMinHash* const* mhs, size_t i) {
    if (sigs && sigs[i]) {
        if (sigs[i]->sketches.empty()) fail(SOURMASH_ERROR_CODE_INTERNAL, "internal error: \"found unsupported sketch type\"");
        return sigs[i]->sketches[0];
    }
    if (!mhs || !mhs[i]) fail(SOURMASH_ERROR_CODE_INTERNAL, "subject " + std::to_string(i) + " has no sketch");
    return *mhs[i];
}
void smb_subjects_sketch_info(const SourmashSignature* const* sigs, const SourmashKmerMinHash* const* mhs, uintptr_t n,
                              SmbSketchInfo* out) {
    guarded_void([&] {
        for (uintptr_t i = 0; i < n; ++i) {
            const MH& m = subject_sketch(sigs, mhs, i);
            out[i] = SmbSketchInfo{};
            out[i].ksize = m.ksize; out[i].num = m.num; out[i].max_hash = m.max_hash; out[i].seed = m.seed;
            out[i].hash_function = (uint32_t)m.hash_function; out[i].has_abund = m.track; out[i].n_mins = m.mins.size();
        }
    });
}
SmbSketchSet* smb_sketchset_from_subjects(const SourmashSignature* const* sigs, const SourmashKmerMinHash* const* mhs,
                                          uintptr_t n, bool with_abunds) {
    return guarded<SmbSketchSet*>([&]() -> SmbSketchSet* {
        std::vector<uint64_t> off(n + 1, 0);
        std::vector<const uint64_t*> src_h(n), src_a(n);
        for (uintptr_t i = 0; i < n; ++i) {
            const MH& m = subject_sketch(sigs, mhs, i);
            if (with_abunds && !m.track)
                fail(SOURMASH_ERROR_CODE_NEEDS_ABUNDANCE_TRACKING, "sketch needs abundance for this operation");
            src_h[i] = m.mins.data(); src_a[i] = m.abunds.data();
            off[i + 1] = off[i] + m.mins.size();
        }
        std::unique_ptr<uint64_t[]> h(new uint64_t[std::max<uint64_t>(off[n], 1)]);
        std::unique_ptr<uint64_t[]> ab(with_abunds ? new uint64_t[std::max<uint64_t>(off[n], 1)] : nullptr);
        pack_rows(n, off, src_h, src_a, h.get(), ab.get());
        return smb_sketchset_from_host(h.get(), off.data(), n, ab.get());
    });
}

// reference ABI: ffi/signature.rs:219-343
SourmashSignature** signatures_load_path(const char* ptr, bool, uintptr_t ksize, const char* select_moltype,
                                         uintptr_t* size) {
    return guarded<SourmashSignature**>([&]() -> SourmashSignature** {
        smb::SigBatch B;
        const char* paths[1] = {ptr};
        // one JSON file, possibly compressed; a .zip collection is NOT accepted here (the reference's loaders rely on that:
        // save_load.py tries this before the zipfile loader, tests/test_index.py::test_zipfile_load_database_fail_if_not_zip)
        std::string err = smb::read_signature_files(paths, 1, 1, smb::SIGS_NO_ZIP, B);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return sigs_from_batch(B, ksize, select_moltype, size);
    });
}
SourmashSignature** signatures_load_buffer(const char* ptr, uintptr_t insize, bool, uintptr_t ksize,
                                           const char* select_moltype, uintptr_t* size) {
    return guarded<SourmashSignature**>([&]() -> SourmashSignature** {
        smb::SigBatch B;
        std::string text;
        if (insize >= 2 && (uint8_t)ptr[0] == 0x1f && (uint8_t)ptr[1] == 0x8b) {   // niffler sniffing
            text = gunzip_bytes((const uint8_t*)ptr, insize);
            ptr = text.data(); insize = text.size();
        }
        std::string err = smb::parse_signature_json(ptr, insize, 0, B);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_SERDE_ERROR, err);
        return sigs_from_batch(B, ksize, select_moltype, size);
    });
}
const uint8_t* signatures_save_buffer(const SourmashSignature* const* ptr, uintptr_t size, uint8_t compression,
                                      uintptr_t* osize) {
    return guarded<const uint8_t*>([&]() -> const uint8_t* {
        std::string text = json_signatures(ptr, size);
        if (compression > 0) text = gzip_bytes(text, compression > 9 ? 9 : compression);
        uint8_t* out = (uint8_t*)malloc(text.size() + 1);
        memcpy(out, text.data(), text.size());
        out[text.size()] = 0;
        *osize = text.size();
        return out;
    });
}
SourmashStr signature_save_json(const SourmashSignature* ptr) {
    std::string out;
    json_signature(out, *ptr);
    return make_str(out);
}
void nodegraph_buffer_free(uint8_t* ptr, uintptr_t) { free(ptr); }
void signatures_array_free(SourmashSignature** ptr, uintptr_t) { free(ptr); }

// ------------------------------------------------------------------------------------------
// ZipStorage: src/core/src/ffi/storage.rs:15-141 over storage/mod.rs:314-448 (read-only)
// ------------------------------------------------------------------------------------------
static std::string utf8_arg(const char* p, uintptr_t n) {
    if (!p) fail(SOURMASH_ERROR_CODE_INTERNAL, "null string argument");
    return std::string(p, n);
}
static SourmashStr** str_array(const std::vector<std::string>& v, uintptr_t* size) {
    // array of boxed strings like the reference's Box<[*mut SourmashStr]>; read with paths[i][0]
    SourmashStr** arr = (SourmashStr**)malloc(sizeof(SourmashStr*) * std::max<size_t>(v.size(), 1));
    for (size_t i = 0; i < v.size(); ++i) {
        arr[i] = (SourmashStr*)malloc(sizeof(SourmashStr));
        *arr[i] = make_str(v[i]);
    }
    *size = v.size();
    return arr;
}

SourmashZipStorage* zipstorage_new(const char* ptr, uintptr_t insize) {
    return guarded<SourmashZipStorage*>([&]() -> SourmashZipStorage* {
        auto z = std::make_unique<SourmashZipStorage>();
        z->path = utf8_arg(ptr, insize);
        std::string err = z->zip.open(z->path.c_str());
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_IO, err);
        // storage/mod.rs:324-335 find_subdirs: exactly one directory entry becomes the default subdir
        size_t n_dirs = 0;
        for (const auto& m : z->zip.members) if (m.is_dir()) { ++n_dirs; z->subdir = m.name; }
        z->has_subdir = n_dirs == 1;
        if (!z->has_subdir) z->subdir.clear();
        return z.release();
    });
}
void zipstorage_free(SourmashZipStorage* ptr) { delete ptr; }
const uint8_t* zipstorage_load(const SourmashZipStorage* ptr, const char* path_ptr, uintptr_t insize, uintptr_t* size) {
    return guarded<const uint8_t*>([&]() -> const uint8_t* {
        const std::string path = utf8_arg(path_ptr, insize);
        const smb::ZipMember* m = ptr->zip.find(path);                       // storage/mod.rs:342-352
        if (!m && ptr->has_subdir) m = ptr->zip.find(ptr->subdir + path);
        if (!m) fail(SOURMASH_ERROR_CODE_STORAGE, "Path can't be found: " + path);
        std::string data;
        std::string err = ptr->zip.read(*m, data);
        if (!err.empty()) fail(SOURMASH_ERROR_CODE_STORAGE, "Error reading data from " + path + " (" + err + ")");
        uint8_t* buf = (uint8_t*)malloc(std::max<size_t>(data.size(), 1));
        memcpy(buf, data.data(), data.size());
        *size = data.size();
        return buf;                                                          // freed with nodegraph_buffer_free
    });
}
SourmashStr** zipstorage_filenames(const SourmashZipStorage* ptr, uintptr_t* size) {
    return guarded<SourmashStr**>([&]() -> SourmashStr** {
        std::vector<std::string> v;
        for (const auto& m : ptr->zip.members) v.push_back(m.name);
        return str_array(v, size);
    });
}
SourmashStr** zipstorage_list_sbts(const SourmashZipStorage* ptr, uintptr_t* size) {
    return guarded<SourmashStr**>([&]() -> SourmashStr** {
        std::vector<std::string> v;
        for (const auto& m : ptr->zip.members) {
            const std::string& s = m.name;
            if (s.size() >= 9 && s.compare(s.size() - 9, 9, ".sbt.json") == 0) v.push_back(s);
        }
        return str_array(v, size);
    });
}
void zipstorage_set_subdir(SourmashZipStorage* ptr, const char* path_ptr, uintptr_t insize) {
    guarded_void([&] {
        ptr->subdir = utf8_arg(path_ptr, insize);
        ptr->has_subdir = true;
    });
}
SourmashStr zipstorage_path(const SourmashZipStorage* ptr) { return make_str(ptr->path); }
SourmashStr zipstorage_subdir(const SourmashZipStorage* ptr) { return make_str(ptr->has_subdir ? ptr->subdir : std::string()); }

}  // extern "C"
