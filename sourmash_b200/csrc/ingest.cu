// ingest.cu -- native host-side readers (see ingest.h).  Host code only (no kernels); compiled
// with the rest of the library so that the boundary stays one C-ABI shared object.
//
// FASTA/FASTQ parsing follows what the reference's CLI gets from screed
// (src/sourmash/command_sketch.py:697-766): record name = the whole header line after the
// marker, sequence = the record's lines joined, with line ends stripped.  The reference's Rust
// benches use needletail + niffler for the same job (src/core/benches/compute.rs:36-45).
#include "ingest.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_set>

#include "md5.h"
#include "zipread.h"

namespace smb {

namespace {

// Growable byte buffer without value-initialisation (std::vector would zero every growth).
struct Bytes {
    uint8_t* p = nullptr;
    size_t n = 0, cap = 0;
    Bytes() {}
    Bytes(const Bytes&) = delete;
    Bytes& operator=(const Bytes&) = delete;
    ~Bytes() { free(p); }
    bool reserve(size_t want) {
        if (want <= cap) return true;
        size_t c = std::max<size_t>(want, cap * 2);
        uint8_t* q = (uint8_t*)realloc(p, c);
        if (!q) return false;
        p = q; cap = c;
        return true;
    }
    const uint8_t* data() const { return p; }
    size_t size() const { return n; }
};

// bzip2 input (the reference reads .bz2 through screed / niffler): the image ships libbz2.so.1.0 without
// its header, so the three streaming entry points are bound at first use; the struct is bzlib.h's.
struct BzStream {
    char* next_in; unsigned avail_in, total_in_lo32, total_in_hi32;
    char* next_out; unsigned avail_out, total_out_lo32, total_out_hi32;
    void* state;
    void* (*bzalloc)(void*, int, int); void (*bzfree)(void*, void*); void* opaque;
};
struct BzApi {
    int (*init)(BzStream*, int, int) = nullptr;
    int (*run)(BzStream*) = nullptr;
    int (*end)(BzStream*) = nullptr;
    bool ok = false;
};
const BzApi& bz_api() {
    static const BzApi api = [] {
        BzApi a;
        void* h = dlopen("libbz2.so.1.0", RTLD_NOW | RTLD_LOCAL);
        if (!h) h = dlopen("libbz2.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!h) return a;
        a.init = (int (*)(BzStream*, int, int))dlsym(h, "BZ2_bzDecompressInit");
        a.run = (int (*)(BzStream*))dlsym(h, "BZ2_bzDecompress");
        a.end = (int (*)(BzStream*))dlsym(h, "BZ2_bzDecompressEnd");
        a.ok = a.init && a.run && a.end;
        return a;
    }();
    return api;
}
inline bool is_bz2(const unsigned char* m, size_t n) { return n >= 3 && m[0] == 'B' && m[1] == 'Z' && m[2] == 'h'; }

// concatenated streams (pbzip2 output) are one file
std::string bunzip(const uint8_t* src, size_t n, Bytes& data) {
    const BzApi& bz = bz_api();
    if (!bz.ok) return "bzip2 input needs libbz2.so.1.0, which could not be loaded";
    if (!data.reserve(n * 5 + (1 << 16))) return "out of host memory";
    size_t fed = 0;
    while (fed < n) {
        if (!is_bz2(src + fed, n - fed)) break;                 // trailing bytes after the last stream
        BzStream zs;
        memset(&zs, 0, sizeof zs);
        if (bz.init(&zs, 0, 0) != 0) return "BZ2_bzDecompressInit failed";
        const size_t start = fed;
        int r = 0;
        for (;;) {
            if (zs.avail_in == 0 && fed < n) {
                const size_t c = std::min<size_t>(n - fed, 1u << 30);
                zs.next_in = (char*)(src + fed); zs.avail_in = (unsigned)c; fed += c;
            }
            if (data.cap - data.n < (1u << 16) && !data.reserve(data.cap * 2)) { bz.end(&zs); return "out of host memory"; }
            const size_t room = std::min<size_t>(data.cap - data.n, 1u << 30);
            zs.next_out = (char*)data.p + data.n; zs.avail_out = (unsigned)room;
            const unsigned in_before = zs.avail_in;
            r = bz.run(&zs);
            data.n += room - zs.avail_out;
            if (r == 4) break;                                  // BZ_STREAM_END
            if (r != 0 || (fed >= n && zs.avail_in == 0 && in_before == 0 && zs.avail_out == room)) {
                bz.end(&zs);
                return "bzip2 stream is corrupt or truncated";
            }
        }
        fed -= zs.avail_in;                                      // unread input belongs to the next stream
        bz.end(&zs);
        if (fed == start) break;
    }
    return "";
}

// xz and zstd, the other two formats niffler sniffs: same arrangement, liblzma.so.5 / libzstd.so.1 bound at first use
struct LzmaStream {                       // lzma/base.h lzma_stream (136 bytes), tail padded
    const uint8_t* next_in; size_t avail_in; uint64_t total_in;
    uint8_t* next_out; size_t avail_out; uint64_t total_out;
    const void* allocator; void* internal;
    void* reserved_ptr[4]; uint64_t reserved_int[2]; size_t reserved_size[2]; int reserved_enum[2];
    uint64_t pad[8];
};
struct LzmaApi {
    int (*decoder)(LzmaStream*, uint64_t, uint32_t) = nullptr;
    int (*code)(LzmaStream*, int) = nullptr;
    void (*end)(LzmaStream*) = nullptr;
    bool ok = false;
};
const LzmaApi& lzma_api() {
    static const LzmaApi api = [] {
        LzmaApi a;
        void* h = dlopen("liblzma.so.5", RTLD_NOW | RTLD_LOCAL);
        if (!h) return a;
        a.decoder = (int (*)(LzmaStream*, uint64_t, uint32_t))dlsym(h, "lzma_stream_decoder");
        a.code = (int (*)(LzmaStream*, int))dlsym(h, "lzma_code");
        a.end = (void (*)(LzmaStream*))dlsym(h, "lzma_end");
        a.ok = a.decoder && a.code && a.end;
        return a;
    }();
    return api;
}
inline bool is_xz(const unsigned char* m, size_t n) { return n >= 6 && !memcmp(m, "\xfd" "7zXZ\0", 6); }

std::string unxz(const uint8_t* src, size_t n, Bytes& data) {
    const LzmaApi& lz = lzma_api();
    if (!lz.ok) return "xz input needs liblzma.so.5, which could not be loaded";
    if (!data.reserve(n * 5 + (1 << 16))) return "out of host memory";
    LzmaStream zs;
    memset(&zs, 0, sizeof zs);
    if (lz.decoder(&zs, UINT64_MAX, 0x08u /* LZMA_CONCATENATED */) != 0) return "lzma_stream_decoder failed";
    zs.next_in = src; zs.avail_in = n;
    for (;;) {
        if (data.cap - data.n < (1u << 16) && !data.reserve(data.cap * 2)) { lz.end(&zs); return "out of host memory"; }
        zs.next_out = data.p + data.n; zs.avail_out = data.cap - data.n;
        const int r = lz.code(&zs, zs.avail_in == 0 ? 3 /* LZMA_FINISH */ : 0 /* LZMA_RUN */);
        data.n = data.cap - zs.avail_out;
        if (r == 1) break;                                       // LZMA_STREAM_END
        if (r != 0) { lz.end(&zs); return "xz stream is corrupt or truncated"; }
    }
    lz.end(&zs);
    return "";
}

struct ZstdBuf { void* p; size_t size, pos; };
struct ZstdApi {
    void* (*create)() = nullptr;
    size_t (*free)(void*) = nullptr;
    size_t (*run)(void*, ZstdBuf*, ZstdBuf*) = nullptr;
    unsigned (*is_error)(size_t) = nullptr;
    bool ok = false;
};
const ZstdApi& zstd_api() {
    static const ZstdApi api = [] {
        ZstdApi a;
        void* h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!h) return a;
        a.create = (void* (*)())dlsym(h, "ZSTD_createDStream");
        a.free = (size_t (*)(void*))dlsym(h, "ZSTD_freeDStream");
        a.run = (size_t (*)(void*, ZstdBuf*, ZstdBuf*))dlsym(h, "ZSTD_decompressStream");
        a.is_error = (unsigned (*)(size_t))dlsym(h, "ZSTD_isError");
        a.ok = a.create && a.free && a.run && a.is_error;
        return a;
    }();
    return api;
}
inline bool is_zstd(const unsigned char* m, size_t n) { return n >= 4 && m[0] == 0x28 && m[1] == 0xb5 && m[2] == 0x2f && m[3] == 0xfd; }

std::string unzstd(const uint8_t* src, size_t n, Bytes& data) {
    const ZstdApi& z = zstd_api();
    if (!z.ok) return "zstd input needs libzstd.so.1, which could not be loaded";
    if (!data.reserve(n * 5 + (1 << 16))) return "out of host memory";
    void* ds = z.create();
    if (!ds) return "ZSTD_createDStream failed";
    ZstdBuf in{(void*)src, n, 0};
    size_t hint = 1;
    for (;;) {
        if (data.cap - data.n < (1u << 16) && !data.reserve(data.cap * 2)) { z.free(ds); return "out of host memory"; }
        ZstdBuf out{data.p + data.n, data.cap - data.n, 0};
        const size_t in_before = in.pos;
        hint = z.run(ds, &out, &in);
        data.n += out.pos;
        if (z.is_error(hint)) { z.free(ds); return "zstd stream is corrupt"; }
        if (in.pos >= in.size && out.pos < out.size) break;      // input eaten and the output flushed
        if (in.pos == in_before && out.pos == 0) { z.free(ds); return "zstd stream is corrupt or truncated"; }
    }
    z.free(ds);
    if (hint != 0) return "zstd stream is corrupt or truncated"; // a frame was left unfinished
    return "";
}

// whole file into memory; gzip (magic 1f 8b), bzip2 ("BZh"), xz and zstd files are decompressed, anything else is read as is
std::string slurp(const char* path, Bytes& data) {
    FILE* fh = fopen(path, "rb");
    if (!fh) return std::string("cannot open ") + path;
    unsigned char magic[6] = {0, 0, 0, 0, 0, 0};
    size_t got = fread(magic, 1, 6, fh);
    fseek(fh, 0, SEEK_END);
    const long fsize = ftell(fh);
    fseek(fh, 0, SEEK_SET);
    const bool gz = got >= 2 && magic[0] == 0x1f && magic[1] == 0x8b;
    if (is_bz2(magic, got) || is_xz(magic, got) || is_zstd(magic, got)) {
        Bytes raw;
        if (!raw.reserve((size_t)std::max<long>(fsize, 0) + 16)) { fclose(fh); return "out of host memory"; }
        raw.n = fread(raw.p, 1, (size_t)std::max<long>(fsize, 0), fh);
        fclose(fh);
        std::string e = is_bz2(magic, got) ? bunzip(raw.p, raw.n, data)
                        : is_xz(magic, got) ? unxz(raw.p, raw.n, data) : unzstd(raw.p, raw.n, data);
        return e.empty() ? e : std::string(path) + ": " + e;
    }
    if (!gz) {
        if (!data.reserve((size_t)std::max<long>(fsize, 0) + 16)) { fclose(fh); return "out of host memory"; }
        data.n = fread(data.p, 1, (size_t)std::max<long>(fsize, 0), fh);
        fclose(fh);
        return "";
    }
    fclose(fh);
    gzFile f = gzopen(path, "rb");
    if (!f) return std::string("cannot open ") + path;
    gzbuffer(f, 1 << 20);
    if (!data.reserve((size_t)std::max<long>(fsize, 1) * 4 + (1 << 16))) { gzclose(f); return "out of host memory"; }
    for (;;) {
        if (data.cap - data.n < (1u << 20) && !data.reserve(data.cap * 2)) { gzclose(f); return "out of host memory"; }
        size_t want = std::min<size_t>(data.cap - data.n, 1u << 30);
        int n = gzread(f, data.p + data.n, (unsigned)want);
        if (n < 0) { int e; std::string m = gzerror(f, &e); gzclose(f); return std::string(path) + ": " + m; }
        if (n == 0) break;
        data.n += (size_t)n;
    }
    gzclose(f);
    return "";
}

// One input file held in memory: plain files are mapped (no copy), gzip files inflated.
struct Loaded {
    const uint8_t* p = nullptr;
    size_t n = 0;
    void* map = nullptr;
    size_t map_len = 0;
    Bytes owned;
    std::string error;
    ~Loaded() { if (map) munmap(map, map_len); }
};

void load_file(const char* path, Loaded& L) {
    int fd = open(path, O_RDONLY);
    if (fd < 0) { L.error = std::string("cannot open ") + path; return; }
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); L.error = std::string("cannot stat ") + path; return; }
    unsigned char magic[6] = {0, 0, 0, 0, 0, 0};
    const ssize_t got = pread(fd, magic, 6, 0);
    const size_t gn = got > 0 ? (size_t)got : 0;
    const bool packed = (gn >= 2 && magic[0] == 0x1f && magic[1] == 0x8b) || is_bz2(magic, gn) || is_xz(magic, gn) ||
                        is_zstd(magic, gn);
    if (!packed && st.st_size > 0 && S_ISREG(st.st_mode)) {
        void* m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
        if (m != MAP_FAILED) {
            madvise(m, (size_t)st.st_size, MADV_SEQUENTIAL);
            L.map = m; L.map_len = (size_t)st.st_size;
            L.p = (const uint8_t*)m; L.n = (size_t)st.st_size;
            close(fd);
            return;
        }
    }
    close(fd);
    L.error = slurp(path, L.owned);
    L.p = L.owned.p; L.n = L.owned.n;
}

struct FileRecords {
    std::vector<uint64_t> start, len;     // per record, relative to the file's output region
    std::string names;
    std::vector<uint64_t> name_off{0};
    uint64_t used = 0;                     // bytes written to the region
    std::string error;
};

inline const uint8_t* line_end(const uint8_t* p, const uint8_t* end) {
    const void* q = memchr(p, '\n', (size_t)(end - p));
    return q ? (const uint8_t*)q : end;
}
// copy [p, e) without trailing '\r' / blanks to dst + w; returns the new write position
inline uint64_t put_trimmed(uint8_t* dst, uint64_t w, const uint8_t* p, const uint8_t* e) {
    while (e > p && (e[-1] == '\r' || e[-1] == ' ' || e[-1] == '\t')) --e;
    memcpy(dst + w, p, (size_t)(e - p));
    return w + (uint64_t)(e - p);
}

// Records of one file; sequence bytes go straight to `dst` (a region of at least data-size bytes:
// the sequence lines of a file never outgrow the file).
void parse_records(const uint8_t* data, size_t size, uint8_t* dst, FileRecords& R) {
    const uint8_t* p = data;
    const uint8_t* end = p + size;
    while (p < end && (*p == '\n' || *p == '\r' || *p == ' ')) ++p;
    if (p == end) return;
    if (*p != '>' && *p != '@') { R.error = "neither FASTA nor FASTQ (first byte is not '>' or '@')"; return; }
    const bool fastq = *p == '@';
    uint64_t w = 0;
    while (p < end) {
        const uint8_t* e = line_end(p, end);
        if (e == p || *p == '\r') { p = e + 1; continue; }          // blank line between records
        if (*p != (fastq ? '@' : '>')) { R.error = "malformed record header"; return; }
        const uint8_t* he = e;
        while (he > p + 1 && (he[-1] == '\r' || he[-1] == ' ')) --he;
        R.names.append((const char*)p + 1, (size_t)(he - p - 1));
        R.name_off.push_back(R.names.size());
        p = e < end ? e + 1 : end;
        const uint64_t seq_begin = w;
        if (!fastq) {
            while (p < end && *p != '>') {
                e = line_end(p, end);
                w = put_trimmed(dst, w, p, e);
                p = e < end ? e + 1 : end;
            }
        } else {
            while (p < end && *p != '+') {                           // sequence lines up to the '+' line
                e = line_end(p, end);
                w = put_trimmed(dst, w, p, e);
                p = e < end ? e + 1 : end;
            }
            if (p < end) { e = line_end(p, end); p = e < end ? e + 1 : end; }   // '+' line
            uint64_t need = w - seq_begin, got = 0;                 // quality: as many symbols as bases
            while (p < end && got < need) {
                e = line_end(p, end);
                const uint8_t* qe = e;
                while (qe > p && (qe[-1] == '\r')) --qe;
                got += (uint64_t)(qe - p);
                p = e < end ? e + 1 : end;
            }
        }
        R.start.push_back(seq_begin);
        R.len.push_back(w - seq_begin);
    }
    R.used = w;
}

// One page-locked staging buffer is kept between calls: pinning hundreds of MB costs far more
// than filling them, and sketching runs are repeated over similar-sized batches.
std::mutex g_pin_mu;
uint8_t* g_pin_buf = nullptr;
size_t g_pin_cap = 0;

uint8_t* pinned_acquire(size_t bytes, size_t& cap) {
    {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        if (g_pin_buf && g_pin_cap >= bytes) {
            uint8_t* p = g_pin_buf; cap = g_pin_cap;
            g_pin_buf = nullptr; g_pin_cap = 0;
            return p;
        }
        if (g_pin_buf) { cudaFreeHost(g_pin_buf); g_pin_buf = nullptr; g_pin_cap = 0; }
    }
    uint8_t* p = nullptr;
    cap = (bytes + (bytes >> 3) + (1u << 20)) & ~size_t(4095);
    if (cudaHostAlloc((void**)&p, cap, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void pinned_release(uint8_t* p, size_t cap) {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    if (!g_pin_buf) { g_pin_buf = p; g_pin_cap = cap; return; }
    if (cap > g_pin_cap) { cudaFreeHost(g_pin_buf); g_pin_buf = p; g_pin_cap = cap; return; }
    cudaFreeHost(p);
}

template <class F>
void run_parallel(size_t n_items, size_t nt, F&& fn) {
    std::atomic<size_t> next{0};
    auto worker = [&] { for (;;) { size_t i = next.fetch_add(1); if (i >= n_items) return; fn(i); } };
    nt = std::min(std::max<size_t>(nt, 1), std::max<size_t>(n_items, 1));
    std::vector<std::thread> pool;
    for (size_t t = 1; t < nt; ++t) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
}

}  // namespace

RecordBatch::~RecordBatch() {
    if (seqs) { if (pinned) pinned_release(seqs, cap); else free(seqs); }
}

std::string read_sequence_files(const char* const* paths, size_t n_paths, int n_threads, bool want_pinned,
                                RecordBatch& out) {
    const size_t nt = (size_t)std::max(1, n_threads);
    // 1. every file into memory (mmap / inflate), in parallel
    std::vector<Loaded> loaded(n_paths);
    run_parallel(n_paths, nt, [&](size_t i) { load_file(paths[i], loaded[i]); });
    for (auto& l : loaded) if (!l.error.empty()) return l.error;
    // 2. one destination buffer; file i owns a region as large as the file (sequence bytes never
    //    outgrow it), 16-byte aligned.  Gaps between regions are never read as sequence.
    std::vector<uint64_t> base(n_paths + 1, 0);
    for (size_t i = 0; i < n_paths; ++i) base[i + 1] = (base[i] + loaded[i].n + 15) & ~15ull;
    const size_t need = (size_t)base[n_paths] + 64;
    out.pinned = false;
    if (want_pinned) { out.seqs = pinned_acquire(need, out.cap); out.pinned = out.seqs != nullptr; }
    if (!out.seqs) { out.cap = (need + 4095) & ~size_t(4095); out.seqs = (uint8_t*)aligned_alloc(4096, out.cap); }
    if (!out.seqs) return "out of host memory";
    // 3. parse straight into the regions, in parallel
    std::vector<FileRecords> files(n_paths);
    run_parallel(n_paths, nt, [&](size_t i) {
        parse_records(loaded[i].p, loaded[i].n, out.seqs + base[i], files[i]);
        if (!files[i].error.empty()) files[i].error = std::string(paths[i]) + ": " + files[i].error;
        // zero the tail of the region so that the buffer holds no stale bytes
        memset(out.seqs + base[i] + files[i].used, 0, (size_t)(base[i + 1] - base[i] - files[i].used));
    });
    for (auto& f : files) if (!f.error.empty()) return f.error;
    memset(out.seqs + base[n_paths], 0, 64);
    // 4. record table
    uint64_t n_rec = 0, name_bytes = 0, seq_bytes = 0;
    for (auto& f : files) { n_rec += f.start.size(); name_bytes += f.names.size(); }
    out.start.clear(); out.start.reserve(n_rec);
    out.len.clear(); out.len.reserve(n_rec);
    out.file.clear(); out.file.reserve(n_rec);
    out.names.clear(); out.names.reserve(name_bytes);
    out.name_off.assign(1, 0); out.name_off.reserve(n_rec + 1);
    for (size_t i = 0; i < n_paths; ++i) {
        const FileRecords& f = files[i];
        for (size_t r = 0; r < f.start.size(); ++r) {
            out.start.push_back(base[i] + f.start[r]);
            out.len.push_back(f.len[r]);
            seq_bytes += f.len[r];
            out.file.push_back((uint32_t)i);
            out.name_off.push_back(out.names.size() + f.name_off[r + 1]);
        }
        out.names += f.names;
    }
    out.extent = base[n_paths];
    out.total = seq_bytes;
    return "";
}

// =============================================================================================
// .sig JSON
// =============================================================================================
namespace {

struct Json {
    const char* p;
    const char* end;
    std::string err;
    bool fail(const char* m) { if (err.empty()) err = m; return false; }
    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) ++p; }
    bool lit(char c) { ws(); if (p < end && *p == c) { ++p; return true; } return false; }
    bool expect(char c) { return lit(c) ? true : fail("malformed JSON"); }

    bool string(std::string& out) {
        ws();
        if (p >= end || *p != '"') return fail("expected a string");
        ++p;
        out.clear();
        while (p < end && *p != '"') {
            if (*p != '\\') { out.push_back(*p++); continue; }
            if (++p >= end) break;
            switch (*p++) {
                case 'n': out.push_back('\n'); break;
                case 't': out.push_back('\t'); break;
                case 'r': out.push_back('\r'); break;
                case 'b': out.push_back('\b'); break;
                case 'f': out.push_back('\f'); break;
                case 'u': {
                    if (end - p < 4) return fail("bad \\u escape");
                    unsigned cp = (unsigned)strtoul(std::string(p, 4).c_str(), nullptr, 16);
                    p += 4;
                    if (cp >= 0xD800 && cp < 0xDC00 && end - p >= 6 && p[0] == '\\' && p[1] == 'u') {
                        unsigned lo = (unsigned)strtoul(std::string(p + 2, 4).c_str(), nullptr, 16);
                        p += 6;
                        cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                    }
                    if (cp < 0x80) out.push_back((char)cp);
                    else if (cp < 0x800) { out.push_back((char)(0xC0 | (cp >> 6))); out.push_back((char)(0x80 | (cp & 63))); }
                    else if (cp < 0x10000) { out.push_back((char)(0xE0 | (cp >> 12))); out.push_back((char)(0x80 | ((cp >> 6) & 63))); out.push_back((char)(0x80 | (cp & 63))); }
                    else { out.push_back((char)(0xF0 | (cp >> 18))); out.push_back((char)(0x80 | ((cp >> 12) & 63))); out.push_back((char)(0x80 | ((cp >> 6) & 63))); out.push_back((char)(0x80 | (cp & 63))); }
                    break;
                }
                default: out.push_back(p[-1]);
            }
        }
        if (p >= end) return fail("unterminated string");
        ++p;
        return true;
    }
    bool u64(uint64_t& v) {
        ws();
        if (p >= end || *p < '0' || *p > '9') return fail("expected an unsigned integer");
        uint64_t x = 0;
        while (p < end && *p >= '0' && *p <= '9') x = x * 10 + (uint64_t)(*p++ - '0');
        if (p < end && (*p == '.' || *p == 'e' || *p == 'E')) {       // tolerate 1.0-style integers
            while (p < end && (*p == '.' || *p == 'e' || *p == 'E' || *p == '+' || *p == '-' || (*p >= '0' && *p <= '9'))) ++p;
        }
        v = x;
        return true;
    }
    bool number(double& v) {
        ws();
        // the buffer need not be NUL-terminated (mapped files, zip members): parse a bounded copy of the token
        char tok[64];
        size_t m = 0;
        while (p + m < end && m + 1 < sizeof tok &&
               ((p[m] >= '0' && p[m] <= '9') || p[m] == '+' || p[m] == '-' || p[m] == '.' || p[m] == 'e' || p[m] == 'E')) {
            tok[m] = p[m];
            ++m;
        }
        tok[m] = 0;
        char* e = nullptr;
        v = strtod(tok, &e);
        if (e == tok) return fail("expected a number");
        p += e - tok;
        return true;
    }
    bool u64_array(std::vector<uint64_t>& dst) {
        if (!expect('[')) return false;
        if (lit(']')) return true;
        for (;;) {
            uint64_t v;
            if (!u64(v)) return false;
            dst.push_back(v);
            if (lit(',')) continue;
            return expect(']');
        }
    }
    int depth = 0;                                  // nesting of skip(): hostile input cannot exhaust the stack
    bool skip() {                                   // any value
        struct Level { int& d; explicit Level(int& x) : d(x) { ++d; } ~Level() { --d; } } level(depth);
        if (depth > 256) return fail("JSON nested too deeply");
        ws();
        if (p >= end) return fail("unexpected end of JSON");
        if (*p == '"') { std::string s; return string(s); }
        if (*p == '{' || *p == '[') {
            const char open = *p, close = open == '{' ? '}' : ']';
            ++p;
            if (lit(close)) return true;
            for (;;) {
                if (open == '{') { std::string k; if (!string(k) || !expect(':')) return false; }
                if (!skip()) return false;
                if (lit(',')) continue;
                return expect(close);
            }
        }
        while (p < end && *p != ',' && *p != '}' && *p != ']' && *p != ' ' && *p != '\n') ++p;   // number / literal
        return true;
    }
    bool null_or_string(std::string& s, bool& present) {
        ws();
        if (end - p >= 4 && !memcmp(p, "null", 4)) { p += 4; present = false; return true; }
        present = true;
        return string(s);
    }
};

bool parse_sketch(Json& J, SigBatch& B, uint32_t sig_index, uint32_t file) {
    SigSketch sk;
    sk.sig_index = sig_index; sk.file = file;
    std::vector<uint64_t> mins, abunds;
    std::string molecule = "dna", key;
    bool have_abund = false;
    if (!J.expect('{')) return false;
    if (!J.lit('}')) for (;;) {
        if (!J.string(key) || !J.expect(':')) return false;
        uint64_t v = 0;
        if (key == "num") { if (!J.u64(v)) return false; sk.num = (uint32_t)v; }
        else if (key == "ksize") { if (!J.u64(v)) return false; sk.ksize = (uint32_t)v; }
        else if (key == "seed") { if (!J.u64(sk.seed)) return false; }
        else if (key == "max_hash") { if (!J.u64(sk.max_hash)) return false; }
        else if (key == "md5sum") { if (!J.string(sk.md5sum)) return false; }
        else if (key == "molecule") { if (!J.string(molecule)) return false; }
        else if (key == "mins") { if (!J.u64_array(mins)) return false; }
        else if (key == "abundances") {
            J.ws();
            if (J.end - J.p >= 4 && !memcmp(J.p, "null", 4)) J.p += 4;
            else { have_abund = true; if (!J.u64_array(abunds)) return false; }
        } else if (!J.skip()) return false;
        if (J.lit(',')) continue;
        if (!J.expect('}')) return false;
        break;
    }
    for (auto& c : molecule) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    if (molecule == "dna") sk.hash_function = 1;
    else if (molecule == "protein") sk.hash_function = 2;
    else if (molecule == "dayhoff") sk.hash_function = 3;
    else if (molecule == "hp") sk.hash_function = 4;
    else return J.fail("unknown molecule type");
    if (sk.max_hash != 0) sk.num = 0;                                   // minhash.rs:146
    if (have_abund && abunds.size() != mins.size()) return J.fail("mins and abundances differ in length");
    sk.has_abund = have_abund;
    // minhash.rs:159-171: files with unsorted mins exist; sort (pairs when abundances are present)
    if (!std::is_sorted(mins.begin(), mins.end())) {
        if (have_abund) {
            std::vector<std::pair<uint64_t, uint64_t>> v(mins.size());
            for (size_t i = 0; i < mins.size(); ++i) v[i] = {mins[i], abunds[i]};
            std::sort(v.begin(), v.end());
            for (size_t i = 0; i < mins.size(); ++i) { mins[i] = v[i].first; abunds[i] = v[i].second; }
        } else {
            std::sort(mins.begin(), mins.end());
        }
    }
    B.mins.insert(B.mins.end(), mins.begin(), mins.end());
    if (have_abund) B.abunds.insert(B.abunds.end(), abunds.begin(), abunds.end());
    else B.abunds.insert(B.abunds.end(), mins.size(), 1);
    B.any_abund = B.any_abund || have_abund;
    B.off.push_back(B.mins.size());
    B.sketches.push_back(std::move(sk));
    return true;
}

bool parse_signature(Json& J, SigBatch& B, uint32_t file) {
    SigRecord rec;
    rec.file = file; rec.license = "CC0"; rec.klass = "sourmash_signature";
    const uint32_t sig_index = (uint32_t)B.sigs.size();
    B.sigs.push_back(rec);                                             // sketches refer to it by index
    std::string key;
    if (!J.expect('{')) return false;
    if (!J.lit('}')) for (;;) {
        if (!J.string(key) || !J.expect(':')) return false;
        SigRecord& r = B.sigs[sig_index];
        if (key == "signatures") {
            if (!J.expect('[')) return false;
            if (!J.lit(']')) for (;;) {
                if (!parse_sketch(J, B, sig_index, file)) return false;
                if (J.lit(',')) continue;
                if (!J.expect(']')) return false;
                break;
            }
        } else if (key == "name") { if (!J.null_or_string(r.name, r.has_name)) return false; }
        else if (key == "filename") { if (!J.null_or_string(r.filename, r.has_filename)) return false; }
        else if (key == "license") { if (!J.string(r.license)) return false; }
        else if (key == "email") { if (!J.string(r.email)) return false; }
        else if (key == "class") { if (!J.string(r.klass)) return false; }
        else if (key == "hash_function") { if (!J.string(r.hash_function)) return false; }
        else if (key == "version") { if (!J.number(r.version)) return false; }
        else if (!J.skip()) return false;
        if (J.lit(',')) continue;
        if (!J.expect('}')) return false;
        break;
    }
    return true;
}

}  // namespace

std::string parse_signature_json(const char* text, size_t len, uint32_t file_index, SigBatch& B) {
    if (B.off.empty()) B.off.push_back(0);
    Json J{text, text + len, ""};
    J.ws();
    if (J.p < J.end && *J.p == '[') {
        ++J.p;
        if (!J.lit(']')) for (;;) {
            if (!parse_signature(J, B, file_index)) return J.err;
            if (J.lit(',')) continue;
            if (!J.expect(']')) return J.err;
            break;
        }
    } else if (!parse_signature(J, B, file_index)) {
        return J.err;
    }
    return J.err;
}

std::string parse_lca_hashvals(const char* text, size_t len, std::vector<uint64_t>& hashes, std::vector<uint32_t>& idx,
                               int64_t* begin, int64_t* end) {
    Json J{text, text + len, ""};
    *begin = *end = -1;
    std::string key;
    if (!J.expect('{')) return J.err;
    if (!J.lit('}')) for (;;) {
        if (!J.string(key) || !J.expect(':')) return J.err;
        if (key != "hashval_to_idx") {
            if (!J.skip()) return J.err;
        } else {
            J.ws();
            *begin = J.p - text;
            if (!J.expect('{')) return J.err;
            if (!J.lit('}')) for (;;) {
                std::string hk;
                if (!J.string(hk) || !J.expect(':')) return J.err;
                uint64_t h = 0;
                if (hk.empty() || hk.size() > 20) return "hash key is not a 64-bit unsigned integer";
                for (char c : hk) {
                    if (c < '0' || c > '9') return "hash key is not a 64-bit unsigned integer";
                    const uint64_t d = (uint64_t)(c - '0');
                    if (h > (UINT64_MAX - d) / 10) return "hash key is not a 64-bit unsigned integer";
                    h = h * 10 + d;
                }
                if (!J.expect('[')) return J.err;
                if (!J.lit(']')) for (;;) {
                    uint64_t v;
                    if (!J.u64(v)) return J.err;
                    if (v > UINT32_MAX) return "idx out of range";
                    hashes.push_back(h);
                    idx.push_back((uint32_t)v);
                    if (J.lit(',')) continue;
                    if (!J.expect(']')) return J.err;
                    break;
                }
                if (J.lit(',')) continue;
                if (!J.expect('}')) return J.err;
                break;
            }
            *end = J.p - text;
        }
        if (J.lit(',')) continue;
        if (!J.expect('}')) return J.err;
        break;
    }
    return J.err;
}

// md5 of one parsed sketch, the identity manifests list (KmerMinHash::md5sum, minhash.rs:290-307:
// the decimal ksize followed by every hash in decimal)
std::string sketch_md5(uint32_t ksize, const uint64_t* mins, size_t n) {
    Md5 ctx;
    char buf[4096];
    size_t fill = (size_t)snprintf(buf, sizeof buf, "%u", ksize);
    for (size_t i = 0; i < n; ++i) {
        if (fill > sizeof buf - 24) { ctx.update((const uint8_t*)buf, fill); fill = 0; }
        char tmp[24];
        int len = 0;
        uint64_t v = mins[i];
        do { tmp[len++] = (char)('0' + v % 10); v /= 10; } while (v);
        while (len) buf[fill++] = tmp[--len];
    }
    ctx.update((const uint8_t*)buf, fill);
    return ctx.hexdigest();
}

namespace {

// keep only the sketches whose md5 the manifest lists (`if ss in manifest`, index/__init__.py:651-657);
// signature records left without a sketch go too
void keep_listed(SigBatch& B, const std::unordered_set<std::string>& md5s) {
    const size_t n = B.sketches.size();
    std::vector<char> keep(n);
    bool all = true;
    for (size_t i = 0; i < n; ++i) {
        const uint64_t lo = B.off[i], hi = B.off[i + 1];
        keep[i] = md5s.count(sketch_md5(B.sketches[i].ksize, B.mins.data() + lo, (size_t)(hi - lo))) != 0;
        all = all && keep[i];
    }
    if (all) return;
    SigBatch R;
    R.off.push_back(0);
    std::vector<int64_t> new_sig(B.sigs.size(), -1);
    for (size_t i = 0; i < n; ++i) {
        if (!keep[i]) continue;
        SigSketch sk = std::move(B.sketches[i]);
        if (new_sig[sk.sig_index] < 0) { new_sig[sk.sig_index] = (int64_t)R.sigs.size(); R.sigs.push_back(std::move(B.sigs[sk.sig_index])); }
        sk.sig_index = (uint32_t)new_sig[sk.sig_index];
        R.mins.insert(R.mins.end(), B.mins.begin() + (ptrdiff_t)B.off[i], B.mins.begin() + (ptrdiff_t)B.off[i + 1]);
        R.abunds.insert(R.abunds.end(), B.abunds.begin() + (ptrdiff_t)B.off[i], B.abunds.begin() + (ptrdiff_t)B.off[i + 1]);
        R.off.push_back(R.mins.size());
        R.any_abund = R.any_abund || sk.has_abund;
        R.sketches.push_back(std::move(sk));
    }
    B = std::move(R);
}

bool ends_with(const std::string& s, const char* suffix) {
    const size_t n = strlen(suffix);
    return s.size() >= n && !memcmp(s.data() + s.size() - n, suffix, n);
}

struct ZipInput {                       // one .zip path: the mapped archive and what its manifest lists
    ZipArchive zip;
    bool has_manifest = false;
    std::unordered_set<std::string> md5s;
};
struct SigTask { uint32_t path; const ZipMember* member; const ZipInput* zin; };   // member == nullptr: the file itself

}  // namespace

std::string read_signature_files(const char* const* paths, size_t n_paths, int n_threads, uint32_t flags, SigBatch& out,
                                 const uint8_t* loose) {
    // 1. classify: a .zip collection expands into one task per member, in the order the reference
    //    visits them -- the manifest's distinct locations when SOURMASH-MANIFEST.csv exists
    //    (index/__init__.py:644-657), else every member named *.sig / *.sig.gz in directory
    //    order (index/__init__.py:659-683)
    std::vector<std::unique_ptr<ZipInput>> zips(n_paths);
    std::vector<SigTask> tasks;
    tasks.reserve(n_paths);
    for (size_t i = 0; i < n_paths; ++i) {
        if (loose && loose[i]) { tasks.push_back({(uint32_t)i, nullptr, nullptr}); continue; }
        unsigned char magic[4] = {0, 0, 0, 0};
        FILE* fh = fopen(paths[i], "rb");
        if (!fh) return std::string("cannot open ") + paths[i];
        const size_t got = fread(magic, 1, 4, fh);
        fclose(fh);
        if ((flags & SIGS_NO_ZIP) || !ZipArchive::has_magic(magic, got)) { tasks.push_back({(uint32_t)i, nullptr, nullptr}); continue; }
        zips[i] = std::make_unique<ZipInput>();
        ZipInput& Z = *zips[i];
        std::string e = Z.zip.open(paths[i]);
        if (!e.empty()) return e;
        const ZipMember* mf = (flags & SIGS_NO_MANIFEST) ? nullptr : Z.zip.find("SOURMASH-MANIFEST.csv");
        if (mf) {
            std::string text;
            ManifestIndex M;
            e = Z.zip.read(*mf, text);
            if (e.empty()) e = parse_manifest_csv(text, M);
            if (!e.empty()) return std::string(paths[i]) + ": " + e;
            Z.has_manifest = true;
            Z.md5s.insert(M.md5s.begin(), M.md5s.end());
            for (const auto& loc : M.locations) {
                const ZipMember* m = Z.zip.find(loc);
                if (!m) return std::string(paths[i]) + ": manifest lists '" + loc + "', which is not in the archive";
                tasks.push_back({(uint32_t)i, m, &Z});
            }
        } else {
            for (const auto& m : Z.zip.members) {
                if (m.is_dir()) continue;
                if ((flags & SIGS_ALL_MEMBERS) || ends_with(m.name, ".sig") || ends_with(m.name, ".sig.gz"))
                    tasks.push_back({(uint32_t)i, &m, &Z});
            }
        }
    }
    // 2. parse: one task at a time per thread
    const size_t n_tasks = tasks.size();
    std::vector<SigBatch> parts(n_tasks);
    std::vector<std::string> errs(n_tasks);
    std::atomic<size_t> next{0};
    auto worker = [&] {
        std::string raw, text;
        for (;;) {
            const size_t t = next.fetch_add(1);
            if (t >= n_tasks) return;
            const SigTask& T = tasks[t];
            const char* path = paths[T.path];
            if (!T.member) {
                Bytes data;
                errs[t] = slurp(path, data);
                if (errs[t].empty()) {
                    errs[t] = parse_signature_json((const char*)data.data(), data.size(), T.path, parts[t]);
                    if (!errs[t].empty()) errs[t] = std::string(path) + ": " + errs[t];
                }
                if (!errs[t].empty() && loose && loose[T.path]) { errs[t].clear(); parts[t] = SigBatch(); }
                continue;
            }
            raw.clear(); text.clear();
            errs[t] = T.zin->zip.read(*T.member, raw);
            if (!errs[t].empty()) { errs[t] = std::string(path) + ": " + errs[t]; continue; }
            // a member that does not hold signatures is passed over, like load_signatures_from_json
            // without do_raise (src/sourmash/signature.py:350-380,412-418,466-468)
            const std::string* doc = &raw;
            if (raw.size() >= 2 && (uint8_t)raw[0] == 0x1f && (uint8_t)raw[1] == 0x8b) {
                if (!inflate_all((const uint8_t*)raw.data(), raw.size(), 15 + 32, 0, text).empty()) continue;
                doc = &text;
            } else if (raw.find("sourmash_signature") == std::string::npos) {
                continue;
            }
            if (!parse_signature_json(doc->data(), doc->size(), T.path, parts[t]).empty()) { parts[t] = SigBatch(); continue; }
            if (T.zin->has_manifest) keep_listed(parts[t], T.zin->md5s);
            for (auto& s : parts[t].sigs) s.location = T.member->name;
        }
    };
    size_t nt = std::min<size_t>((size_t)std::max(1, n_threads), std::max<size_t>(n_tasks, 1));
    std::vector<std::thread> pool;
    for (size_t t = 1; t < nt; ++t) pool.emplace_back(worker);
    worker();
    for (auto& t : pool) t.join();
    for (auto& e : errs) if (!e.empty()) return e;
    // 3. concatenate in task order
    if (out.off.empty()) out.off.push_back(0);
    size_t tot = 0, nsk = 0;
    for (auto& p : parts) { tot += p.mins.size(); nsk += p.sketches.size(); }
    out.mins.reserve(out.mins.size() + tot);
    out.abunds.reserve(out.abunds.size() + tot);
    out.sketches.reserve(out.sketches.size() + nsk);
    for (auto& p : parts) {
        const uint32_t sig_base = (uint32_t)out.sigs.size();
        const uint64_t h_base = out.mins.size();
        for (auto& s : p.sigs) out.sigs.push_back(std::move(s));
        for (auto& sk : p.sketches) { sk.sig_index += sig_base; out.sketches.push_back(std::move(sk)); }
        for (size_t r = 1; r < p.off.size(); ++r) out.off.push_back(h_base + p.off[r]);
        out.mins.insert(out.mins.end(), p.mins.begin(), p.mins.end());
        out.abunds.insert(out.abunds.end(), p.abunds.begin(), p.abunds.end());
        out.any_abund = out.any_abund || p.any_abund;
        SigBatch().mins.swap(p.mins);                    // give the part's memory back as we go
        SigBatch().abunds.swap(p.abunds);
    }
    return "";
}

}  // namespace smb
