// ingest.h -- native host-side readers that feed the GPU paths without per-record Python:
//   * FASTA / FASTQ (optionally gzip) -> concatenated sequence bytes + record table
//     (replaces the screed record loop of src/sourmash/command_sketch.py:697-766)
//   * sourmash .sig JSON (optionally gzip) -> CSR of sketches + per-sketch metadata
//     (replaces per-object loading through signature.py:383-527 / ffi/signature.rs:219-343;
//      format: src/core/src/signature.rs:401-445, sketch fields sketch/minhash.rs:103-184)
// Internal C++ interface; the public boundary is include/sourmash_b200.h (smb_records_*, smb_sigs_*).
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

namespace smb {

struct RecordBatch {
    uint8_t* seqs = nullptr;            // one buffer; every file owns a 16-byte aligned region of it
    size_t cap = 0;                     // allocated bytes
    uint64_t extent = 0;                // bytes of the buffer in use (what gets uploaded)
    uint64_t total = 0;                 // sum of the record lengths
    bool pinned = false;                // page-locked (taken from / returned to a one-buffer pool)
    std::vector<uint64_t> start, len;   // [n] byte offset and length of every record
    std::vector<uint32_t> file;         // [n] index of the input file
    std::string names;                  // header lines back to back
    std::vector<uint64_t> name_off;     // [n + 1]
    ~RecordBatch();
};

// Reads every file (FASTA or FASTQ, plain or gzip, decided per file from its content) with up to
// n_threads worker threads, records in input order.  Returns an error message, empty on success.
std::string read_sequence_files(const char* const* paths, size_t n_paths, int n_threads, bool want_pinned,
                                RecordBatch& out);

struct SigSketch {
    uint32_t sig_index = 0;             // which signature object of which file it came from
    uint32_t file = 0;
    uint32_t ksize = 0, num = 0;        // ksize as stored in the file (3 x residues for proteins)
    uint64_t max_hash = 0, seed = 42;
    uint32_t hash_function = 1;         // 1 dna, 2 protein, 3 dayhoff, 4 hp
    bool has_abund = false;
    std::string md5sum;
};
struct SigRecord {                      // one signature object (signature.rs:401-445)
    uint32_t file = 0;
    std::string name, filename, license, email, klass, hash_function;
    std::string location;               // member name when the file is a .zip collection (internal_location)
    double version = 0.4;
    bool has_name = false, has_filename = false;
};
struct SigBatch {
    std::vector<SigRecord> sigs;
    std::vector<SigSketch> sketches;
    std::vector<uint64_t> off;          // [n_sketches + 1] into mins / abunds
    std::vector<uint64_t> mins;         // each row sorted ascending (loader re-sorts, minhash.rs:159-171)
    std::vector<uint64_t> abunds;       // parallel to mins; 1 where a sketch has no abundances
    bool any_abund = false;
};

// Parses .sig / .sig.gz files (JSON array of signatures, or one signature object) and .zip
// collections of them (zipread.h; members in the order ZipFileLinearIndex.signatures() visits them).
enum : uint32_t {
    SIGS_NO_MANIFEST = 1,   // ignore SOURMASH-MANIFEST.csv (ZipFileLinearIndex use_manifest=False)
    SIGS_ALL_MEMBERS = 2,   // without a manifest, try every member, not only *.sig / *.sig.gz (traverse_yield_all)
    SIGS_NO_ZIP = 4,        // every path is one (possibly compressed) JSON file: a .zip archive is a parse error, as it is for
                            // the reference's Signature::from_path (signature.rs:569-590) behind signatures_load_path
};
// optional: a path i with loose[i] != 0 is read as one JSON file whatever its contents, and contributes nothing when
// it cannot be read or parsed (MultiIndex.load_from_directory with force, index/__init__.py:1033-1045)
std::string read_signature_files(const char* const* paths, size_t n_paths, int n_threads, uint32_t flags,
                                 SigBatch& out, const uint8_t* loose = nullptr);
// md5 identity of a sketch (KmerMinHash::md5sum, minhash.rs:290-307)
std::string sketch_md5(uint32_t ksize, const uint64_t* mins, size_t n);
// Same from memory (one document).
std::string parse_signature_json(const char* text, size_t len, uint32_t file_index, SigBatch& out);

// The "hashval_to_idx" member of an LCA database's top-level JSON object ({"<hash>": [idx, ...], ...}, the only large
// table of the format; LCA_Database.load, lca_db.py:384-391) as one (hash, idx) pair per listed idx, in file order.
// *begin / *end: the byte span of the member's value, so that the caller can parse the rest of the document without
// it; both -1 when the object has no such member.  Other members are scanned over, not kept.
std::string parse_lca_hashvals(const char* text, size_t len, std::vector<uint64_t>& hashes, std::vector<uint32_t>& idx,
                               int64_t* begin, int64_t* end);

}  // namespace smb
