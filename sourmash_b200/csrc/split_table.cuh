// split_table.cuh -- the shared-memory "table" of the intersection kernel and its probes.
// __host__ __device__ so that tests/host_emul can run exactly this code on the CPU.
//
// A table is one sorted-unique row of u64 keys (< 2^64-1, at most 32 759 of them) stored as
//   lo[p], hi[p]   low / high 32-bit words of key p (two sentinel entries 0xffffffff follow),
//   dir[b]         (start << 1) | crowded, for bucket b = key >> shift, b in [0, nb]:
//                  start = number of keys whose bucket is < b, crowded = 1 iff >= 3 keys share b.
// Building runs in three phases separated by a barrier; `tid` of `nthreads` cooperating workers.
#pragma once
#include "common.cuh"

namespace smb {

struct SplitTable {
    const u32* lo;
    const u32* hi;
    const u16* dir;
};

#ifdef __CUDA_ARCH__
__device__ __forceinline__ u64 table_src_key(const u64* p) { return ld_nc_u64(p); }
#else
inline u64 table_src_key(const u64* p) { return *p; }
#endif

// phase 1: copy the keys, write the sentinels, preset every directory entry to "past the end"
__host__ __device__ __forceinline__ void split_table_load(u32* lo, u32* hi, u16* dir, const u64* keys, int n,
                                                          int nb, int tid, int nthreads) {
    for (int p = tid; p < n; p += nthreads) {
        const u64 k = table_src_key(keys + p);
        lo[p] = (u32)k; hi[p] = (u32)(k >> 32);
    }
    if (tid < 2) { lo[n + tid] = 0xffffffffu; hi[n + tid] = 0xffffffffu; }
    for (int b = tid; b <= nb; b += nthreads) dir[b] = (u16)(n << 1);
}

// phase 2: every key that opens a bucket writes its index into that bucket and the empty ones before it
__host__ __device__ __forceinline__ void split_table_heads(const u32* lo, const u32* hi, u16* dir, int n,
                                                           u32 shift, int tid, int nthreads) {
    for (int p = tid; p < n; p += nthreads) {
        const int bp = (int)((((u64)hi[p] << 32) | lo[p]) >> shift);
        const int bprev = p == 0 ? -1 : (int)((((u64)hi[p - 1] << 32) | lo[p - 1]) >> shift);
        for (int b = bprev + 1; b <= bp; ++b) dir[b] = (u16)(p << 1);
    }
}

// phase 3: crowded flag
__host__ __device__ __forceinline__ void split_table_flags(u16* dir, int nb, int tid, int nthreads) {
    for (int b = tid; b < nb; b += nthreads) {
        const u32 st2 = dir[b] & 0xfffeu, en2 = dir[b + 1] & 0xfffeu;
        dir[b] = (u16)(st2 | (en2 - st2 >= 6u ? 1u : 0u));
    }
}

// fast path of one probe: directory entry + the low words of the bucket's first two slots.
// Returns "a low word matched"; ORs the entry (its bit 0 = crowded) into ov.
__host__ __device__ __forceinline__ bool split_probe_low(const SplitTable& t, u64 q, u32 shift, u32& ov) {
    const u32 ent = t.dir[(u32)(q >> shift)];
    ov |= ent;
    // byte offset of slot 0 = start * 4 = (entry & ~1) * 2: one LOP + one LEA
    const u32* slot = reinterpret_cast<const u32*>(reinterpret_cast<const unsigned char*>(t.lo) +
                                                   ((ent & 0xfffeu) << 1));
    const u32 qlo = (u32)q;
    return (slot[0] == qlo) | (slot[1] == qlo);
}

// exact check of the two slots: high words are read only where a low word matched.  0 or 1.
__host__ __device__ __forceinline__ u32 split_probe_verify(const SplitTable& t, u64 q, u32 shift) {
    const u32 st = (t.dir[(u32)(q >> shift)] & 0xfffeu) >> 1;
    const u32 qlo = (u32)q, qhi = (u32)(q >> 32);
    u32 m = 0;
    if (t.lo[st] == qlo) m |= (t.hi[st] == qhi);
    if (t.lo[st + 1] == qlo) m |= (t.hi[st + 1] == qhi);
    return m;
}

// crowded bucket: continue past the two slots of the fast path.  0 or 1.
__host__ __device__ __forceinline__ u32 split_probe_rest(const SplitTable& t, u64 q, u32 shift) {
    const u32 ent = t.dir[(u32)(q >> shift)];
    if (!(ent & 1u)) return 0;
    u32 p = (ent >> 1) + 2;
    for (;;) {
        const u64 k = ((u64)t.hi[p] << 32) | t.lo[p];
        if (k >= q) return k == q;
        ++p;
    }
}

// position of q in the table, -1 when absent: the fast path's directory entry and low words reject most misses, a
// possible hit or a crowded bucket walks the bucket from its start (the sentinels end the walk)
__host__ __device__ __forceinline__ int split_probe_find(const SplitTable& t, u64 q, u32 shift) {
    u32 ent = 0;
    if (!split_probe_low(t, q, shift, ent) && !(ent & 1u)) return -1;
    for (u32 p = (ent & 0xfffeu) >> 1;; ++p) {
        const u64 k = ((u64)t.hi[p] << 32) | t.lo[p];
        if (k >= q) return k == q ? (int)p : -1;
    }
}

}  // namespace smb
