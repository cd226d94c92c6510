// common.cuh -- shared device/host helpers for the sm_90a kernels of sourmash_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

typedef uint64_t u64;
typedef uint32_t u32;
typedef uint16_t u16;
typedef uint8_t u8;

#define SMB_U64_MAX 0xffffffffffffffffULL

// Number of SMs on an H100 SXM; grids for persistent-style kernels are sized in multiples of it.
#define SMB_SMS 132

// L2 cache of the devices the library is built for (sm_90a: H100 SXM / PCIe, H200, GH200 all have 50 MB); sizes
// the windows that keep scattered writes L2-resident.
#define SMB_L2_BYTES (50ull * 1024 * 1024)

// Shared memory of kernels that tests/host_emul/simt.h also runs on the CPU (SMB_SIMT_EMUL: one CTA at a
// time as cooperative fibers, so block-shared storage is plain static storage there).
#ifdef SMB_SIMT_EMUL
#define SMB_SHARED static
#define SMB_DYN_SHARED(T, name) T* name = reinterpret_cast<T*>(smb_emu::dyn_smem())
#else
#define SMB_SHARED __shared__
#define SMB_DYN_SHARED(T, name) extern __shared__ __align__(16) T name[]
#endif

#ifdef __CUDACC__
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ u64 ld_nc_u64(const u64* p) {
    return __ldg(reinterpret_cast<const unsigned long long*>(p));
}
#endif

// Streaming accesses (evict-first): data that is read or written exactly once should not push the reused
// working set (the tag stream of the stripe join, a query bitmap) out of L2.
#ifdef SMB_SIMT_EMUL
inline u32 ld_stream_u32(const u32* p) { return *p; }
inline u64 ld_stream_u64(const u64* p) { return *p; }
inline ulonglong2 ld_stream_u64x2(const ulonglong2* p) { return *p; }
inline void st_stream_f64(double* p, double v) { *p = v; }
#elif defined(__CUDACC__)
__device__ __forceinline__ ulonglong2 ld_stream_u64x2(const ulonglong2* p) { return __ldcs(p); }
__device__ __forceinline__ u32 ld_stream_u32(const u32* p) { return __ldcs(p); }
__device__ __forceinline__ u64 ld_stream_u64(const u64* p) { return __ldcs(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ void st_stream_f64(double* p, double v) { __stcs(p, v); }
#endif

// MurmurHash3 x64-128 building blocks (device + host), see murmur.cuh.
__host__ __device__ __forceinline__ u64 smb_rotl64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
__host__ __device__ __forceinline__ u64 smb_fmix64(u64 x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33; return x;
}
#define SMB_C1 0x87c37b91114253d5ULL
#define SMB_C2 0x4cf5ad432745937fULL
