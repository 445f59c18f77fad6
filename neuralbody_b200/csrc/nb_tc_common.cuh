// Helpers shared by the dense and the sparse (empty-sample-skipping) tensor-core render kernels.
#pragma once
#include "nb_device.cuh"
#include "nb_tc_ptx.cuh"

namespace nb {
namespace tcr {

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void sts_v2(uint32_t addr, uint2 v) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}

// Diagnostics: CTA 0 records (code << 48 | clock) per role into P.trace[role * 4096 + n] (first ~40 tiles).
struct Tracer {
    unsigned long long* buf;
    int n;
    __device__ __forceinline__ void init(unsigned long long* base, int role) {
        buf = (base && blockIdx.x == 0) ? base + role * 4096 : nullptr;
        n = 0;
    }
    __device__ __forceinline__ void ev(int code) { val(code, (unsigned long long)clock64()); }
    // an event that carries a value (e.g. cycles spent waiting) in place of the clock
    __device__ __forceinline__ void val(int code, unsigned long long v) {
        if (buf && n < 4096) buf[n++] = ((unsigned long long)code << 48) | (v & 0xFFFFFFFFFFFFull);
    }
};

// Gather granule: one lane accumulates 4 consecutive channels of one corner vector; the 8 lanes of a group
// cover a 32-channel unit, so a group's load of one corner is one contiguous 128-byte (fp32) / 64-byte (fp16)
// run = a single L1 wavefront, instead of 8 scattered 16-byte pieces.
template <typename VT> struct Quad;
template <> struct Quad<float> {
    using raw = uint4;
    static __device__ __forceinline__ raw zero() { return make_uint4(0u, 0u, 0u, 0u); }
    static __device__ __forceinline__ raw load_bytes(const unsigned char* p) { return ldg_nc_v4(p); }
    static __device__ __forceinline__ raw load_shared(uint32_t addr) {
        uint4 r;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
        return r;
    }
    static __device__ __forceinline__ void fma(float (&a)[4], const raw& v, float w) {
        a[0] = fmaf(__uint_as_float(v.x), w, a[0]); a[1] = fmaf(__uint_as_float(v.y), w, a[1]);
        a[2] = fmaf(__uint_as_float(v.z), w, a[2]); a[3] = fmaf(__uint_as_float(v.w), w, a[3]);
    }
};
template <> struct Quad<__half> {
    using raw = uint2;
    static __device__ __forceinline__ raw zero() { return make_uint2(0u, 0u); }
    static __device__ __forceinline__ raw load(const __half* p) {
        uint2 r;
        asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        return r;
    }
    static __device__ __forceinline__ raw load_bytes(const unsigned char* p) { return load(reinterpret_cast<const __half*>(p)); }
    static __device__ __forceinline__ raw load_shared(uint32_t addr) {
        uint2 r;
        asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(addr) : "memory");
        return r;
    }
    static __device__ __forceinline__ void fma(float (&a)[4], const raw& v, float w) {
        const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
        const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        a[0] = fmaf(f0.x, w, a[0]); a[1] = fmaf(f0.y, w, a[1]);
        a[2] = fmaf(f1.x, w, a[2]); a[3] = fmaf(f1.y, w, a[3]);
    }
};

}  // namespace tcr
}  // namespace nb
